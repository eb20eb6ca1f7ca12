// The camera ray through a pixel of a reel image, shared by k_random_rays_from_reel (rayops.cu) and the mesh renderer (mesh_raycast.cu),
// so that a trainer drawing a pixel casts exactly the ray whose first hit rendered that pixel. Both units are built with -fmad=false, so
// each product and sum below is rounded as written (PermutoSDFGPU.cuh:24-127).
#pragma once

namespace {
// (sx, sy): the pixel centre, (x + 0.5, y + 0.5); Ki [3,3] and T [4,4] the image's K and tf_world_cam, row-major -> origin o and unit
// direction d (scaled by rsqrtf)
__device__ __forceinline__ void reel_ray(float sx, float sy, const float* __restrict__ Ki, const float* __restrict__ T, float3& o,
                                         float3& d) {
    const float cxp = (sx - Ki[2]) / Ki[0], cyp = (sy - Ki[5]) / Ki[4];
    const float tx = T[3], ty = T[7], tz = T[11];
    const float wx = T[0] * cxp + T[1] * cyp + T[2] + tx;
    const float wy = T[4] * cxp + T[5] * cyp + T[6] + ty;
    const float wz = T[8] * cxp + T[9] * cyp + T[10] + tz;
    const float vx = wx - tx, vy = wy - ty, vz = wz - tz;
    const float inv = rsqrtf(vx * vx + vy * vy + vz * vz);
    o = make_float3(tx, ty, tz);
    d = make_float3(vx * inv, vy * inv, vz * inv);
}
}  // namespace
