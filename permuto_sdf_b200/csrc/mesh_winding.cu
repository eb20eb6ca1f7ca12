// Generalized winding numbers of an indexed triangle mesh (Jacobson et al. 2013) through the BVH of mesh_bvh.cu, with the
// hierarchical far field of Barill et al. 2018 for triangle soups, sm_90a. Built with -fmad=false: each face's solid angle is rounded
// operation by operation as include/psdf_b200.h states it. w(p) = (1/4 pi) sum over faces of the signed solid angle of the face seen from
// p; oracle/winding.py sums the same faces in fp64, so at beta = +inf (no far field) the only difference is the rounding of each term.
//
// Build (psdf_mesh_winding_build): bottom-up over the existing tree, climb of mesh_bvh.cuh as the box refit. Each internal node gets its
// area-weighted centroid c (fp32), the radius r of the sphere about c holding its box, and the moments of its faces about c up to order
// 2: sum A n, sum int (x - c) n^T dA and 1/2 sum int (x - c)(x - c)^T n dA (symmetric in the first two indices, 6 pairs x 3). A leaf's
// moments are integrated exactly; a node's are its children's, child 0 then child 1, shifted to its own c, all in fp64 and stored in
// fp32, so they are the same bits whichever child arrives second.
// Query: one point per thread, depth first, child 0 first. A node whose c is farther than beta r contributes its order-2 expansion;
// otherwise its children are visited; leaves contribute their exact solid angle. Terms are summed in fp64 in that order, rounded once.
//
//   k_wn_build   moments, centroid and radius of every internal node, the second child to arrive going on   thread per leaf
//   k_wn_query   w_out[p] = the sum of exact and far-field terms over the tree / 4 pi                       thread per point
#include "mesh_bvh.cuh"
#include "../../include/psdf_b200.h"

using namespace psdf;

namespace {
constexpr int kSlots = 9;                       // float4 per internal node: (c, r), (sum A n, A), 27 higher moments and a zero
constexpr double kFourPi = 12.566370614359172;

struct WnWs {
    float4* mom;                                // [9 (F - 1)]
    int* flags;                                 // [F - 1] arrivals
};

long long carve_wn(void* ws, long long F, WnWs* W) {
    Sections s{static_cast<char*>(ws)};
    WnWs w;
    const long long ni = F > 1 ? F - 1 : 0;
    s.take(w.mom, 16 * kSlots * ni);
    s.take(w.flags, 4 * ni);
    if (W) *W = w;
    return s.size;
}

// index of the symmetric pair (j, k) in xx, xy, xz, yy, yz, zz
__host__ __device__ constexpr int pair_of(int j, int k) {
    return j > k ? pair_of(k, j) : (j == 0 ? k : (j == 1 ? 2 + k : 5));
}

// cross(p1 - p0, p2 - p0) == 0 in fp32: equal corners (every face that repeats a vertex) or collinear ones. Such a face has no solid
// angle, but its det can round away from 0 while den < 0, and atan2 would then give +-pi
__device__ __forceinline__ bool zero_area(float3 p0, float3 p1, float3 p2) {
    const float3 n = cross3(sub3(p1, p0), sub3(p2, p0));
    return n.x == 0.0f && n.y == 0.0f && n.z == 0.0f;
}
__device__ __forceinline__ double comp(double3 v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : v.z); }
__device__ __forceinline__ double3 to_d(float3 v) { return make_double3(v.x, v.y, v.z); }

// ---------------------------------------------------------------- build
// moments of one face or subtree about the parent's centroid, summed into the parent's
struct Moments {
    double m0[3];
    double m1[9];                               // [j][i]: int (x - c)_j n_i dA
    double m2[18];                              // [pair (j, k)][i]: 1/2 int (x - c)_j (x - c)_k n_i dA
};

// area and centroid of sorted leaf i; a face of zero fp32 area (as the query skips it) or with a corner that is not finite has none
__device__ __forceinline__ void leaf_shape(const Ws& W, long long i, double& area, double3& cen, double3 e[3], double3& n) {
    float3 p0, p1, p2;
    leaf_corners(W, i, p0, p1, p2);
    const bool ok = !zero_area(p0, p1, p2) && isfinite(p0.x + p0.y + p0.z + p1.x + p1.y + p1.z + p2.x + p2.y + p2.z);
    e[0] = to_d(p0); e[1] = to_d(p1); e[2] = to_d(p2);
    const double3 u = make_double3(e[1].x - e[0].x, e[1].y - e[0].y, e[1].z - e[0].z);
    const double3 v = make_double3(e[2].x - e[0].x, e[2].y - e[0].y, e[2].z - e[0].z);
    n = ok ? make_double3(0.5 * (u.y * v.z - u.z * v.y), 0.5 * (u.z * v.x - u.x * v.z), 0.5 * (u.x * v.y - u.y * v.x)) : make_double3(0, 0, 0);
    area = sqrt(n.x * n.x + n.y * n.y + n.z * n.z);
    cen = ok ? make_double3((e[0].x + e[1].x + e[2].x) / 3.0, (e[0].y + e[1].y + e[2].y) / 3.0, (e[0].z + e[1].z + e[2].z) / 3.0)
             : make_double3(0, 0, 0);
}

// a leaf about c, exactly: with e_m = p_m - c and s = e_0 + e_1 + e_2, int (x - c) dA = A s / 3 and
// int (x - c)(x - c)^T dA = A / 12 (sum_m e_m e_m^T + s s^T); n A = N, the half cross product
__device__ void add_leaf(const Ws& W, long long i, double3 c, Moments& M) {
    double area;
    double3 cen, e[3], n;
    leaf_shape(W, i, area, cen, e, n);
    if (area == 0.0) return;
    double d[3][3], s[3];
    #pragma unroll
    for (int m = 0; m < 3; m++) {
        d[m][0] = e[m].x - c.x;
        d[m][1] = e[m].y - c.y;
        d[m][2] = e[m].z - c.z;
    }
    #pragma unroll
    for (int k = 0; k < 3; k++) s[k] = (d[0][k] + d[1][k]) + d[2][k];
    const double N[3] = {n.x, n.y, n.z};
    #pragma unroll
    for (int i = 0; i < 3; i++) {
        M.m0[i] += N[i];
        #pragma unroll
        for (int j = 0; j < 3; j++) M.m1[3 * j + i] += s[j] / 3.0 * N[i];
    }
    #pragma unroll
    for (int j = 0; j < 3; j++)
        #pragma unroll
        for (int k = j; k < 3; k++) {
            const double q = ((d[0][j] * d[0][k] + d[1][j] * d[1][k]) + d[2][j] * d[2][k]) + s[j] * s[k];
            #pragma unroll
            for (int i = 0; i < 3; i++) M.m2[3 * pair_of(j, k) + i] += q / 24.0 * N[i];
        }
}

// an internal node's stored moments about its centroid c0, shifted to c by delta = c0 - c:
// m1_ji += delta_j m0_i; m2_jki += 1/2 (delta_j m1_ki + delta_k m1_ji) + 1/2 delta_j delta_k m0_i
__device__ void add_node(const float4* __restrict__ q, double3 c, Moments& M) {
    const float4 h = __ldcg(q), a = __ldcg(q + 1);
    const double dl[3] = {(double)h.x - c.x, (double)h.y - c.y, (double)h.z - c.z};
    float x[28];
    #pragma unroll
    for (int k = 0; k < 7; k++) {
        const float4 v = __ldcg(q + 2 + k);
        x[4 * k] = v.x; x[4 * k + 1] = v.y; x[4 * k + 2] = v.z; x[4 * k + 3] = v.w;
    }
    const double m0[3] = {a.x, a.y, a.z};
    #pragma unroll
    for (int i = 0; i < 3; i++) {
        M.m0[i] += m0[i];
        #pragma unroll
        for (int j = 0; j < 3; j++) M.m1[3 * j + i] += (double)x[3 * j + i] + dl[j] * m0[i];
    }
    #pragma unroll
    for (int j = 0; j < 3; j++)
        #pragma unroll
        for (int k = j; k < 3; k++)
            #pragma unroll
            for (int i = 0; i < 3; i++) {
                const int pk = 3 * pair_of(j, k) + i;
                M.m2[pk] += (double)x[9 + pk] + 0.5 * (dl[j] * (double)x[3 * k + i] + dl[k] * (double)x[3 * j + i]) + 0.5 * dl[j] * dl[k] * m0[i];
            }
}

// area and centroid of child ch (a leaf when ch >= nl)
__device__ __forceinline__ void child_shape(const Ws& W, const WnWs& M, int ch, int nl, double& area, double3& cen) {
    if (ch >= nl) {
        double3 e[3], n;
        leaf_shape(W, ch - nl, area, cen, e, n);
    } else {
        const float4 h = __ldcg(M.mom + (long long)kSlots * ch), a = __ldcg(M.mom + (long long)kSlots * ch + 1);
        area = a.w;
        cen = make_double3(h.x, h.y, h.z);
    }
}

// nothing is published before an arrival: the second child combines both children's records and writes its node's
__global__ void __launch_bounds__(kThreads) k_wn_build(int F, Ws W, WnWs M) {
    const long long i = thread_index();
    if (i >= F) return;
    const int nl = F - 1;
    climb(W, F, i, M.flags, [](int, int) {}, [&](int p) {
        const NodeView nd = load_node(W, p);
        double a0, a1;
        double3 c0, c1;
        child_shape(W, M, nd.child[0], nl, a0, c0);
        child_shape(W, M, nd.child[1], nl, a1, c1);
        const Box &b0 = nd.box[0], &b1 = nd.box[1];
        const double lo[3] = {fminf(b0.lo.x, b1.lo.x), fminf(b0.lo.y, b1.lo.y), fminf(b0.lo.z, b1.lo.z)};
        const double hi[3] = {fmaxf(b0.hi.x, b1.hi.x), fmaxf(b0.hi.y, b1.hi.y), fmaxf(b0.hi.z, b1.hi.z)};
        const double area = a0 + a1;
        double cd[3];
        #pragma unroll
        for (int k = 0; k < 3; k++)
            cd[k] = area > 0.0 ? (a0 * comp(c0, k) + a1 * comp(c1, k)) / area : 0.5 * (lo[k] + hi[k]);
        const float3 cf = make_float3((float)cd[0], (float)cd[1], (float)cd[2]);
        const double3 c = to_d(cf);                           // the moments are taken about the stored centroid
        double r2 = 0.0;
        #pragma unroll
        for (int k = 0; k < 3; k++) {
            const double e = fmax(fabs(comp(c, k) - lo[k]), fabs(hi[k] - comp(c, k)));
            r2 += e * e;
        }
        Moments m{};
        for (int s = 0; s < 2; s++) {
            const int ch = nd.child[s];
            if (ch >= nl) add_leaf(W, ch - nl, c, m);
            else add_node(M.mom + (long long)kSlots * ch, c, m);
        }
        float4* q = M.mom + (long long)kSlots * p;
        q[0] = make_float4(cf.x, cf.y, cf.z, __double2float_ru(sqrt(r2)));
        q[1] = make_float4((float)m.m0[0], (float)m.m0[1], (float)m.m0[2], (float)area);
        float x[28];
        #pragma unroll
        for (int k = 0; k < 9; k++) x[k] = (float)m.m1[k];
        for (int k = 0; k < 18; k++) x[9 + k] = (float)m.m2[k];
        x[27] = 0.0f;
        #pragma unroll
        for (int k = 0; k < 7; k++) q[2 + k] = make_float4(x[4 * k], x[4 * k + 1], x[4 * k + 2], x[4 * k + 3]);
    });
}

// ---------------------------------------------------------------- query
// the signed solid angle of sorted leaf i seen from p (Van Oosterom and Strackee 1983), fp32 rounded as written; 0 for a face of zero
// fp32 area and wherever det == 0 (p in the face's plane, on a corner) or is NaN
__device__ __forceinline__ float solid_angle(const Ws& W, long long i, float3 p) {
    float3 p0, p1, p2;
    leaf_corners(W, i, p0, p1, p2);
    if (zero_area(p0, p1, p2)) return 0.0f;
    const float3 a = sub3(p0, p), b = sub3(p1, p), c = sub3(p2, p);
    const float det = dot3(a, cross3(b, c));
    if (det == 0.0f || det != det) return 0.0f;
    const float la = sqrtf(dot3(a, a)), lb = sqrtf(dot3(b, b)), lc = sqrtf(dot3(c, c));
    const float den = (((la * lb) * lc + dot3(a, b) * lc) + dot3(b, c) * la) + dot3(c, a) * lb;
    return 2.0f * atan2f(det, den);
}

// 4 pi times the order-2 expansion of the node at q about its centroid c: with r = c - p, s = |r|,
// m0 . r / s^3 + tr(m1) / s^3 - 3 r^T m1 r / s^5 - 3 (2 sum_ji m2_jii r_j + sum_ji m2_jji r_i) / s^5 + 15 sum m2_jki r_j r_k r_i / s^7
__device__ __forceinline__ double far_field(const float4* __restrict__ q, float4 h, float3 p) {
    const double r[3] = {(double)h.x - p.x, (double)h.y - p.y, (double)h.z - p.z};
    const float4 a = __ldg(q + 1);
    float x[28];
    #pragma unroll
    for (int k = 0; k < 7; k++) {
        const float4 v = __ldg(q + 2 + k);
        x[4 * k] = v.x; x[4 * k + 1] = v.y; x[4 * k + 2] = v.z; x[4 * k + 3] = v.w;
    }
    const double s2 = (r[0] * r[0] + r[1] * r[1]) + r[2] * r[2];
    const double is2 = 1.0 / s2, is3 = is2 / sqrt(s2), is5 = is3 * is2, is7 = is5 * is2;
    const double t0 = ((double)a.x * r[0] + (double)a.y * r[1]) + (double)a.z * r[2];
    double tr = 0.0, rmr = 0.0, a1 = 0.0, a2 = 0.0, c3 = 0.0;
    #pragma unroll
    for (int j = 0; j < 3; j++) {
        tr += x[4 * j];
        #pragma unroll
        for (int i = 0; i < 3; i++) {
            rmr += r[j] * (double)x[3 * j + i] * r[i];
            a1 += (double)x[9 + 3 * pair_of(j, i) + i] * r[j];
            a2 += (double)x[9 + 3 * pair_of(j, j) + i] * r[i];
            #pragma unroll
            for (int k = 0; k < 3; k++) c3 += (double)x[9 + 3 * pair_of(j, k) + i] * r[j] * r[k] * r[i];
        }
    }
    return (t0 + tr) * is3 - 3.0 * rmr * is5 - 3.0 * (2.0 * a1 + a2) * is5 + 15.0 * c3 * is7;
}

__global__ void __launch_bounds__(kThreads) k_wn_query(int F, long long P, const float* __restrict__ points, Ws W, WnWs M, float beta,
                                                       float* __restrict__ w_out) {
    const long long t = thread_index();
    if (t >= P) return;
    const float3 p = load3(points, t);
    double sum = 0.0;
    if (F > 0) {
        const int nl = F - 1;                                 // ids at or above nl are leaves; id 0 is the root (leaf 0 when F = 1)
        int stack[kStack];
        int sp = 0;
        stack[sp++] = 0;
        while (sp > 0) {
            const int node = stack[--sp];
            if (node >= nl) {
                sum += (double)solid_angle(W, node - nl, p);
                continue;
            }
            const float4* q = M.mom + (long long)kSlots * node;
            const float4 h = __ldg(q);
            const float3 d = sub3(p, make_float3(h.x, h.y, h.z));
            const float br = beta * h.w;
            if (dot3(d, d) > br * br) {                       // false for beta = +inf (inf, or NaN when r = 0)
                sum += far_field(q, h, p);
                continue;
            }
            const int4 ch = __ldg(&W.nodes[node].d);
            stack[sp++] = ch.y;                               // child 0 is popped first
            stack[sp++] = ch.x;
        }
    }
    w_out[t] = (float)(sum / kFourPi);
}
}  // namespace

extern "C" {

long long psdf_mesh_winding_workspace_bytes(long long nr_vertices, long long nr_faces) {
    if (nr_vertices < 0 || nr_faces < 0) return PSDF_ERR_ARG;
    if (nr_vertices > kIntMax || nr_faces > kIntMax) return PSDF_ERR_UNSUPPORTED;
    return carve_wn(nullptr, nr_faces, nullptr);
}

int psdf_mesh_winding_build(int V, int F, const float* verts, const int* faces, const uint8_t* bvh_workspace, uint8_t* workspace,
                            void* stream) {
    if (V < 0 || F < 0 || !bvh_workspace || (F > 1 && !workspace)) return PSDF_ERR_ARG;
    (void)verts;
    (void)faces;
    if (F < 2) return PSDF_OK;                                // no internal node
    Ws W;
    carve(const_cast<uint8_t*>(bvh_workspace), V, F, &W);
    WnWs M;
    carve_wn(workspace, F, &M);
    cudaMemsetAsync(M.flags, 0, 4 * (size_t)(F - 1), ST);
    k_wn_build<<<blocks(F), kThreads, 0, ST>>>(F, W, M);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

int psdf_mesh_winding_number(int V, int F, long long P, const float* points, const uint8_t* bvh_workspace, const uint8_t* workspace,
                             float beta, float* w_out, void* stream) {
    if (V < 0 || F < 0 || P < 0 || !bvh_workspace || (F > 1 && !workspace) || (P > 0 && (!points || !w_out)) || !(beta > 0.0f))
        return PSDF_ERR_ARG;
    if (P > (long long)kThreads * kIntMax) return PSDF_ERR_UNSUPPORTED;
    if (P == 0) return PSDF_OK;
    Ws W;
    carve(const_cast<uint8_t*>(bvh_workspace), V, F, &W);
    WnWs M;
    carve_wn(const_cast<uint8_t*>(workspace), F, &M);
    k_wn_query<<<blocks(P), kThreads, 0, ST>>>(F, P, points, W, M, beta, w_out);
    PSDF_CHECK_LAUNCH();
    return PSDF_OK;
}

}  // extern "C"
