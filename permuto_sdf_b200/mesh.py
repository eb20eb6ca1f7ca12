"""Meshes from a volume, a trained SDF or a trained NeRF density on the GPU (extract_mesh_from_sdf_model and
extract_mesh_from_density_model, permuto_sdf_py/utils/sdf_utils.py:252-292 and :339-380).

The reference evaluates the SDF in 64^3 chunks into a dense host array of N^3 floats and runs skimage's marching cubes on the CPU. Here
the grid is evaluated a slab of slices at a time by a fused forward kernel (FusedSDF, or the density-only FusedNerfHash.density), and
each slab goes straight to the marching-cubes kernels (csrc/marching_cubes.cu), which carry the vertex numbering from slab to slab.
The N^3 volume never exists; memory is O(N^2 * slab) plus the mesh. The output is a fixed function of the volume (see the header), the same for any slab split and on every run.
Mesh.connected_components, remove_small_components and keep_largest_component clean an extracted mesh of floaters and bubbles on the GPU
(csrc/mesh_components.cu): labels, counts and the kept vertices are a fixed function of the mesh as well.
Mesh.decimate reduces a mesh to a target face count by quadric edge collapse, in parallel rounds of independent collapses on the GPU
(csrc/mesh_decimate.cu), and Mesh.recalculate_normals sets NV from the faces; both give the same bits on every run.
Mesh.load reads PLY, OBJ and STL files on the host, the torch ops below weld, compact and place a mesh as train_sdf_from_mesh.py does,
and Mesh.upsample runs midpoint or Loop subdivision on the GPU (csrc/mesh_subdivide.cu), the same bits on every run.
Mesh.occluded and Mesh.ambient_occlusion cast rays against the faces through a linear BVH on the GPU (csrc/mesh_raycast.cu), and
load_mesh_sequence assembles the point sequence of train_4d_sdf.py from a folder of meshes. Mesh.closest_points and
Mesh.signed_distance query the nearest point of the faces through the same BVH (csrc/mesh_distance.cu), and mesh_distance measures how
far apart two meshes are from surface samples of each. Mesh.first_hit finds the first face each ray meets through that BVH, and
Mesh.render shades the first hits of the rays of reel cameras (cameras.py), so a mesh becomes a training scene with a known answer.
Mesh.winding_number sums the faces' solid angles through the same BVH with a hierarchical far field (csrc/mesh_winding.cu), which gives
an inside/outside for any triangle soup: Mesh.signed_distance(points, sign="winding").
"""
import math
import os
import re

import numpy as np
import torch
import torch.nn.functional as F

from ._lib import call, load_library

# grid points per slab: the slab's evaluation, values and edge ids (about 30 B per point in all)
_SLAB_POINTS = 1 << 24
_INT_MAX = 2 ** 31 - 1
# workspace of psdf_mesh_components: int64 info[4] in the first 256 bytes, then int32 labels [V], then int32 face counts [V]
_CC_HEADER = 256
# the images Mesh.render can produce, in the order of psdf_mesh_render's outputs
RENDER_OUTPUTS = ("rgb", "mask", "depth", "normal", "face")


def _check_f(fn, Fc):
    if not isinstance(Fc, torch.Tensor) or Fc.dtype != torch.int32:
        raise RuntimeError("%s: F must be an int32 tensor of shape [F,3], got %s" % (fn, getattr(Fc, "dtype", type(Fc).__name__)))
    if Fc.dim() != 2 or Fc.shape[1] != 3:
        raise RuntimeError("%s: F must have shape [F,3], got %s" % (fn, list(Fc.shape)))


def _check_sizes(fn, nv, nf):
    if nv > _INT_MAX or nf > _INT_MAX:
        raise RuntimeError("%s: %d vertices and %d faces; both must be below 2^31" % (fn, nv, nf))


def _checked_call(fn, workspace_bytes, entry, nv, nf, args, out=(), repeats_allowed=False):
    """entry(nv, nf, *args, workspace, *out) on a new workspace of workspace_bytes(nv, nf) bytes on the device of args[-1]; raises on the
    faces with an index outside [0, nv) that it counted into info[0], and unless repeats_allowed on those with a repeated vertex that it
    counted into info[1] -> (workspace, info[2])"""
    ws = torch.empty(int(workspace_bytes(nv, nf)), dtype=torch.uint8, device=args[-1].device)
    call(entry, nv, nf, *args, ws, *out)
    bad, rep, info2 = ws[:24].view(torch.int64).tolist()
    if bad:
        raise RuntimeError("%s: %d faces have a vertex index outside [0, %d)" % (fn, bad, nv))
    if rep and not repeats_allowed:
        raise RuntimeError("%s: %d faces repeat a vertex" % (fn, rep))
    return ws, info2


def _slab_slices(N0, N1, N2):
    return max(1, min(N0 - 1, _SLAB_POINTS // (N1 * N2)))


class _SlabMarchingCubes:
    """the slab sequence of one volume: workspace, running vertex count and the pieces of the output"""

    def __init__(self, N0, S, N1, N2, threshold, device, affine=(1.0, 1.0, 0.0)):
        nbytes = int(load_library().psdf_marching_cubes_workspace_bytes(S, N1, N2))
        if nbytes < 0:
            raise RuntimeError("marching_cubes: a slab of %d slices of %d x %d points is more than the kernels index in 32 bits" % (S, N1, N2))
        self.N0, self.N1, self.N2, self.thr, self.affine = N0, N1, N2, float(threshold), affine
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.counts = torch.zeros(3, dtype=torch.int64, device=device)
        self.vbase = 0
        self.verts, self.faces = [], []

    def run(self, vol, i0):
        """vol [S + 1, N1, N2]: slices i0 .. i0 + S; `last` when they end the volume"""
        S = vol.shape[0] - 1
        last = int(i0 + S == self.N0 - 1)
        args = (S, self.N1, self.N2, i0, last, self.thr, vol)
        call("psdf_marching_cubes_count", *args, self.ws, self.counts)
        nv, nf, nx = self.counts.tolist()
        if self.vbase + nx > _INT_MAX:
            raise RuntimeError("marching_cubes: more than 2^31 - 1 vertices, which int32 faces cannot index")
        dev = vol.device
        verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(nf, 3, dtype=torch.int32, device=dev)
        call("psdf_marching_cubes_emit", *args, self.vbase, self.affine, self.ws, verts, faces)
        self.vbase += nv
        self.verts.append(verts)
        self.faces.append(faces)

    def result(self):
        return torch.cat(self.verts), torch.cat(self.faces)


def _check_volume(volume, threshold):
    if not isinstance(volume, torch.Tensor) or volume.dtype != torch.float32 or not volume.is_cuda:
        raise RuntimeError("marching_cubes: volume must be a float32 CUDA tensor")
    if volume.dim() != 3 or min(volume.shape) < 2:
        raise RuntimeError("marching_cubes: volume must have shape [N0, N1, N2] with every dimension >= 2, got %s" % list(volume.shape))
    if not math.isfinite(float(threshold)):
        raise RuntimeError("marching_cubes: threshold must be finite, got %r" % threshold)


def _marching_cubes(volume, threshold, slab):
    _check_volume(volume, threshold)
    vol = volume.contiguous()
    N0, N1, N2 = vol.shape
    S = min(slab, N0 - 1) if slab else _slab_slices(N0, N1, N2)
    with torch.cuda.device(vol.device):
        mc = _SlabMarchingCubes(N0, S, N1, N2, threshold, vol.device)
        for i0 in range(0, N0 - 1, S):
            mc.run(vol[i0:min(i0 + S, N0 - 1) + 1], i0)
        return mc.result()


def marching_cubes(volume, threshold=0.0):
    """skimage.measure.marching_cubes(volume, threshold) for a dense float32 CUDA volume [N0, N1, N2] (each >= 2), axis 0 = x.
    -> (verts float32 [V,3] in index space, faces int32 [F,3]). A corner is inside when value < threshold; faces wind counter-clockwise
    seen from outside (the right-hand normal points from inside to outside). Vertices come slice by slice along axis 0 and faces cell by
    cell, in an order that depends only on the volume."""
    return _marching_cubes(volume, threshold, None)


class Mesh:
    """the fields of EasyPBR's Mesh that the reference's programs read from an extracted mesh: V [V,3], F [F,3] int32, NV [V,3] (device
    tensors)"""

    def __init__(self, V, F, NV=None):
        self.V, self.F, self.NV = V, F, NV

    def remove_marked_vertices(self, mask, keep):
        """keep=True keeps the marked vertices (create_my_meshes.py:74 with check_point_inside_primitive), keep=False removes them. Faces
        that touch a removed vertex go; the remaining vertices keep their order and are renumbered. mask: bool [V] or [V,1], a tensor or a
        numpy array. -> self"""
        m = torch.as_tensor(mask).to(device=self.V.device).reshape(-1).bool()
        if m.shape[0] != self.V.shape[0]:
            raise RuntimeError("Mesh.remove_marked_vertices: mask has %d entries for %d vertices" % (m.shape[0], self.V.shape[0]))
        kept = m if keep else ~m
        new_id = torch.cumsum(kept.to(torch.int64), 0) - 1
        F_ = self.F.long()
        face_kept = kept[F_].all(1)
        self.F = new_id[F_[face_kept]].to(torch.int32).reshape(-1, 3)
        self.V = self.V[kept]
        if self.NV is not None:
            self.NV = self.NV[kept]
        return self

    def _components(self, fn):
        """psdf_mesh_components of F -> (workspace, number of components); raises on faces that index outside [0, V)"""
        Fc, V = self.F, self.V
        _check_f(fn, Fc)
        if not Fc.is_cuda:
            raise RuntimeError("%s: F must be a CUDA tensor (there is no CPU path)" % fn)
        if not isinstance(V, torch.Tensor) or V.device != Fc.device:
            raise RuntimeError("%s: V must be a tensor on F's device %s" % (fn, Fc.device))
        nv, nf = V.shape[0], Fc.shape[0]
        _check_sizes(fn, nv, nf)
        with torch.cuda.device(Fc.device):
            ws = torch.empty(int(load_library().psdf_mesh_components_workspace_bytes(nv, nf)), dtype=torch.uint8, device=Fc.device)
            call("psdf_mesh_components", nv, nf, Fc.contiguous(), ws)
            nr, bad = ws[:16].view(torch.int64).tolist()
        if bad:
            raise RuntimeError("%s: %d faces have a vertex index outside [0, %d)" % (fn, bad, nv))
        return ws, nr

    def connected_components(self, with_face_counts=False):
        """connected components of the vertex graph (each face joins its three vertices) on the GPU -> (labels int32 [V], number of
        components). The label of a vertex is the smallest vertex index of its component, so the labels are the same bits for any face
        order and on every run; a vertex no face references is a component of its own. with_face_counts: also the faces of each
        component, int32 [V] indexed by label (0 at non-root vertices), a face counting for the component of its first vertex. F must be
        an int32 CUDA tensor [F,3] with indices in [0, V) (checked on the device), V and F below 2^31; there is no CPU path."""
        ws, nr = self._components("Mesh.connected_components")
        nv = self.V.shape[0]
        labels = ws[_CC_HEADER:_CC_HEADER + 4 * nv].view(torch.int32)
        if with_face_counts:
            return labels, nr, ws[_CC_HEADER + 4 * nv:_CC_HEADER + 8 * nv].view(torch.int32)
        return labels, nr

    def _keep_components(self, fn, largest, min_faces):
        ws, _ = self._components(fn)
        keep = torch.empty(self.V.shape[0], dtype=torch.bool, device=self.F.device)
        with torch.cuda.device(self.F.device):
            call("psdf_mesh_components_keep", self.V.shape[0], int(largest), min_faces, ws, keep)
        return self.remove_marked_vertices(keep, True)

    def remove_small_components(self, min_faces):
        """keeps the vertices of the components (connected_components) with at least min_faces faces and compacts the mesh as
        remove_marked_vertices(mask, keep=True) does: faces that touch a removed vertex go, V, NV and the vertex ids of F keep their
        order. min_faces = 0 keeps everything; 1 drops vertices no face uses. -> self"""
        if isinstance(min_faces, bool) or not isinstance(min_faces, (int, np.integer)) or min_faces < 0:
            raise RuntimeError("Mesh.remove_small_components: min_faces must be a non-negative integer, got %r" % (min_faces,))
        return self._keep_components("Mesh.remove_small_components", False, int(min_faces))

    def keep_largest_component(self):
        """keeps only the component with the most faces, ties broken by the smallest label, and compacts the mesh as
        remove_small_components does. A mesh without faces keeps its vertex 0 (a component of 0 faces with the smallest label); an empty
        mesh stays empty. -> self"""
        return self._keep_components("Mesh.keep_largest_component", True, 0)

    def _check_vf(self, fn):
        """V float32 CUDA [V,3] with finite values, F int32 [F,3] on V's device, both below 2^31 -> (V, F) contiguous"""
        V, Fc = self.V, self.F
        if not isinstance(V, torch.Tensor) or V.dtype != torch.float32:
            raise RuntimeError("%s: V must be a float32 tensor of shape [V,3], got %s" % (fn, getattr(V, "dtype", type(V).__name__)))
        if V.dim() != 2 or V.shape[1] != 3:
            raise RuntimeError("%s: V must have shape [V,3], got %s" % (fn, list(V.shape)))
        _check_f(fn, Fc)
        if not V.is_cuda:
            raise RuntimeError("%s: V must be a CUDA tensor (there is no CPU path)" % fn)
        if Fc.device != V.device:
            raise RuntimeError("%s: F must be on V's device %s, got %s" % (fn, V.device, Fc.device))
        _check_sizes(fn, V.shape[0], Fc.shape[0])
        if not bool(torch.isfinite(V).all()):
            raise RuntimeError("%s: V has values that are not finite" % fn)
        return V.contiguous(), Fc.contiguous()

    def _decimate(self, nr_target_faces):
        """the rounds of decimate before the final compaction -> (V, F, removed [V] bool, rounds); None when the target is at or above
        the face count"""
        fn = "Mesh.decimate"
        if isinstance(nr_target_faces, bool) or not isinstance(nr_target_faces, (int, np.integer)) or nr_target_faces < 0:
            raise RuntimeError("%s: nr_target_faces must be a non-negative integer, got %r" % (fn, nr_target_faces))
        target = int(nr_target_faces)
        V, Fc = self._check_vf(fn)
        nv, nf = V.shape[0], Fc.shape[0]
        if target >= nf:
            return None
        dev = V.device
        with torch.cuda.device(dev):
            V, Fc = V.clone(), Fc.clone()
            removed = torch.empty(nv, dtype=torch.bool, device=dev)
            ws, _ = _checked_call(fn, load_library().psdf_mesh_decimate_workspace_bytes, "psdf_mesh_decimate_begin", nv, nf, (V, Fc),
                                  (removed,))
            cur, rounds = nf, 0
            while True:
                allowed = (cur - target + 1) // 2
                if allowed <= 0:
                    break
                call("psdf_mesh_decimate_round", nv, nf, cur, allowed, V, Fc, ws, removed)
                applied = int(ws[24:32].view(torch.int64).item())
                rounds += 1
                if applied == 0:
                    break
                cur -= 2 * applied
        return V, Fc[:cur], removed, rounds

    def decimate(self, nr_target_faces):
        """quadric edge-collapse decimation on the GPU (Garland-Heckbert, in parallel rounds of collapses that share no vertex or
        neighbour; the rules are in include/psdf_b200.h). Interior edges collapse in order of quadric error until the mesh has
        nr_target_faces or nr_target_faces - 1 faces (each collapse removes two), or fewer when no edge passes the checks (link
        condition, no face flips or degenerates, no opposite vertex in 3 faces or fewer, no end in more than 64 faces); 0 decimates as far as
        they allow. Boundary,
        non-manifold and inconsistently oriented edges lock their vertices, which never move, so such edges stay exactly as they are.
        Removed vertices go and the rest keep their order, as remove_marked_vertices does; vertices no face uses stay. NV, when present,
        is recalculated (recalculate_normals). The same bits on every run. A target at or above the face count returns the mesh as it
        is. V must be float32 CUDA [V,3] with finite values and F int32 [F,3] on its device, both below 2^31; faces with an index outside
        [0, V) or a repeated vertex are refused (checked on the device). There is no CPU path. -> self"""
        out = self._decimate(nr_target_faces)
        if out is None:
            return self
        self.V, self.F, removed, _ = out
        self.remove_marked_vertices(removed, False)
        if self.NV is not None:
            self.recalculate_normals()
        return self

    def recalculate_normals(self):
        """NV = the normalised sum of the cross products (p1 - p0) x (p2 - p0) of each vertex's faces, summed in fp32 in ascending face
        order; zero for a vertex without faces. On the GPU, with the checks of decimate: faces with an index outside [0, V) or a
        repeated vertex are refused. -> self"""
        fn = "Mesh.recalculate_normals"
        V, Fc = self._check_vf(fn)
        nv, nf = V.shape[0], Fc.shape[0]
        with torch.cuda.device(V.device):
            NV = torch.empty_like(V)
            _checked_call(fn, load_library().psdf_mesh_normals_workspace_bytes, "psdf_mesh_normals", nv, nf, (V, Fc), (NV,))
        self.NV = NV
        return self

    def upsample(self, nr_subdivisions, smooth):
        """nr_subdivisions rounds of subdivision on the GPU, each splitting every face into four: smooth=False is midpoint subdivision
        (libigl's upsample), smooth=True Loop subdivision (libigl's loop). New vertices follow the old ones; the rules, the numbering and
        the fp32 arithmetic are in include/psdf_b200.h, and the result is the same bits on every run. Boundary and non-manifold edges are
        creases: their vertices are midpoints and their ends follow the boundary rule or stay. NV, when present, is recalculated
        (recalculate_normals). The checks of decimate apply; a result with 2^31 or more faces (4^rounds F) is refused before anything
        runs, and one with 2^31 or more vertices before its round. -> self"""
        fn = "Mesh.upsample"
        if isinstance(nr_subdivisions, bool) or not isinstance(nr_subdivisions, (int, np.integer)) or nr_subdivisions < 0:
            raise RuntimeError("%s: nr_subdivisions must be a non-negative integer, got %r" % (fn, nr_subdivisions))
        rounds = int(nr_subdivisions)
        if isinstance(self.F, torch.Tensor) and self.F.dim() == 2 and self.F.shape[0] * 4 ** rounds > _INT_MAX:
            raise RuntimeError("%s: %d faces become %d after %d rounds; int32 faces hold fewer than 2^31" % (
                fn, self.F.shape[0], self.F.shape[0] * 4 ** rounds, rounds))
        V, Fc = self._check_vf(fn)
        if rounds == 0:
            return self
        with torch.cuda.device(V.device):
            for _ in range(rounds):
                nv, nf = V.shape[0], Fc.shape[0]
                ws, E = _checked_call(fn, load_library().psdf_mesh_subdivide_workspace_bytes, "psdf_mesh_subdivide_count", nv, nf, (Fc,))
                if nv + E > _INT_MAX:
                    raise RuntimeError("%s: %d vertices and %d edges make %d vertices; V must stay below 2^31" % (fn, nv, E, nv + E))
                Vn = torch.empty(nv + E, 3, dtype=torch.float32, device=V.device)
                Fn = torch.empty(4 * nf, 3, dtype=torch.int32, device=V.device)
                call("psdf_mesh_subdivide_emit", nv, nf, int(bool(smooth)), V, Fc, ws, Vn, Fn)
                V, Fc = Vn, Fn
                del ws
        self.V, self.F = V, Fc
        if self.NV is not None:
            self.recalculate_normals()
        return self

    # ------------------------------------------------------------------ ray casting
    def _bvh(self, fn):
        """the BVH of the faces (psdf_mesh_bvh_build) -> (V, F, workspace); raises on faces with an index outside [0, V)"""
        V, Fc = self._check_vf(fn)
        ws, _ = _checked_call(fn, load_library().psdf_mesh_bvh_workspace_bytes, "psdf_mesh_bvh_build", V.shape[0], Fc.shape[0], (V, Fc),
                              repeats_allowed=True)
        return V, Fc, ws

    def occluded(self, origins, dirs, tnear=1e-4, tfar=math.inf):
        """any-hit ray casting on the GPU: bool [R], True where ray r (origins [R,3], dirs [R,3], float32 CUDA tensors on V's device with
        finite values; dirs need not be unit) passes the two-sided fp32 ray-triangle test of include/psdf_b200.h against some face at a
        parameter t with tnear < t < tfar (both rounded to fp32). The answer is that of testing every face; a BVH built on each call only
        chooses which faces are tested. Faces that repeat a vertex are never hit. V and F are checked as decimate checks them, except that
        faces repeating a vertex are allowed."""
        fn = "Mesh.occluded"
        o, d = _check_rays(fn, origins, dirs, self.V)
        _check_window(fn, tnear, tfar)
        with torch.cuda.device(o.device):
            V, Fc, ws = self._bvh(fn)
            hit = torch.empty(o.shape[0], dtype=torch.uint8, device=o.device)
            call("psdf_mesh_occluded", V.shape[0], Fc.shape[0], o.shape[0], o, d, float(tnear), float(tfar), ws, hit)
        return hit.bool()

    def ambient_occlusion(self, nr_samples=100):
        """the visible fraction of every vertex, float32 [V]: of the nr_samples rays from V[i] along the fixed Fibonacci directions
        (fibonacci_directions: the same for every vertex), each negated when it points against NV[i] (fp32 dot < 0), the share that
        hits no face at 1e-4 < t < inf, float(S - hits) / float(S). The same bits on every run. NV is required (recalculate_normals).
        This is what the reference reads as compute_embree_ao(n) then C[:, 0]. EasyPBR's compute_embree_ao is not in the reference's
        checkout; as far as we recall it wraps libigl's embree ambient_occlusion with random directions and stores 1 - the hit fraction,
        so the directions here are ours and the values agree with it only up to its sampling noise."""
        fn = "Mesh.ambient_occlusion"
        if isinstance(nr_samples, bool) or not isinstance(nr_samples, (int, np.integer)) or not 1 <= nr_samples <= _INT_MAX:
            raise RuntimeError("%s: nr_samples must be a positive integer, got %r" % (fn, nr_samples))
        if self.NV is None:
            raise RuntimeError("%s: the mesh has no vertex normals (NV); call mesh.recalculate_normals() first" % fn)
        S = int(nr_samples)
        NV = self.NV
        if not isinstance(NV, torch.Tensor) or NV.dtype != torch.float32 or not isinstance(self.V, torch.Tensor) or \
                NV.shape != self.V.shape or NV.device != self.V.device:
            raise RuntimeError("%s: NV must be a float32 tensor shaped and placed like V" % fn)
        with torch.cuda.device(self.V.device):
            V, Fc, ws = self._bvh(fn)
            dirs = torch.from_numpy(fibonacci_directions(S)).to(V.device)
            vis = torch.empty(V.shape[0], dtype=torch.float32, device=V.device)
            call("psdf_mesh_ambient_occlusion", V.shape[0], Fc.shape[0], S, V, NV.contiguous(), dirs, ws, vis)
        return vis

    def first_hit(self, origins, dirs, tnear=0.0, tfar=math.inf):
        """first-hit ray casting on the GPU -> (t float32 [R], face int32 [R], bary float32 [R,3]): of the faces that pass occluded's
        ray-triangle test for ray r with tnear < t < tfar, the one with the smallest fp32 t, ties to the smallest face index; bary =
        ((1 - u) - v, u, v) of the test's u and v, so the hit point is (b0 a + b1 b) + b2 c. A miss is (+inf, -1, 0). The answer is that
        of testing every face (a BVH built on each call only prunes) and the same bits on every run. Rays, V and F are checked as occluded
        checks them."""
        fn = "Mesh.first_hit"
        o, d = _check_rays(fn, origins, dirs, self.V)
        _check_window(fn, tnear, tfar)
        with torch.cuda.device(o.device):
            V, Fc, ws = self._bvh(fn)
            R = o.shape[0]
            t = torch.empty(R, dtype=torch.float32, device=o.device)
            face = torch.empty(R, dtype=torch.int32, device=o.device)
            bary = torch.empty(R, 3, dtype=torch.float32, device=o.device)
            call("psdf_mesh_first_hit", V.shape[0], Fc.shape[0], R, o, d, float(tnear), float(tfar), ws, t, face, bary)
        return t, face, bary

    def render(self, K, tf_world_cam, H, W, colors=None, tnear=0.0, tfar=math.inf, outputs=RENDER_OUTPUTS):
        """renders the mesh from I reel cameras on the GPU, one ray per pixel: the ray of pixel (x, y) of image i is the one
        PermutoSDF.rays_from_reel_indices forms for pix = y W + x, img = i, bit for bit (a trainer drawing that pixel casts the ray that
        rendered it), and its first_hit within (tnear, tfar) is shaded:
          normal  (b0 N_a + b1 N_b) + b2 N_c of NV when the mesh has it, else the face's cross(p_b - p_a, p_c - p_a), normalised (0 when its
                  length is 0); in world coordinates and not flipped toward the camera
          rgb     (b0 C_a + b1 C_b) + b2 C_c of colors [V,3] when given, else 0.5 + 0.5 normal (bench.analytic_reel's shading)
          mask 1, depth t, face the face index; a missed pixel is 0 everywhere and face -1 (a reel's rgb is already multiplied by its mask)
        K float32 [I,3,3] and tf_world_cam float32 [I,4,4] (camera to world), finite, on V's device; H, W positive with H W < 2^31.
        -> dict of the names in `outputs` (any of "rgb", "mask", "depth", "normal", "face"): rgb and normal float32 [I,3,H,W], mask and depth
        float32 [I,1,H,W], face int32 [I,1,H,W]; other outputs are not computed. The same bits on every run. V and F are checked as
        occluded checks them."""
        fn = "Mesh.render"
        V = self.V
        if not isinstance(V, torch.Tensor) or not V.is_cuda:
            raise RuntimeError("%s: V must be a CUDA tensor (there is no CPU path)" % fn)
        for name, v in (("H", H), ("W", W)):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
                raise RuntimeError("%s: %s must be a positive integer, got %r" % (fn, name, v))
        H, W = int(H), int(W)
        if H * W > _INT_MAX:
            raise RuntimeError("%s: a %d x %d image has 2^31 or more pixels" % (fn, H, W))
        K = _check_camera(fn, "K", K, (3, 3), V.device)
        tf = _check_camera(fn, "tf_world_cam", tf_world_cam, (4, 4), V.device)
        if K.shape[0] != tf.shape[0]:
            raise RuntimeError("%s: %d K and %d tf_world_cam" % (fn, K.shape[0], tf.shape[0]))
        outputs = tuple(outputs)
        bad = [o for o in outputs if o not in RENDER_OUTPUTS]
        if bad:
            raise RuntimeError("%s: unknown output %r; the outputs are %s" % (fn, bad[0], ", ".join(RENDER_OUTPUTS)))
        _check_window(fn, tnear, tfar)
        NV = _check_vertex_field(fn, "NV", self.NV, V)
        C = _check_vertex_field(fn, "colors", colors, V)
        I = K.shape[0]
        with torch.cuda.device(V.device):
            Vc, Fc, ws = self._bvh(fn)
            shapes = {"rgb": (3, torch.float32), "mask": (1, torch.float32), "depth": (1, torch.float32), "normal": (3, torch.float32),
                      "face": (1, torch.int32)}
            out = {o: torch.empty(I, shapes[o][0], H, W, dtype=shapes[o][1], device=V.device) for o in outputs}
            call("psdf_mesh_render", Vc.shape[0], Fc.shape[0], Vc, Fc, NV, C, I, H, W, K, tf, float(tnear), float(tfar), ws,
                 *[out.get(o) for o in RENDER_OUTPUTS])
        return out

    # ------------------------------------------------------------------ distances
    def _closest(self, fn, p):
        """psdf_mesh_closest_points of the checked points p -> (V, F, BVH workspace, dist2 [P], face [P], bary [P,3])"""
        V, Fc, ws = self._bvh(fn)
        P = p.shape[0]
        dist2 = torch.empty(P, dtype=torch.float32, device=V.device)
        face = torch.empty(P, dtype=torch.int32, device=V.device)
        bary = torch.empty(P, 3, dtype=torch.float32, device=V.device)
        call("psdf_mesh_closest_points", V.shape[0], Fc.shape[0], P, p, V, Fc, ws, dist2, face, bary)
        return V, Fc, ws, dist2, face, bary

    def closest_points(self, points):
        """the nearest point of the faces to each of points [P,3] (float32 CUDA on V's device, finite), on the GPU ->
        (dist float32 [P], face int32 [P], closest float32 [P,3]): dist = sqrt of the fp32 squared distance, face the original face index,
        closest = (b0 a + b1 b) + b2 c of its barycentrics. The answer is that of testing every face with the fp32 closest-point formula
        of include/psdf_b200.h: the smallest squared distance, ties to the smallest face index; a BVH built on each call only prunes.
        Faces that repeat a vertex are skipped; zero-area faces count as their edges. Without such faces: (+inf, -1, NaN). V and F are
        checked as occluded checks them."""
        fn = "Mesh.closest_points"
        p = _check_points(fn, points, self.V)
        with torch.cuda.device(p.device):
            V, Fc, _, dist2, face, bary = self._closest(fn, p)
            corners = V[Fc[face.clamp(min=0).long()].long()] if Fc.shape[0] else torch.full((face.shape[0], 3, 3), math.nan,
                                                                                               device=V.device)
            closest = (bary[:, 0:1] * corners[:, 0] + bary[:, 1:2] * corners[:, 1]) + bary[:, 2:3] * corners[:, 2]
            closest[face < 0] = math.nan
            return torch.sqrt(dist2), face, closest

    def _pseudonormals(self, fn):
        """angle-weighted pseudonormals (Baerentzen and Aanaes 2005) on the GPU -> (face_n float32 [F,3] unit, vert_n float32 [V,3],
        edge_n float32 [F,3,3]): vertex and edge sums in ascending face order, the same bits on every run (include/psdf_b200.h). Not
        normalised except face_n; only their directions are used."""
        V, Fc = self._check_vf(fn)
        nv, nf = V.shape[0], Fc.shape[0]
        with torch.cuda.device(V.device):
            face_n = torch.empty(nf, 3, dtype=torch.float32, device=V.device)
            vert_n = torch.empty(nv, 3, dtype=torch.float32, device=V.device)
            edge_n = torch.empty(nf, 3, 3, dtype=torch.float32, device=V.device)
            _checked_call(fn, load_library().psdf_mesh_pseudonormals_workspace_bytes, "psdf_mesh_pseudonormals", nv, nf, (V, Fc),
                          (face_n, vert_n, edge_n), repeats_allowed=True)
        return face_n, vert_n, edge_n

    def signed_distance(self, points, sign="pseudonormal"):
        """signed distance from the faces to each of points [P,3] (float32 CUDA on V's device, finite), on the GPU -> float32 [P],
        negative inside: sqrt of closest_points' squared distance, with a sign by one of two definitions:
          "pseudonormal" (the default)  the sign of dot(p - q, n), n the angle-weighted pseudonormal of the vertex, edge or face holding the
                  closest point q (include/psdf_b200.h); a zero dot gives +0. Exact and one traversal, but right only for a closed,
                  consistently oriented (outward), edge-manifold mesh, such as marching_cubes gives; topology is not checked.
          "winding"  negative where winding_number(points) > 0.5, else +: defined for any triangle soup (holes, overlaps, unwelded or
                  non-manifold faces), but approximate far from the faces (beta = 2); use it for meshes that are not closed manifolds.
        In both, a zero distance is +0 and a mesh without faces gives +inf."""
        fn = "Mesh.signed_distance"
        if sign not in ("pseudonormal", "winding"):
            raise RuntimeError("%s: unknown sign %r; the signs are 'pseudonormal' and 'winding'" % (fn, sign))
        p = _check_points(fn, points, self.V)
        if sign == "winding":
            with torch.cuda.device(p.device):
                V, Fc, ws, dist2, _, _ = self._closest(fn, p)
                w = self._winding(fn, p, V, Fc, ws, 2.0)
            dist = torch.sqrt(dist2)
            return torch.where((w > 0.5) & (dist > 0), -dist, dist)
        with torch.cuda.device(p.device):
            face_n, vert_n, edge_n = self._pseudonormals(fn)
            V, Fc, ws = self._bvh(fn)
            P = p.shape[0]
            dist2 = torch.empty(P, dtype=torch.float32, device=p.device)
            face = torch.empty(P, dtype=torch.int32, device=p.device)
            bary = torch.empty(P, 3, dtype=torch.float32, device=p.device)
            sdf = torch.empty(P, dtype=torch.float32, device=p.device)
            call("psdf_mesh_signed_distance", V.shape[0], Fc.shape[0], P, p, V, Fc, ws, face_n, vert_n, edge_n, dist2, face, bary, sdf)
        return sdf

    def _winding(self, fn, p, V, Fc, bvh, beta):
        """psdf_mesh_winding_build on the BVH workspace bvh of (V, Fc), then psdf_mesh_winding_number of the checked points p -> float32 [P]"""
        nv, nf = V.shape[0], Fc.shape[0]
        ws = torch.empty(int(load_library().psdf_mesh_winding_workspace_bytes(nv, nf)), dtype=torch.uint8, device=V.device)
        call("psdf_mesh_winding_build", nv, nf, V, Fc, bvh, ws)
        w = torch.empty(p.shape[0], dtype=torch.float32, device=p.device)
        call("psdf_mesh_winding_number", nv, nf, p.shape[0], p, bvh, ws, float(beta), w)
        return w

    def winding_number(self, points, beta=2.0):
        """generalized winding number of each of points [P,3] (float32 CUDA on V's device, finite) against the faces, on the GPU ->
        float32 [P]: (1/4 pi) times the sum of the signed solid angles of the faces seen from the point (Jacobson et al. 2013). About 1
        inside and 0 outside a closed, outward mesh, -1 inside an inward one, k where k closed copies overlap, and in between across holes;
        it depends on the triangles alone, not on connectivity, welding or manifoldness. Faces with two equal corners (those repeating a
        vertex included) and faces whose plane holds the point contribute 0. A BVH node whose centroid is farther than beta times its
        radius contributes its order-2 moment expansion (Barill et al. 2018); beta = math.inf sums every face exactly (fp32 solid angles,
        fp64 sum). The same bits on every run and for any order of the points. V and F are checked as occluded checks them."""
        fn = "Mesh.winding_number"
        if isinstance(beta, bool) or not isinstance(beta, (int, float, np.integer, np.floating)) or not float(beta) > 0:
            raise RuntimeError("%s: beta must be a positive number (math.inf for the exact sum), got %r" % (fn, beta))
        p = _check_points(fn, points, self.V)
        with torch.cuda.device(p.device):
            V, Fc, bvh = self._bvh(fn)
            return self._winding(fn, p, V, Fc, bvh, beta)

    def _area_cdf(self, fn):
        """the cdf psdf_mesh_sample_surface draws faces from -> (V, F, cdf fp64 [F]): the face areas |(b - a) x (c - a)| / 2 in fp64 (0 for
        faces that repeat a vertex), as int64 fixed point floor(area * 2^62 / (F * max area)), summed by an int64 cumsum on the device
        (integer sums are exact, so the bits are the same on every call; torch's CUDA cumsum of floats is not deterministic) and
        converted to fp64. A face below 2^-62 F of the largest area gets no samples. Faces with an index outside [0, V) and a mesh of
        zero area are refused."""
        V, Fc = self._check_vf(fn)
        nv, nf = V.shape[0], Fc.shape[0]
        with torch.cuda.device(V.device):
            out = ((Fc < 0) | (Fc >= nv)).any(1)
            if bool(out.any()):
                raise RuntimeError("%s: %d faces have a vertex index outside [0, %d)" % (fn, int(out.sum()), nv))
            p = V.double()[Fc.long()]
            area = torch.linalg.vector_norm(torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=1), dim=1) * 0.5
            area[(Fc[:, 0] == Fc[:, 1]) | (Fc[:, 1] == Fc[:, 2]) | (Fc[:, 2] == Fc[:, 0])] = 0
            amax = float(area.max()) if nf else 0.0
            if not amax > 0:
                raise RuntimeError("%s: the mesh has no face of positive area" % fn)
            q = torch.floor(area * (2.0 ** 62 / (amax * nf))).to(torch.int64)
            return V, Fc, torch.cumsum(q, 0).double()

    def _sample_surface(self, fn, nr_samples, seed):
        """nr_samples points drawn by area on the GPU -> (points float32 [N,3], face int32 [N]): sample k depends only on (seed, k)
        (psdf_mesh_sample_surface: SplitMix64, the face by the area cdf of _area_cdf, the sqrt(u) barycentric map), so a larger N extends
        a smaller one, and the result is the same bits on every call."""
        V, Fc, cdf = self._area_cdf(fn)
        with torch.cuda.device(V.device):
            N = int(nr_samples)
            pts = torch.empty(N, 3, dtype=torch.float32, device=V.device)
            face = torch.empty(N, dtype=torch.int32, device=V.device)
            call("psdf_mesh_sample_surface", V.shape[0], Fc.shape[0], V, Fc, cdf, N, int(seed), pts, face)
        return pts, face

    def interpolate(self, other, t):
        """Mesh(torch.lerp(V, other.V, t), F.clone(), None): the in-between mesh of two frames of one topology (EasyPBR's interpolate as
        train_4d_sdf.py uses it); the caller recalculates normals. Refused unless F equals other.F and V has other.V's shape."""
        if not isinstance(other, Mesh):
            raise RuntimeError("Mesh.interpolate: other must be a Mesh, got %s" % type(other).__name__)
        if self.V.shape != other.V.shape:
            raise RuntimeError("Mesh.interpolate: V has shape %s and other.V %s" % (list(self.V.shape), list(other.V.shape)))
        if self.F.shape != other.F.shape or not torch.equal(self.F, other.F.to(self.F.device)):
            raise RuntimeError("Mesh.interpolate: the meshes have different faces; only frames of one topology are interpolated")
        return Mesh(torch.lerp(self.V, other.V, float(t)), self.F.clone(), None)

    # ------------------------------------------------------------------ reading, welding and placing a mesh
    @staticmethod
    def load(path, device="cuda", weld=None):
        """reads a PLY (ascii, binary little or big endian), OBJ or STL (binary or ASCII) file -> Mesh with V float32 [V,3], F int32 [F,3]
        and NV on `device` (device="cpu" reads without a GPU; the GPU operations still need CUDA tensors). The format is told by the
        content (PLY magic, a binary STL's size of 84 + 50 n bytes, a leading "solid"), else by the extension. Polygons are fan-triangulated
        in file order, (p0, pj, pj+1).
        PLY: vertex x y z (float or double) and nx ny nz when all three are there (NV); other fixed-size properties and elements are
        skipped; the face list is vertex_indices or vertex_index with any integer count and index types; other list elements are refused.
        Mesh.save_to_file followed by load gives back V, F and NV bit for bit.
        OBJ: v x y z [w] and f with a, a/b, a//c or a/b/c, 1-based or negative (relative to the vertices read so far); vn is per corner in
        OBJ, so NV is None; other keywords are ignored.
        STL: three vertices per facet, NV None. weld=None welds STL only, through remove_duplicate_vertices, which the connectivity of
        components, decimation, normals and subdivision needs; weld=True welds any format, weld=False keeps the triangle soup.
        Truncated data, indices outside [0, V), unsupported property types and unreadable files raise RuntimeError naming the path; V and
        F must stay below 2^31."""
        path = str(path)
        try:
            with open(path, "rb") as f:
                data = f.read()
        except OSError as e:
            raise RuntimeError("Mesh.load: %s: %s" % (path, e.strerror)) from None
        ext = path.lower().rsplit(".", 1)[-1] if "." in path else ""
        if data.startswith(b"ply\n") or data.startswith(b"ply\r\n"):
            kind, (V, Fc, NV) = "ply", _load_ply(path, data)
        elif _is_binary_stl(data) or data.lstrip().startswith(b"solid") or ext == "stl":
            kind, (V, Fc, NV) = "stl", _load_stl(path, data)
        elif ext == "obj":
            kind, (V, Fc, NV) = "obj", _load_obj(path, data)
        elif ext == "ply":
            raise RuntimeError("Mesh.load: %s: not a PLY file (no 'ply' magic)" % path)
        else:
            raise RuntimeError("Mesh.load: %s: cannot tell the format (PLY, OBJ or STL) from the content or the extension" % path)
        if V.shape[0] > _INT_MAX or Fc.shape[0] > _INT_MAX:
            raise RuntimeError("Mesh.load: %s: %d vertices and %d faces; both must be below 2^31" % (path, V.shape[0], Fc.shape[0]))
        if Fc.size and (Fc.min() < 0 or Fc.max() >= V.shape[0]):
            raise RuntimeError("Mesh.load: %s: %d faces have a vertex index outside [0, %d)" % (
                path, int(((Fc < 0) | (Fc >= V.shape[0])).any(1).sum()), V.shape[0]))
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        m = Mesh(t(V), t(Fc.astype(np.int32)), None if NV is None else t(NV))
        if weld or (weld is None and kind == "stl"):
            m.remove_duplicate_vertices()
        return m

    def remove_duplicate_vertices(self):
        """merges vertices with equal fp32 positions (-0.0 equal to +0.0; exact, no tolerance): each group keeps the vertex with the
        smallest index, the survivors keep their order (and their NV), F is remapped, and faces that then repeat a vertex are dropped.
        V must be finite. CPU or CUDA tensors. -> self"""
        if not bool(torch.isfinite(self.V).all()):
            raise RuntimeError("Mesh.remove_duplicate_vertices: V has values that are not finite")
        nv = self.V.shape[0]
        if nv == 0:
            return self
        key = (self.V.float() + 0.0).view(torch.int32).long()          # + 0.0 turns -0.0 into +0.0
        _, group = torch.unique(key, dim=0, return_inverse=True)
        idx = torch.arange(nv, device=self.V.device)
        first = torch.full((int(group.max()) + 1,), nv, dtype=torch.int64, device=self.V.device).scatter_reduce(0, group, idx, "amin")
        rep = first[group]
        kept = rep == idx
        new_id = torch.cumsum(kept.to(torch.int64), 0) - 1
        Fn = new_id[rep[self.F.long()]]
        Fn = Fn[(Fn[:, 0] != Fn[:, 1]) & (Fn[:, 1] != Fn[:, 2]) & (Fn[:, 2] != Fn[:, 0])]
        self.F = Fn.to(torch.int32).reshape(-1, 3)
        self.V = self.V[kept]
        if self.NV is not None:
            self.NV = self.NV[kept]
        return self

    def remove_unreferenced_verts(self):
        """drops the vertices no face uses and compacts the mesh as remove_marked_vertices does. -> self"""
        used = torch.zeros(self.V.shape[0], dtype=torch.bool, device=self.V.device)
        used[self.F.long().reshape(-1)] = True
        return self.remove_marked_vertices(used, True)

    def _bounds(self, fn):
        if self.V.shape[0] == 0:
            raise RuntimeError("%s: the mesh has no vertices" % fn)
        return self.V.min(0).values, self.V.max(0).values

    def normalize_position(self):
        """translates V by minus the centre of its bounding box, c = (min + max) / 2 (fp32, over all vertices), and returns c (float32
        tensor [3]); translate(c) undoes it. EasyPBR's definition is not in the reference's checkout, so this formula is ours, not pinned
        to it."""
        lo, hi = self._bounds("Mesh.normalize_position")
        c = (lo + hi) / 2
        self.translate(-c)
        return c

    def normalize_size(self):
        """scales V by s = 1 / d with d = |max - min| the bounding-box diagonal, d = sqrt((dx dx + dy dy) + dz dz) in fp32 and s = 1.0 / d
        in fp64, applied as scale_mesh(s); returns s (a float), so scale_mesh(1.0 / s) undoes it. EasyPBR's definition is not in the
        reference's checkout, so this formula is ours, not pinned to it."""
        lo, hi = self._bounds("Mesh.normalize_size")
        e = hi - lo
        d = float(torch.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]))
        if not d > 0:
            raise RuntimeError("Mesh.normalize_size: the bounding box has zero size")
        s = 1.0 / d
        self.scale_mesh(s)
        return s

    def scale_mesh(self, s):
        """V = V * s (fp32). -> self"""
        self.V = self.V * s
        return self

    def translate(self, t):
        """V = V + t (fp32), t a 3-vector. -> self"""
        self.V = self.V + torch.as_tensor(t, dtype=self.V.dtype, device=self.V.device)
        return self

    def save_to_file(self, path):
        """binary little-endian PLY: x y z nx ny nz (float) per vertex (zero normals when there are none), uchar int vertex_indices per
        face"""
        V = self.V.detach().float().cpu().contiguous()
        NV = self.NV.detach().float().cpu() if self.NV is not None else torch.zeros_like(V)
        Fc = self.F.detach().to(torch.int32).cpu().contiguous()
        header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                  "property float nx\nproperty float ny\nproperty float nz\nelement face %d\nproperty list uchar int vertex_indices\n"
                  "end_header\n" % (V.shape[0], Fc.shape[0]))
        vbytes = torch.cat([V, NV], 1).numpy().astype("<f4").tobytes()
        frec = np.empty(Fc.shape[0], dtype=[("n", "u1"), ("idx", "<i4", (3,))])
        frec["n"] = 3
        frec["idx"] = Fc.numpy()
        with open(path, "wb") as f:
            f.write(header.encode("ascii"))
            f.write(vbytes)
            f.write(frec.tobytes())


def _check_rays(fn, origins, dirs, V):
    if not isinstance(V, torch.Tensor) or not V.is_cuda:
        raise RuntimeError("%s: V must be a CUDA tensor (there is no CPU path)" % fn)
    out = []
    for name, x in (("origins", origins), ("dirs", dirs)):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or x.dim() != 2 or x.shape[1] != 3:
            raise RuntimeError("%s: %s must be a float32 tensor of shape [R,3]" % (fn, name))
        if x.device != V.device:
            raise RuntimeError("%s: %s must be on V's device %s, got %s" % (fn, name, V.device, x.device))
        if not bool(torch.isfinite(x).all()):
            raise RuntimeError("%s: %s has values that are not finite" % (fn, name))
        out.append(x.contiguous())
    if out[0].shape[0] != out[1].shape[0]:
        raise RuntimeError("%s: %d origins and %d dirs" % (fn, out[0].shape[0], out[1].shape[0]))
    return out


def _check_window(fn, tnear, tfar):
    if not (math.isfinite(float(tnear)) and not math.isnan(float(tfar))):
        raise RuntimeError("%s: tnear must be finite and tfar a number, got %r, %r" % (fn, tnear, tfar))


def _check_camera(fn, name, x, shape, device):
    """float32 [I, *shape] finite on device -> contiguous"""
    if not isinstance(x, torch.Tensor) or x.dim() != 3 or tuple(x.shape[1:]) != shape:
        raise RuntimeError("%s: %s must be a tensor of shape [I,%d,%d], got %s" % (
            fn, name, shape[0], shape[1], list(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__))
    if x.dtype != torch.float32:
        raise RuntimeError("%s: %s must be float32, got %s" % (fn, name, x.dtype))
    if x.device != device:
        raise RuntimeError("%s: %s must be on V's device %s, got %s" % (fn, name, device, x.device))
    if not bool(torch.isfinite(x).all()):
        raise RuntimeError("%s: %s has values that are not finite" % (fn, name))
    return x.contiguous()


def _check_vertex_field(fn, name, x, V):
    """None, or float32 [V,3] on V's device -> contiguous"""
    if x is None:
        return None
    if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or tuple(x.shape) != tuple(V.shape):
        raise RuntimeError("%s: %s must be a float32 tensor of shape [V,3] = %s" % (fn, name, list(V.shape)))
    if x.device != V.device:
        raise RuntimeError("%s: %s must be on V's device %s, got %s" % (fn, name, V.device, x.device))
    return x.contiguous()


def _check_points(fn, points, V):
    if not isinstance(V, torch.Tensor) or not V.is_cuda:
        raise RuntimeError("%s: V must be a CUDA tensor (there is no CPU path)" % fn)
    if not isinstance(points, torch.Tensor) or points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("%s: points must be a float32 tensor of shape [P,3]" % fn)
    if points.device != V.device:
        raise RuntimeError("%s: points must be on V's device %s, got %s" % (fn, V.device, points.device))
    if not bool(torch.isfinite(points).all()):
        raise RuntimeError("%s: points has values that are not finite" % fn)
    return points.contiguous()


def mesh_distance(a, b, nr_samples=1_000_000, seed=0):
    """how far apart two meshes are, on the GPU: nr_samples area-weighted samples of each surface (the same seed for both, so swapping a
    and b swaps the two directions exactly), each queried against the other mesh with Mesh.closest_points. -> dict:
      accuracy      mean distance from the samples of a to b
      completeness  mean distance from the samples of b to a
      chamfer       (accuracy + completeness) / 2
      hausdorff     the larger of the two maximum distances
      dist_a_to_b, dist_b_to_a   the per-sample distances, float32 [nr_samples] on the device
    The means are fp64 sums of the fp32 distances, the same bits on every call. Sample k of a mesh depends only on (seed, k): SplitMix64
    picks a face by its share of the area (fixed point, summed exactly) and a point by the sqrt(u) barycentric map (psdf_mesh_sample_surface). Both meshes are
    checked as Mesh.occluded checks them (V float32 CUDA and finite, F int32 on its device with indices in [0, V)) and need a face of
    positive area; each mesh's BVH is built once, for the queries against it. Thresholded precision, recall or F-score follow from the
    returned distances."""
    fn = "mesh_distance"
    for name, m in (("a", a), ("b", b)):
        if not isinstance(m, Mesh):
            raise RuntimeError("%s: %s must be a Mesh, got %s" % (fn, name, type(m).__name__))
    if isinstance(nr_samples, bool) or not isinstance(nr_samples, (int, np.integer)) or not 1 <= nr_samples <= 256 * _INT_MAX:
        raise RuntimeError("%s: nr_samples must be a positive integer, got %r" % (fn, nr_samples))
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 64:
        raise RuntimeError("%s: seed must be an integer in [0, 2^64), got %r" % (fn, seed))
    a._check_vf(fn)
    b._check_vf(fn)
    if b.V.device != a.V.device:
        raise RuntimeError("%s: the meshes are on %s and %s; both must be on one device" % (fn, a.V.device, b.V.device))
    with torch.cuda.device(a.V.device):
        sa, _ = a._sample_surface(fn, int(nr_samples), int(seed))
        sb, _ = b._sample_surface(fn, int(nr_samples), int(seed))
        d_ab = b.closest_points(sa)[0]
        d_ba = a.closest_points(sb)[0]
        acc, comp = d_ab.double().mean(), d_ba.double().mean()
        hd = torch.maximum(d_ab.max(), d_ba.max())
        acc, comp, hd = torch.stack([acc, comp, hd.double()]).tolist()
    return {"accuracy": acc, "completeness": comp, "chamfer": (acc + comp) / 2, "hausdorff": hd, "dist_a_to_b": d_ab,
            "dist_b_to_a": d_ba}


def fibonacci_directions(S):
    """the S directions of Mesh.ambient_occlusion, float32 [S,3] on the host: z = 1 - (2s + 1) / S, phi = s pi (3 - sqrt 5),
    (sqrt(1 - z^2) cos phi, sqrt(1 - z^2) sin phi, z), computed in fp64 and rounded to fp32"""
    s = np.arange(S, dtype=np.float64)
    z = 1.0 - (2.0 * s + 1.0) / S
    phi = s * (math.pi * (3.0 - math.sqrt(5.0)))
    r = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(np.float32)


# ---------------------------------------------------------------- mesh sequences (train_4d_sdf.py:47-141)
_SEQ_MAX_INDEX = 12          # the reference reads files while i <= min(12, n): at most 13
_SEQ_MULTIPLICITY = 20       # in-between meshes per pair of frames
_SEQ_AO_SAMPLES = 100
_SEQ_AO_MIN = 0.01


def natural_key(name):
    """sort key that orders the digit runs of a name by value: f_2.obj < f_10.obj (natsort's default for such names)"""
    return [int(t) if i % 2 else t for i, t in enumerate(re.split(r"(\d+)", name))]


def sequence_files(names):
    """the frames load_mesh_sequence reads of a folder's file names: those ending in .obj or .ply, natural-sorted, at most the first 13.
    The reference matches ".obj" or ".py"; ".py" is read as a typo for ".ply"."""
    files = sorted((n for n in names if n.endswith(".obj") or n.endswith(".ply")), key=natural_key)
    return files[:min(_SEQ_MAX_INDEX, len(files)) + 1]


def load_mesh_sequence(folder, device="cuda"):
    """train_4d_sdf.py's load_mesh_sequence -> (points_time float32 [P,4], normals float32 [P,3]) on `device`, step by step:
    - the frames are sequence_files(os.listdir(folder)), loaded with Mesh.load; fewer than 2 are refused, and so is a frame whose faces
      differ from frame 0's (named);
    - frame 0: s = normalize_size(), c = normalize_position(); every other frame: scale_mesh(s), translate(-c). The reference's EasyPBR
      calls are scale_mesh(1.0 / scale) and translate_model_matrix(pos): its normalize_size returns the inverse of the factor it applies
      and normalize_position the translation, while ours return the factor and the centre, hence s and -c here;
    - every frame: recalculate_normals(), upsample(2, True) (Loop, normals recalculated);
    - frame 0's ambient_occlusion(100) < 0.01 marks the vertices removed from every frame: remove_marked_vertices(mask, False), then
      remove_unreferenced_verts();
    - each consecutive pair (a, b) gives 20 meshes a.interpolate(b, j / 20), j = 0 .. 19, each with recalculate_normals(); the last frame is
      never an endpoint itself;
    - the K = 20 (n - 1) meshes are concatenated in order, mesh k with the time column fp32(k / (K - 1)).
    The viewer colouring of the reference is left out."""
    fn = "load_mesh_sequence"
    folder = str(folder)
    files = sequence_files(os.listdir(folder))
    if len(files) < 2:
        raise RuntimeError("%s: %s: %d mesh files (.obj or .ply); a sequence needs at least 2" % (fn, folder, len(files)))
    frames, mask, F0 = [], None, None
    for i, name in enumerate(files):
        path = os.path.join(folder, name)
        m = Mesh.load(path, device=device)
        if i == 0:
            F0, nv0 = m.F, m.V.shape[0]
            s = m.normalize_size()
            c = m.normalize_position()
        else:
            if m.F.shape != F0.shape or not torch.equal(m.F, F0) or m.V.shape[0] != nv0:
                raise RuntimeError("%s: %s: its faces (or vertex count) differ from those of %s; every frame must have one topology" % (
                    fn, path, files[0]))
            m.scale_mesh(s)
            m.translate(-c)
        m.recalculate_normals()
        m.upsample(2, True)
        if i == 0:
            mask = m.ambient_occlusion(_SEQ_AO_SAMPLES) < _SEQ_AO_MIN
        m.remove_marked_vertices(mask, False)
        m.remove_unreferenced_verts()
        frames.append(m)
    meshes = []
    for a, b in zip(frames[:-1], frames[1:]):
        for j in range(_SEQ_MULTIPLICITY):
            meshes.append(a.interpolate(b, j / _SEQ_MULTIPLICITY).recalculate_normals())
    K = len(meshes)
    pts, nrm = [], []
    for k, m in enumerate(meshes):
        pts.append(torch.cat([m.V, torch.full((m.V.shape[0], 1), k / (K - 1), dtype=torch.float32, device=m.V.device)], 1))
        nrm.append(m.NV)
    return torch.cat(pts), torch.cat(nrm)


# ---------------------------------------------------------------- reading meshes (host side)
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
              "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _fan(polys):
    """[n, c] polygons -> [n (c - 2), 3] triangles (p0, pj, pj+1), j = 1 .. c - 2, polygon by polygon"""
    n, c = polys.shape
    if c < 3:
        return np.zeros((0, 3), dtype=np.int64)
    j = np.arange(1, c - 1)
    return np.stack([np.broadcast_to(polys[:, :1], (n, c - 2)), polys[:, j], polys[:, j + 1]], 2).reshape(-1, 3)


def _ply_type(path, t):
    if t not in _PLY_TYPES:
        raise RuntimeError("Mesh.load: %s: unsupported PLY property type %r" % (path, t))
    return _PLY_TYPES[t]


def _ply_header(path, data):
    """-> (format, [(element, count, [(name, type) or (name, count type, item type)])], body offset)"""
    end = data.find(b"end_header")
    if end < 0:
        raise RuntimeError("Mesh.load: %s: PLY header without end_header" % path)
    nl = data.find(b"\n", end)
    body = len(data) if nl < 0 else nl + 1
    fmt, elements = None, []
    for line in data[:end].decode("ascii", "replace").splitlines()[1:]:
        w = line.split()
        if not w or w[0] in ("comment", "obj_info"):
            continue
        if w[0] == "format" and len(w) >= 2:
            fmt = w[1]
        elif w[0] == "element" and len(w) == 3:
            elements.append((w[1], int(w[2]), []))
        elif w[0] == "property" and elements and len(w) == 5 and w[1] == "list":
            elements[-1][2].append((w[4], _ply_type(path, w[2]), _ply_type(path, w[3])))
        elif w[0] == "property" and elements and len(w) == 3:
            elements[-1][2].append((w[2], _ply_type(path, w[1])))
        else:
            raise RuntimeError("Mesh.load: %s: cannot read the PLY header line %r" % (path, line))
    if fmt not in ("ascii", "binary_little_endian", "binary_big_endian"):
        raise RuntimeError("Mesh.load: %s: unsupported PLY format %r" % (path, fmt))
    return fmt, elements, body


def _ply_lists(path, buf, off, n, pre, post, cdt, idt):
    """n records of (pre bytes, count cdt, count x idt, post bytes) from buf at off, read a run of equal counts at a time ->
    (triangles [m, 3] int64, in file order, the offset after the records)"""
    cs, isz = cdt.itemsize, idt.itemsize
    tris, i = [], 0
    while i < n:
        if off + pre + cs > len(buf):
            raise RuntimeError("Mesh.load: %s: truncated PLY face data (%d of %d faces)" % (path, i, n))
        c0 = np.frombuffer(buf, cdt, 1, off + pre)[0]
        c = int(c0)
        if c < 0 or c != c0:
            raise RuntimeError("Mesh.load: %s: a PLY face with %d vertices" % (path, c))
        rec = pre + cs + c * isz + post
        j, w = 1, 64
        while i + j < n:
            k = min(w, n - i - j, max((len(buf) - off - j * rec - pre - cs) // rec + 1, 0))
            if k <= 0:
                break
            counts = np.ndarray((k,), cdt, buf, off + j * rec + pre, (rec,))
            bad = np.flatnonzero(counts != c)
            if bad.size:
                j += int(bad[0])
                break
            j += k
            w *= 2
        if off + j * rec > len(buf):
            raise RuntimeError("Mesh.load: %s: truncated PLY face data (%d of %d faces)" % (path, i, n))
        idx = np.ndarray((j, c), idt, buf, off + pre + cs, (rec, isz))
        if idx.dtype.kind == "f" and not (idx == np.floor(idx)).all():
            raise RuntimeError("Mesh.load: %s: a PLY face index that is not an integer" % path)
        tris.append(_fan(idx.astype(np.int64)))
        off += j * rec
        i += j
    return (np.concatenate(tris) if tris else np.zeros((0, 3), dtype=np.int64)), off


def _load_ply(path, data):
    fmt, elements, off = _ply_header(path, data)
    if fmt == "ascii":
        # every value becomes an fp64 token, and the binary reader runs over them with every type 8 bytes wide
        try:
            buf = np.array(data[off:].split(), dtype=np.float64).tobytes()
        except ValueError:
            raise RuntimeError("Mesh.load: %s: a PLY value that is not a number" % path) from None
        to = lambda t: np.dtype("f8")
        off = 0
    else:
        buf, bo = data, "<" if fmt == "binary_little_endian" else ">"
        to = lambda t: np.dtype(bo + t)
    V = NV = Fc = None
    for name, n, props in elements:
        lists = [p for p in props if len(p) == 3]
        if not lists:
            dt = np.dtype([(p[0], to(p[1])) for p in props])
            if off + n * dt.itemsize > len(buf):
                raise RuntimeError("Mesh.load: %s: truncated PLY %s data (%d records expected)" % (path, name, n))
            rec = np.frombuffer(buf, dt, n, off)
            off += n * dt.itemsize
            if name == "vertex":
                names = dt.names or ()
                for a in ("x", "y", "z", "nx", "ny", "nz"):
                    if a in names and dt[a].kind != "f":
                        raise RuntimeError("Mesh.load: %s: unsupported type of vertex property %s (float or double)" % (path, a))
                if not all(a in names for a in "xyz"):
                    raise RuntimeError("Mesh.load: %s: the PLY vertices have no x y z" % path)
                V = np.stack([rec[a] for a in "xyz"], 1).astype(np.float32)
                if all(a in names for a in ("nx", "ny", "nz")):
                    NV = np.stack([rec[a] for a in ("nx", "ny", "nz")], 1).astype(np.float32)
            continue
        if name != "face" or len(lists) != 1 or lists[0][0] not in ("vertex_indices", "vertex_index"):
            raise RuntimeError("Mesh.load: %s: unsupported PLY list element %r (%s)" % (path, name, ", ".join(p[0] for p in lists)))
        _, ct, it = lists[0]
        if np.dtype(ct).kind not in "iu" or np.dtype(it).kind not in "iu":
            raise RuntimeError("Mesh.load: %s: unsupported PLY face list type (%s %s): integers expected" % (path, ct, it))
        k = props.index(lists[0])
        size = lambda ps: sum(to(p[1]).itemsize for p in ps)
        tri, off = _ply_lists(path, buf, off, n, size(props[:k]), size(props[k + 1:]), to(ct), to(it))
        Fc = tri
    if V is None:
        raise RuntimeError("Mesh.load: %s: the PLY file has no vertex element" % path)
    return V, (np.zeros((0, 3), dtype=np.int64) if Fc is None else Fc), NV


def _load_obj(path, data):
    vs, faces = [], []
    for ln, line in enumerate(data.decode("utf-8", "replace").splitlines(), 1):
        w = line.split()
        if not w:
            continue
        try:
            if w[0] == "v":
                vs.append([float(x) for x in w[1:4]] if len(w) >= 4 else None)
                if vs[-1] is None:
                    raise ValueError
            elif w[0] == "f":
                idx = [int(x.split("/")[0]) for x in w[1:]]
                faces.append([i - 1 if i > 0 else len(vs) + i if i < 0 else -(2 ** 40) for i in idx])
        except ValueError:
            raise RuntimeError("Mesh.load: %s: cannot read OBJ line %d: %r" % (path, ln, line)) from None
    tris = [(f[0], f[j], f[j + 1]) for f in faces for j in range(1, len(f) - 1)]
    V = np.array(vs, dtype=np.float64).reshape(-1, 3).astype(np.float32)
    return V, np.array(tris, dtype=np.int64).reshape(-1, 3), None


_STL_REC = np.dtype([("n", "<f4", (3,)), ("v", "<f4", (3, 3)), ("attr", "<u2")])


def _is_binary_stl(data):
    return len(data) >= 84 and 84 + 50 * int(np.frombuffer(data, "<u4", 1, 80)[0]) == len(data)


def _load_stl(path, data):
    if _is_binary_stl(data):
        n = int(np.frombuffer(data, "<u4", 1, 80)[0])
        V = np.frombuffer(data, _STL_REC, n, 84)["v"].reshape(-1, 3).astype(np.float32)
    else:
        import re
        text = data.decode("ascii", "replace")
        if not text.lstrip().startswith("solid"):
            raise RuntimeError("Mesh.load: %s: neither a binary STL (84 + 50 n bytes for n facets) nor an ASCII STL" % path)
        try:
            V = np.array(re.findall(r"\bvertex\s+(\S+)\s+(\S+)\s+(\S+)", text), dtype=np.float64).reshape(-1, 3).astype(np.float32)
        except ValueError:
            raise RuntimeError("Mesh.load: %s: an STL vertex that is not a number" % path) from None
        if V.shape[0] % 3 or V.shape[0] // 3 != len(re.findall(r"\bendfacet\b", text)):
            raise RuntimeError("Mesh.load: %s: truncated ASCII STL: %d vertices in %d complete facets" % (
                path, V.shape[0], len(re.findall(r"\bendfacet\b", text))))
    return V, np.arange(V.shape[0], dtype=np.int64).reshape(-1, 3), None


def _mesh_grid(N, min_val, max_val, threshold, dev, values):
    """the grid linspace(min_val, max_val, N)^3 (axis 0 = x) a slab of slices at a time: values(pts [n,3], out [n]) writes the volume's
    values at the slab's points into out (a view of the slab buffer), and each slab goes through the marching-cubes kernels with
    `threshold` as it comes. Vertices rescaled as the reference does, v / fp32(N - 1) * fp32(max_val - min_val) + min_val in fp32.
    -> (V [V,3], F [F,3] int32)"""
    lin = torch.linspace(min_val, max_val, N, device=dev)
    S = _slab_slices(N, N, N)
    vals = torch.empty(S + 1, N, N, device=dev)
    mc = _SlabMarchingCubes(N, S, N, N, threshold, dev, affine=(float(N - 1), float(max_val - min_val), float(min_val)))
    for i0 in range(0, N - 1, S):
        i1 = min(i0 + S, N - 1)
        first = 0 if i0 == 0 else 1
        if first:
            vals[0].copy_(vals[S])               # the shared slice of the previous slab
        rows = lin[i0 + first:i1 + 1]
        pts = torch.stack(torch.meshgrid(rows, lin, lin, indexing="ij"), -1).reshape(-1, 3)
        values(pts, vals[first:i1 - i0 + 1].view(-1))
        del pts
        mc.run(vals[:i1 - i0 + 1], i0)
    return mc.result()


def _check_extraction_args(fn, model, kind, nr_points_per_dim, min_val, max_val, threshold):
    if getattr(model, "in_channels", None) != 3:
        raise RuntimeError("%s: the model has in_channels %s; meshes are extracted from a 3-D %s (in_channels 3), %s" % (
            fn, getattr(model, "in_channels", None), kind[0], kind[1]))
    N = int(nr_points_per_dim)
    if N < 2:
        raise RuntimeError("%s: nr_points_per_dim must be >= 2, got %d" % (fn, N))
    if not all(math.isfinite(float(x)) for x in (min_val, max_val, threshold)):
        raise RuntimeError("%s: min_val, max_val and threshold must be finite" % fn)
    return N


@torch.no_grad()
def extract_mesh_from_sdf_model(model, nr_points_per_dim, min_val, max_val, threshold=0, iter_nr=9999999):
    """sdf_utils.py:252-292 for an SDF with in_channels 3: the grid linspace(min_val, max_val, N)^3 (axis 0 = x), evaluated by the model's
    FusedSDF (value only) a slab of slices at a time and meshed on the GPU as it comes; vertices rescaled as the reference does,
    v / fp32(N - 1) * fp32(max_val - min_val) + min_val in fp32; normals F.normalize of the SDF gradient at the vertices (outward).
    iter_nr selects the coarse-to-fine window (the reference's 9999999: all levels). Restores model.training and model.last_iter_nr and
    attaches nothing to the model. -> Mesh"""
    from .fused import FusedSDF
    N = _check_extraction_args("extract_mesh_from_sdf_model", model, ("SDF", "a space-time SDF (in_channels 4) has no single surface"),
                               nr_points_per_dim, min_val, max_val, threshold)
    fused = getattr(model, "fused", None) or FusedSDF(model)
    dev = model.encoding.lattice_values.device
    was_training, last_iter_nr = model.training, model.last_iter_nr
    model.eval()
    try:
        with torch.cuda.device(dev):
            def sdf(pts, out):
                out.copy_(fused(pts, iter_nr, with_gradient=False, with_geom=False)[0].view(-1))
            V, Fc = _mesh_grid(N, min_val, max_val, threshold, dev, sdf)
            NV = torch.empty_like(V)
            for a in range(0, V.shape[0], _SLAB_POINTS):
                g = fused(V[a:a + _SLAB_POINTS], iter_nr, with_gradient=True, with_geom=False)[1]
                NV[a:a + _SLAB_POINTS] = F.normalize(g, dim=1)
        return Mesh(V, Fc, NV)
    finally:
        model.train(was_training)
        model.last_iter_nr = last_iter_nr


@torch.no_grad()
def extract_mesh_from_density_model(model, nr_points_per_dim, min_val, max_val, threshold=0, iter_nr=9999999):
    """sdf_utils.py:339-380 for a NeRF density model (NerfHash with in_channels 3, e.g. NerfTrainer.model): the grid
    linspace(min_val, max_val, N)^3 (axis 0 = x), evaluated by the density-only fused kernel (FusedNerfHash.density) a slab of slices
    at a time and meshed on the GPU as it comes. Inside is density > threshold: the marching-cubes kernels see -density against
    -threshold (negation is exact, so the vertices are those of the density at threshold, and faces wind counter-clockwise seen from
    outside the dense region). Vertices rescaled as extract_mesh_from_sdf_model does. Normals: F.normalize of the central difference
    density(v - h e_i) - density(v + h e_i), i = x, y, z, with h = fp32(max_val - min_val) / fp32(N - 1) (one grid spacing); they point
    out of the dense region. The reference's unused `lattice` argument is dropped. iter_nr selects the coarse-to-fine window (the
    reference's 9999999: all levels). Restores model.training and model.last_iter_nr and attaches nothing to the model. -> Mesh"""
    from .fused import FusedNerfHash
    N = _check_extraction_args("extract_mesh_from_density_model", model,
                               ("NeRF density model", "a background NerfHash (in_channels 4) has no single surface"),
                               nr_points_per_dim, min_val, max_val, threshold)
    fused = getattr(model, "fused", None) or FusedNerfHash(model)
    dev = model.encoding.lattice_values.device
    was_training, last_iter_nr = model.training, model.last_iter_nr
    model.eval()
    try:
        with torch.cuda.device(dev):
            def neg_density(pts, out):
                torch.neg(fused.density(pts, iter_nr).view(-1), out=out)
            V, Fc = _mesh_grid(N, min_val, max_val, -float(threshold), dev, neg_density)
            h = float(np.float32(max_val - min_val) / np.float32(N - 1))
            offs = h * torch.eye(3, device=dev)
            NV = torch.empty_like(V)
            step = _SLAB_POINTS // 6
            for a in range(0, V.shape[0], step):
                v = V[a:a + step]
                d = fused.density(torch.cat([v - offs[i] for i in range(3)] + [v + offs[i] for i in range(3)]), iter_nr).view(6, -1)
                NV[a:a + step] = F.normalize((d[:3] - d[3:]).t().contiguous(), dim=1)
        return Mesh(V, Fc, NV)
    finally:
        model.train(was_training)
        model.last_iter_nr = last_iter_nr


__all__ = ["Mesh", "marching_cubes", "extract_mesh_from_sdf_model", "extract_mesh_from_density_model", "load_mesh_sequence",
           "fibonacci_directions", "mesh_distance"]
