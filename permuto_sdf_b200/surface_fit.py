"""SDF from an oriented point cloud on the fused kernels: the loop of train_sdf_from_mesh.py:116-165 as a direct, graph-replayable
kernel sequence.

Each iteration of the reference draws 3000 cloud points with their normals and 30 000 uniform points in the bounding box, evaluates the
SDF and its gradient at all of them, applies `sdf_loss` (sdf_utils.py:16-57) divided by 30 000 and runs AdamW. `SurfaceFit.step()`
issues the same mathematics without autograd:

    torch.randint + torch.rand          the draws (cloud rows, box coordinates)                                        2 launches
    psdf_surface_fit_points             cloud rows + normals (index_select) and box points into one [Ns + No, 3]       1
    coarse-to-fine window               from the device-resident iteration (element-wise torch ops while it ramps)
    psdf_sdf_fused_forward              sdf and d sdf/dx at every row (out_dim 1: the reference's geom_feat_size_out=0)   1
    psdf_surface_fit_loss               the four means, the weighted total and the seeds d loss / d {sdf, d sdf/dx}    1
    psdf_sdf_fused_backward_multi       one sample set, into the optimizer's .grad views                              2 kernels
    psdf_adamw_multi_step               AdamW over the model's parameters                                              1
    psdf_sdf_mlp_pack_advance           operand re-pack + the device-resident step count and iteration                1

Buffers depend only on (Ns, No, P), and the step count and iteration number live on the device in eager runs too, so an eager run and a
run replayed from a captured CUDA graph (`enable_cuda_graph()`) give the same bits. The autograd formulation of the reference (`sdf_loss`
below, `loss.backward()`, the optimizer step) is the fallback and the yardstick of the tests and of tools/bench_surface_fit.py.

`SpaceTimeFit` is the same loop for train_4d_sdf.py:194-241: a space-time SDF (SDF(4, ...)) fitted to a point sequence [P,4] (x, y, z, t),
box points with a uniform time column, and the sdf_loss of the SPATIAL gradient (the reference keeps [:, 0:3] of the [N,4] gradient). Its
direct sequence runs psdf_spacetime_fit_points and the pos_dim = 4 fused pair (psdf_sdf_fused_forward_dim, _backward_multi_dim), which
form exactly that spatial gradient."""
import os

import torch
import torch.nn.functional as F

from ._lib import call
from .models import SDF, DeviceIter
from .permuto_sdf import AABB

_INT32_MAX = 2 ** 31 - 1
SDF_LOSS_WEIGHTS = (5e1, 1e2, 3e3, 1e2)         # eikonal, normal, |sdf|, off-surface (sdf_utils.py:47)
LOSS_SCALE = 1.0 / 30000                        # train_sdf_from_mesh.py:136


def sdf_loss(surface_sdf, surface_sdf_gradients, offsurface_sdf, offsurface_sdf_gradients, gt_normals, eik_clamp=None):
    """sdf_utils.py:16-57 (equation 6 of Gropp et al. 2020) without the Gaussian eikonal clamp -> the weighted total. The four unweighted
    means are left in sdf_loss.terms (eikonal, normal, sdf, off-surface)."""
    if eik_clamp is not None:
        raise NotImplementedError("sdf_loss: eik_clamp is not supported")
    all_gradients = torch.cat([surface_sdf_gradients, offsurface_sdf_gradients], 0)
    eikonal_loss = torch.abs(all_gradients.norm(dim=-1) - 1)
    loss_surface_sdf = torch.abs(surface_sdf)
    loss_surface_normal = 1 - F.cosine_similarity(surface_sdf_gradients, gt_normals, dim=-1)
    loss_offsurface_high_sdf = torch.exp(-1e2 * torch.abs(offsurface_sdf))
    terms = (eikonal_loss.mean(), loss_surface_normal.mean(), loss_surface_sdf.mean(), loss_offsurface_high_sdf.mean())
    sdf_loss.terms = terms
    w = SDF_LOSS_WEIGHTS
    return terms[0] * w[0] + terms[1] * w[1] + terms[2] * w[2] + terms[3] * w[3]


def _check_cloud(points, normals, D=3, who="SurfaceFit"):
    """-> P; RuntimeError with the reason for clouds the kernels cannot take (points [P,D], normals [P,3])"""
    for name, t, w in (("points", points, D), ("normals", normals, 3)):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError("%s: %s must be a tensor" % (who, name))
        if t.dim() != 2 or t.shape[1] != w:
            raise RuntimeError("%s: %s should have shape [P,%d] but has %s" % (who, name, w, tuple(t.shape)))
        if t.dtype != torch.float32:
            raise RuntimeError("%s: %s must be float32, got %s" % (who, name, t.dtype))
    if points.shape[0] != normals.shape[0]:
        raise RuntimeError("%s: %d points but %d normals" % (who, points.shape[0], normals.shape[0]))
    if points.device != normals.device:
        raise RuntimeError("%s: points on %s but normals on %s" % (who, points.device, normals.device))
    P = int(points.shape[0])
    if P == 0:
        raise RuntimeError("%s: the point cloud is empty" % who)
    if D * P > _INT32_MAX:
        raise RuntimeError("%s: %d points are more than the kernels' 32-bit row indexing takes (at most %d)" % (who, P, _INT32_MAX // D))
    if points.device.type != "cuda":
        raise RuntimeError("%s: the point cloud must be on a CUDA device, got %s" % (who, points.device))
    return P


def _check_counts(nr_surface, nr_offsurface, D=3, who="SurfaceFit"):
    Ns, No = int(nr_surface), int(nr_offsurface)
    if Ns < 1 or No < 1:
        raise RuntimeError("%s.step: needs at least one surface and one box point per iteration (got %d and %d); the reference's "
                           "mean over an empty set is NaN" % (who, Ns, No))
    if D * (Ns + No) > _INT32_MAX:
        raise RuntimeError("%s.step: %d rows are more than the kernels' 32-bit row indexing takes (at most %d)"
                           % (who, Ns + No, _INT32_MAX // D))
    return Ns, No


class SurfaceFit:
    """Fit the SDF network to an oriented point cloud: the state and the loop of train_sdf_from_mesh.py (SDF(3, AABB, 0, 5000) with the
    reference's 24 levels, 2^18 entries and 32-wide MLP, AdamW with betas (0.9, 0.99), eps 1e-15, no weight decay, constant lr).

    points, normals: [P,3] float32 on the GPU. Each `step()` draws `nr_surface` cloud rows and `nr_offsurface` uniform box points from
    torch's generator. optimizer "fused" (flat-buffer AdamW kernel) or "adamw" (torch.optim.AdamW). direct: None = the direct kernel
    sequence whenever the configuration allows it (fused training kernels, fused optimizer), True = require it, False = the autograd
    formulation. deterministic: the library's deterministic mode for this device (order-independent reductions). `execution` records
    which path runs and why."""
    POS_DIM = 3                                                 # columns of a point (SpaceTimeFit: 4)
    DRAWS = ("surface_fit_idx", "surface_fit_u01")              # names of the random draws of one iteration (fixed_random keys)
    STATE_FILE = "surface_fit_state.pt"
    # the pos_dim-specific entry points of the direct sequence, with their leading arguments
    POINTS_FN, FORWARD_FN, BACKWARD_FN = ("psdf_surface_fit_points",), ("psdf_sdf_fused_forward",), ("psdf_sdf_fused_backward_multi",)
    # with fused_training, the model's own get_sdf_and_gradient (the autograd formulation) also runs on the fused training pair. The direct
    # sequence does not depend on it: it calls the kernels itself. SpaceTimeFit: False (that call returns d sdf / dt, which the pair does
    # not form)
    MODEL_ON_FUSED_PAIR = True

    def __init__(self, points, normals, nr_levels=24, capacity=2 ** 18, hidden=32, box_size=(1, 1, 1), box_translation=(0, 0, 0),
                 nr_iters_for_c2f=5000, lr=1e-3, optimizer="fused", deterministic=False, direct=None, seed=0, fused_training=True):
        who = type(self).__name__
        self.nr_points = _check_cloud(points, normals, self.POS_DIM, who)
        if optimizer not in ("fused", "adamw"):
            raise RuntimeError("%s: optimizer must be 'fused' or 'adamw', got %r" % (who, optimizer))
        dev = points.device
        self.points, self.normals = points.detach().contiguous(), normals.detach().contiguous()
        torch.manual_seed(seed)
        with torch.cuda.device(dev):
            self.aabb = AABB(box_size, box_translation)
            self.model_sdf = SDF(self.POS_DIM, self.aabb, 0, nr_iters_for_c2f, nr_levels, capacity, hidden).to(dev)
            call("psdf_set_deterministic", 1 if deterministic else 0, nr_levels * capacity * 2, 1)
        self.model_sdf.enable_fused_inference()
        self.execution = {"sdf_training": "per-op kernels + autograd"}
        if fused_training and self.MODEL_ON_FUSED_PAIR:
            self.model_sdf.enable_fused_training()
            self.execution["sdf_training"] = "fused wgmma"
        params = list(self.model_sdf.parameters())
        if optimizer == "fused":
            from .optim import FusedAdamW
            self.optimizer = FusedAdamW([{"params": params, "weight_decay": 0.0, "lr": lr, "name": "model_sdf"}], betas=(0.9, 0.99),
                                        eps=1e-15, lr=lr)
            self.model_sdf.encoding.grad_in_place = True
        else:
            self.optimizer = torch.optim.AdamW(params, amsgrad=False, betas=(0.9, 0.99), eps=1e-15, weight_decay=0.0, lr=lr)
        why = None
        if direct is False:
            why = "disabled by the caller (direct=False)"
        elif not fused_training:
            why = "the SDF model is not on the fused training kernels (fused_training=False)"
        elif optimizer != "fused":
            why = "needs the flat-buffer optimizer (gradients accumulate into persistent .grad views)"
        if why is not None and direct:
            raise RuntimeError("%s(direct=True): %s" % (who, why))
        self._direct_why = why
        self.direct = why is None
        self.execution["step"] = "direct kernel sequence (surface_fit.py)" if self.direct else "torch.autograd (%s)" % why
        self.iter_nr = 0
        self.fixed_random = None        # tests: {"surface_fit_idx": [Ns] int64, "surface_fit_u01": [No,3]} replace the torch RNG draws
        self.last = {}
        self._ws = None                 # buffers of the direct sequence, sized by (Ns, No, P)
        self._dev = None                # device-resident iteration, step count and captured graph
        self._cg = None                 # CUDA-graph state (enable_cuda_graph)

    # ------------------------------------------------------------------------------------ draws
    def draw(self, name, fn):
        """random draw `name` of the iteration: fn() (torch RNG) unless a test pinned it in self.fixed_random"""
        fr = self.fixed_random
        return fr[name] if (fr is not None and name in fr) else fn()

    def _draws(self, Ns, No):
        """-> (cloud row indices [Ns], box draw [No,3]) in the reference's order"""
        dev = self.points.device
        idx = self.draw("surface_fit_idx", lambda: torch.randint(self.nr_points, (Ns,), device=dev))
        u01 = self.draw("surface_fit_u01", lambda: torch.rand(No, 3, device=dev))
        return idx, u01

    def _autograd_points(self, Ns, No):
        """the reference's points of one iteration from the same draws -> (points [Ns+No, POS_DIM], surface normals [Ns,3])"""
        with torch.no_grad():
            idx, u01 = self._draws(Ns, No)[:2]
            surface_points = torch.index_select(self.points, 0, idx)
            surface_normals = torch.index_select(self.normals, 0, idx)
            a = self.aabb
            dev = u01.device
            size = torch.as_tensor(a.bounding_box_sizes_xyz, device=dev)
            offsurface_points = u01 * size - size / 2 + torch.as_tensor(a.bounding_box_translation, device=dev)
            return torch.cat([surface_points, offsurface_points], 0), surface_normals

    # ------------------------------------------------------------------------------------ the iteration
    def step(self, nr_surface=3000, nr_offsurface=30000):
        """one iteration -> detached 0-d loss (no host sync); last['terms'] = the four unweighted means {eikonal, normal, sdf, off}"""
        return self.fit(1, nr_surface, nr_offsurface)

    def fit(self, nr_iters, nr_surface=3000, nr_offsurface=30000):
        """`nr_iters` iterations -> detached 0-d loss of the last one (None when nr_iters is 0). The iteration number drives the
        coarse-to-fine window of the SDF encoding (iter_nr, then iter_nr + 1, ...)."""
        Ns, No = _check_counts(nr_surface, nr_offsurface, self.POS_DIM, type(self).__name__)
        n = max(int(nr_iters), 0)
        self.model_sdf.train()
        loss = None
        if not self.direct:
            for _ in range(n):
                loss = self._step_autograd(Ns, No)
            return loss
        self.execution["step"] = "direct kernel sequence (surface_fit.py)" + (", CUDA-graph replay" if self._cg is not None else "")
        opt = self.optimizer
        dev = opt.flat_param.device
        st = self._dev
        if st is None:
            st = self._dev = dict(it_dev=torch.zeros((), device=dev), step_dev=torch.zeros(1, dtype=torch.int32, device=dev), graph=None,
                                  warm=None)
        # device-resident iteration and AdamW step count: the same sequence runs eagerly and from the captured graph
        st["it_dev"].fill_(float(self.iter_nr))
        st["step_dev"].fill_(opt.step_count)
        opt.sync_hyper()
        opt.zero_grad(set_to_none=False)          # gradients start clean; the AdamW sweep re-zeroes them
        fr = self.fixed_random or {}
        key = (Ns, No) + tuple(None if fr.get(k) is None else fr[k].data_ptr() for k in self.DRAWS)

        def one(dit):
            out = self._direct_forward_backward(dit, Ns, No)
            opt.step_groups_deferred([0], st["step_dev"])
            self.model_sdf.fused.repack(advance=(st["step_dev"], st["it_dev"]))
            return out

        with torch.cuda.device(dev):
            for _ in range(n):
                dit = DeviceIter(self.iter_nr, st["it_dev"])
                g = st["graph"]
                if self._cg is None:
                    loss = one(dit)
                elif g is not None and g["key"] == key and g["lo"] <= self.iter_nr < g["hi"]:
                    g["graph"].replay()
                    loss = g["loss"]
                elif st["warm"] != key:
                    # first iteration of this shape: eager, on the capture stream (workspaces and lazy library state are created there)
                    side, cur = self._cg["stream"], torch.cuda.current_stream()
                    side.wait_stream(cur)
                    with torch.cuda.stream(side):
                        loss = one(dit)
                    cur.wait_stream(side)
                    st["warm"] = key
                else:
                    torch.cuda.synchronize()
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=self._cg["stream"]):
                        loss = one(dit)
                    st["graph"] = dict(graph=graph, key=key, lo=dit.lo, hi=dit.hi, loss=loss, last=self.last)
                    self._cg["captures"] += 1
                    graph.replay()                    # the capture recorded the iteration, it did not run it
                opt.step_count += 1
                self.iter_nr += 1
        if st["graph"] is not None and self._cg is not None:
            self.last = st["graph"]["last"]
        opt._clean = True
        return loss

    def _workspace(self, Ns, No):
        dev = self.points.device
        key = (Ns, No, self.nr_points, str(dev))
        ws = self._ws
        if ws is None or ws["key"] != key:
            from ._lib import load_library
            N = Ns + No
            f = lambda *s: torch.empty(*s, device=dev)
            ws = self._ws = dict(key=key, x=f(N, self.POS_DIM), n=f(Ns, 3), sdf=f(N), grad=f(N, 3), g_sdf=f(N), g_grad=f(N, 3),
                                 acc=torch.zeros(5, device=dev), loss=torch.zeros(1, device=dev), terms=torch.zeros(4, device=dev),
                                 ws=torch.empty(int(load_library().psdf_sdf_fused_backward_multi_workspace_bytes(N, 0, 0)),
                                                dtype=torch.uint8, device=dev))
        return ws

    def _direct_forward_backward(self, it, Ns, No):
        """draws, points, forward, loss and backward of iteration `it` (int or DeviceIter); the parameter gradients are ACCUMULATED into
        the optimizer's .grad views. -> detached 0-d loss; last['terms']"""
        m_sdf, fs, enc = self.model_sdf, self.model_sdf.fused, self.model_sdf.encoding
        ws = self._workspace(Ns, No)
        N = Ns + No
        a = self.aabb
        with torch.no_grad():
            draws = [d.contiguous() for d in self._draws(Ns, No)]
            call(*self.POINTS_FN, self.nr_points, Ns, No, self.points, self.normals, *draws, a.bounding_box_sizes_xyz, a.bounding_box_translation,
                 ws["x"], ws["n"])
            if fs._versions != fs._cur_versions():
                fs.repack()
            m_sdf.last_iter_nr = int(it)
            win = m_sdf.window(it).view(-1).contiguous()
            sdf_args = (enc.nr_levels, enc.capacity, enc.lattice_values.detach(), enc.scale_factor, enc.shift_tensor(), win,
                        enc.concat_points_scaling, fs.hidden, fs.out_dim, fs.blob)
            call(*self.FORWARD_FN, N, enc.nr_levels, enc.capacity, ws["x"], enc.lattice_values.detach(), enc.scale_factor,
                 enc.shift_tensor(), win, enc.concat_points_scaling, fs.hidden, fs.out_dim, fs.blob, ws["sdf"], ws["grad"], None)
            call("psdf_surface_fit_loss", Ns, No, ws["sdf"], ws["grad"], ws["n"], *SDF_LOSS_WEIGHTS, LOSS_SCALE, ws["g_sdf"], ws["g_grad"],
                 ws["acc"], ws["loss"], ws["terms"])
            lin = fs.lin
            call(*self.BACKWARD_FN, *sdf_args, N, ws["x"], ws["g_sdf"], ws["g_grad"], None, 0, None, None, None, None,
                 0, None, None, None, None, enc.lattice_values.grad, ws["ws"],
                 lin[0].weight.grad, lin[1].weight.grad, lin[2].weight.grad, lin[3].weight.grad,
                 lin[0].bias.grad, lin[1].bias.grad, lin[2].bias.grad, lin[3].bias.grad)
        self.last = dict(terms=ws["terms"])
        return ws["loss"].view(())

    def _autograd_forward_backward(self, it, Ns, No):
        """the reference's loop body (train_sdf_from_mesh.py:119-161) with the same draws: sdf_loss / 30000 and loss.backward() (gradients
        accumulate into .grad) -> detached 0-d loss; last['terms']"""
        points, surface_normals = self._autograd_points(Ns, No)
        sdf, sdf_gradients, _ = self.model_sdf.get_sdf_and_gradient(points, it)
        if sdf_gradients.shape[1] != 3:
            sdf_gradients = sdf_gradients[:, 0:3]          # train_4d_sdf.py:213: the spatial part of the space-time gradient
        loss = sdf_loss(sdf[:Ns], sdf_gradients[:Ns], sdf[-No:], sdf_gradients[-No:], surface_normals) / 30000
        terms = sdf_loss.terms
        loss.backward()
        self.last = dict(terms=torch.stack([t.detach() for t in terms]))
        return loss.detach()

    def _step_autograd(self, Ns, No):
        opt = self.optimizer
        fused_opt = hasattr(opt, "flat_grad")
        opt.zero_grad(set_to_none=not fused_opt)
        loss = self._autograd_forward_backward(self.iter_nr, Ns, No)
        opt.step()
        if getattr(self.model_sdf, "fused", None) is not None:
            self.model_sdf.fused.repack()          # raw-pointer updates do not bump tensor versions
        self.iter_nr += 1
        return loss

    # ------------------------------------------------------------------------------------ CUDA-graph replay
    def enable_cuda_graph(self):
        """later steps of the direct sequence replay one captured CUDA graph per shape and stretch of the coarse-to-fine schedule: the
        first step of a shape runs eagerly, the next one is captured; one more capture follows where the window's ramp ends (iteration
        nr_iters_for_c2f). The autograd formulation is not captured."""
        if self._cg is None:
            self._cg = dict(stream=torch.cuda.Stream(device=self.points.device), captures=0)

    def disable_cuda_graph(self):
        self._cg = None
        if self._dev is not None:
            self._dev["graph"], self._dev["warm"] = None, None

    # ------------------------------------------------------------------------------------ checkpoints
    def save(self, ckpt_folder, experiment_name, iter_nr=None, with_optimizer=True):
        """<ckpt>/<experiment>/<iter>/models/sdf_model.pt, the reference's SDF.save layout and keys (train_sdf_from_mesh.py:168-169), and
        beside it surface_fit_state.pt (optimizer moments and step count, iter_nr) so that a run resumes bit for bit. -> models path"""
        it = self.iter_nr if iter_nr is None else iter_nr
        path = self.model_sdf.save(ckpt_folder, experiment_name, it)
        if with_optimizer:
            torch.save({"optimizer": self.optimizer.state_dict(), "iter_nr": self.iter_nr}, os.path.join(path, self.STATE_FILE))
        return path

    def load(self, ckpt_path_full, with_optimizer=True):
        """inverse of save(); a checkpoint of the reference (sdf_model.pt only) loads with iter_nr = 0 and the optimizer left as it is.
        Parameters are copied into the existing storages, so the flat-buffer optimizer's views stay valid."""
        dev = self.points.device
        self.model_sdf.load_state_dict(torch.load(os.path.join(ckpt_path_full, "sdf_model.pt"), map_location=dev))
        st = os.path.join(ckpt_path_full, self.STATE_FILE)
        if with_optimizer and os.path.exists(st):
            sd = torch.load(st, map_location=dev)
            self.optimizer.load_state_dict(sd["optimizer"])
            self.iter_nr = int(sd["iter_nr"])
        else:
            self.iter_nr = 0
        if getattr(self.model_sdf, "fused", None) is not None:
            self.model_sdf.fused.repack()


class SpaceTimeFit(SurfaceFit):
    """Fit a space-time SDF to a point sequence: the state and the loop of train_4d_sdf.py (SDF(4, AABB([1,1,1], [0,0,0]), 0, 3000) with the
    reference's 24 levels, 2^18 entries and 32-wide MLP, AdamW with betas (0.9, 0.99), eps 1e-15, no weight decay, lr 1e-3).

    points_time: [P,4] float32 (x, y, z, t) on the GPU, normals: [P,3]. Each `step()` draws `nr_surface` sequence rows, `nr_offsurface`
    uniform box points and their uniform times, in the reference's order (torch.randint, aabb.rand_points_inside, torch.rand((No, 1))).
    The loss is sdf_loss / 30000 of the spatial gradient d sdf / d (x, y, z), which is what the reference reads of the [N,4] gradient.
    Options as SurfaceFit; the direct sequence runs the pos_dim = 4 fused kernels, the fallback (direct=False, optimizer "adamw") the
    reference's loop on the per-op kernels (get_sdf_and_gradient [N,4] under autograd, then [:, :3]). Checkpoints: the reference's
    sdf_model.pt and spacetime_fit_state.pt."""
    POS_DIM = 4
    DRAWS = SurfaceFit.DRAWS + ("spacetime_fit_ut",)
    STATE_FILE = "spacetime_fit_state.pt"
    POINTS_FN, FORWARD_FN, BACKWARD_FN = ("psdf_spacetime_fit_points",), ("psdf_sdf_fused_forward_dim", 4), ("psdf_sdf_fused_backward_multi_dim", 4)
    MODEL_ON_FUSED_PAIR = False

    def __init__(self, points_time, normals, nr_levels=24, capacity=2 ** 18, hidden=32, box_size=(1, 1, 1), box_translation=(0, 0, 0),
                 nr_iters_for_c2f=3000, lr=1e-3, optimizer="fused", deterministic=False, direct=None, seed=0):
        super().__init__(points_time, normals, nr_levels, capacity, hidden, box_size, box_translation, nr_iters_for_c2f, lr, optimizer,
                         deterministic, direct, seed)
        # the model's own get_sdf_and_gradient stays on the per-op kernels (MODEL_ON_FUSED_PAIR); only the direct sequence is fused
        self.execution["sdf_training"] = "fused wgmma (direct sequence)" if self.direct else "per-op kernels + autograd"

    def _draws(self, Ns, No):
        """-> (sequence row indices [Ns], box draw [No,3], time draw [No,1]) in the reference's order (train_4d_sdf.py:202-206)"""
        idx, u01 = super()._draws(Ns, No)
        ut = self.draw("spacetime_fit_ut", lambda: torch.rand(No, 1, device=self.points.device))
        return idx, u01, ut

    def _autograd_points(self, Ns, No):
        with torch.no_grad():
            idx, u01, ut = self._draws(Ns, No)
            surface_points_time = torch.index_select(self.points, 0, idx)
            surface_normals = torch.index_select(self.normals, 0, idx)
            a = self.aabb
            dev = u01.device
            size = torch.as_tensor(a.bounding_box_sizes_xyz, device=dev)
            offsurface_points = u01 * size - size / 2 + torch.as_tensor(a.bounding_box_translation, device=dev)
            offsurface_points_time = torch.cat([offsurface_points, ut], 1)
            return torch.cat([surface_points_time, offsurface_points_time], 0), surface_normals

    def step(self, nr_surface=3000, nr_offsurface=3000):
        """one iteration -> detached 0-d loss (no host sync); last['terms'] = the four unweighted means {eikonal, normal, sdf, off}"""
        return self.fit(1, nr_surface, nr_offsurface)

    def fit(self, nr_iters, nr_surface=3000, nr_offsurface=3000):
        """`nr_iters` iterations -> detached 0-d loss of the last one (None when nr_iters is 0)"""
        return super().fit(nr_iters, nr_surface, nr_offsurface)
