"""Fused dense AdamW over flat parameter / gradient buffers (csrc/optim.cu).

The reference uses torch.optim.AdamW or apex FusedAdam with betas (0.9, 0.99), eps 1e-15, per-group weight decay
(train_permuto_sdf.py:293-304). Here every parameter of every group is re-homed into ONE flat fp32 buffer (and its
gradient into one flat gradient buffer, so autograd accumulates straight into it): a step is one streaming kernel
per group (28 B/param, gradient zeroing folded in), and data-parallel training needs a single all-reduce of
`flat_grad`. `param_groups` keeps the torch layout (lr / weight_decay / name can be edited by schedulers: in CUDA-graph mode
the kernel reads both from a small device array that `sync_hyper()` refreshes before every replay, so an edit takes effect
without re-capturing).

Gradient semantics: the step kernel leaves `flat_grad` zeroed; `zero_grad()` really zeroes whenever a backward may have run
without a following step (same behaviour as torch.optim.AdamW + zero_grad in the reference loop)."""
import torch

from ._lib import call


class FusedAdamW:
    def __init__(self, groups, betas=(0.9, 0.99), eps=1e-15, lr=1e-3, weight_decay=0.0):
        self.betas, self.eps = betas, eps
        self.param_groups = []
        total = 0
        layout = []
        for g in groups:
            ps = [p for p in g["params"] if p.requires_grad]
            n = sum(p.numel() for p in ps)
            n_pad = (n + 3) // 4 * 4                     # keep every group 16-byte aligned
            layout.append((ps, total, n, n_pad))
            total += n_pad
        dev = layout[0][0][0].device
        self.flat_param = torch.zeros(total, device=dev)
        self.flat_grad = torch.zeros(total, device=dev)
        self.exp_avg = torch.zeros(total, device=dev)
        self.exp_avg_sq = torch.zeros(total, device=dev)
        self.step_count = 0
        self.device_step = False        # True: the step count is kept in self.step_dev (device) for CUDA-graph replay
        self.step_dev = None
        self._clean = True              # flat_grad is known to be all zero (fresh, or just swept by the step kernel)
        self.hyper_dev = None           # [groups, 2] device copy of (lr, weight_decay), read by the kernel in device_step mode
        self._peer = None               # data-parallel peer-memory step (enable_peer_step)
        self._hyper_host = None
        self._hyper_cached = None
        for g, (ps, off, n, n_pad) in zip(groups, layout):
            o = off
            for p in ps:
                k = p.numel()
                self.flat_param[o:o + k].copy_(p.data.reshape(-1))
                p.data = self.flat_param[o:o + k].view_as(p)
                p.grad = self.flat_grad[o:o + k].view_as(p)
                o += k
            self.param_groups.append({"params": ps, "lr": g.get("lr", lr), "weight_decay": g.get("weight_decay", weight_decay),
                                      "name": g.get("name", ""), "_off": off, "_n": n_pad})

    # ------------------------------------------------------------------------------------ data parallel over NVLink peer memory
    def enable_peer_step(self, group=None):
        """Data-parallel step WITHOUT an all-reduce: parameters and gradients move into symmetric (peer-mapped) memory
        (torch.distributed._symmetric_memory), every rank owns 1/world of each parameter group and one kernel per group
        (psdf_adamw_dp_step, csrc/optim.cu) sums that shard of all ranks' gradients through NVLink peer loads, applies AdamW and
        stores the new parameters into all ranks' buffers. Optimizer state is sharded (only the owner's moments are current;
        state_dict() gathers them). Two device-side barriers bracket the kernels."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        grp = group if group is not None else dist.group.WORLD
        world, rank = dist.get_world_size(grp), dist.get_rank(grp)
        if world > 8:
            raise RuntimeError("peer step supports up to 8 ranks of one NVLink domain")
        dev = self.flat_param.device
        total = self.flat_param.numel()
        new_p = symm.empty(total, dtype=torch.float32, device=dev)
        new_g = symm.empty(total, dtype=torch.float32, device=dev)
        new_p.copy_(self.flat_param)
        new_g.copy_(self.flat_grad)
        hp, hg = symm.rendezvous(new_p, grp), symm.rendezvous(new_g, grp)
        for g in self.param_groups:
            o = g["_off"]
            for p in g["params"]:
                k = p.numel()
                p.data = new_p[o:o + k].view_as(p)
                p.grad = new_g[o:o + k].view_as(p)
                o += k
        self.flat_param, self.flat_grad = new_p, new_g
        shards, gptrs, pptrs = [], [], []
        for g in self.param_groups:
            n4 = g["_n"] // 4
            base, rem = divmod(n4, world)
            lo4 = rank * base + min(rank, rem)
            cnt4 = base + (1 if rank < rem else 0)
            shards.append((lo4 * 4, cnt4 * 4))
            gptrs.append(torch.tensor([int(hg.buffer_ptrs[r]) + 4 * g["_off"] for r in range(world)], dtype=torch.int64))
            pptrs.append(torch.tensor([int(hp.buffer_ptrs[r]) + 4 * g["_off"] for r in range(world)], dtype=torch.int64))
        import os
        # NVSwitch multicast (in-switch reduction + replication) cuts the per-rank NVLink bytes from (W-1)/W to 1/W of the buffers: pays
        # from 4 ranks on; at 2 ranks the unicast kernel is expected to be faster (compare with tools/dp_step_timing.py)
        want = os.environ.get("PSDF_DP_MULTICAST", "auto")
        mc = (want == "1" or (want == "auto" and world >= 4)) and bool(getattr(hp, "has_multicast_support", False)) and \
            int(hp.multicast_ptr) != 0 and int(hg.multicast_ptr) != 0
        self._peer = dict(world=world, rank=rank, hp=hp, hg=hg, shards=shards, gptrs=gptrs, pptrs=pptrs, group=grp,
                          mc_grad=int(hg.multicast_ptr) if mc else 0, mc_param=int(hp.multicast_ptr) if mc else 0, multicast=mc)
        torch.cuda.synchronize()
        dist.barrier(group=grp)

    def _peer_step(self, grad_scale, advance):
        pe = self._peer
        if advance:
            self.step_count += 1
        b1, b2 = self.betas
        step_dev = None
        if self.device_step:
            if self.step_dev is None:
                self.step_dev = torch.full((1,), self.step_count - 1, dtype=torch.int32, device=self.flat_param.device)
            if advance:
                self.step_dev.add_(1)
            step_dev = self.step_dev
            if self.hyper_dev is None:
                self.sync_hyper()
        pe["hg"].barrier(channel=0)                  # every rank's backward has finished: all gradient buffers are final
        for gi, g in enumerate(self.param_groups):
            off, n = g["_off"], g["_n"]
            lo, cnt = pe["shards"][gi]
            if cnt == 0:
                continue
            hyper = self.hyper_dev[gi] if self.device_step else None
            call("psdf_adamw_dp_step", cnt, lo, pe["world"], pe["rank"], pe["gptrs"][gi].data_ptr(), pe["pptrs"][gi].data_ptr(),
                 pe["mc_grad"] + 4 * off if pe["multicast"] else 0, pe["mc_param"] + 4 * off if pe["multicast"] else 0,
                 self.exp_avg[off:off + n], self.exp_avg_sq[off:off + n], float(g["lr"]), b1, b2, self.eps, float(g["weight_decay"]),
                 self.step_count, step_dev, hyper, float(grad_scale))
        pe["hp"].barrier(channel=0)                  # every owner has written its shard into every rank's parameters
        self.flat_grad.zero_()                       # ... and has read this rank's gradients
        self._clean = True

    def zero_grad(self, set_to_none=False):
        # the step kernel zeroes the gradients it consumed; a backward that was not followed by a step leaves them dirty
        if not self._clean:
            self.flat_grad.zero_()
        self._clean = False             # the caller is about to run a backward

    def check_aliasing(self):
        """parameters must still be views into flat_param (a later model.to() / .cuda() re-homes p.data and breaks the step)"""
        for g in self.param_groups:
            o = g["_off"]
            for p in g["params"]:
                if p.data_ptr() != self.flat_param.data_ptr() + 4 * o or p.grad is None or p.grad.data_ptr() != self.flat_grad.data_ptr() + 4 * o:
                    raise RuntimeError("FusedAdamW: parameter storage was re-assigned after the optimizer was built "
                                       "(model.to()/cuda() after construction?); rebuild the optimizer")
                o += p.numel()

    def sync_hyper(self):
        """device copy of (lr, weight_decay) per group; call outside graph capture, before every replay (cheap: host compare,
        one 8 B x groups copy only when a scheduler changed something)"""
        cur = tuple((float(g["lr"]), float(g["weight_decay"])) for g in self.param_groups)
        if self.hyper_dev is None:
            self.hyper_dev = torch.zeros(len(cur), 2, device=self.flat_param.device)
            self._hyper_host = torch.zeros(len(cur), 2).pin_memory() if torch.cuda.is_available() else torch.zeros(len(cur), 2)
        if cur != self._hyper_cached:
            self._hyper_host.copy_(torch.tensor(cur, dtype=torch.float32).view(-1, 2))
            self.hyper_dev.copy_(self._hyper_host, non_blocking=True)
            self._hyper_cached = cur

    def _multi_tables(self):
        """host tables of device addresses for psdf_adamw_multi_step (all groups in one launch)"""
        import ctypes
        gs = [g for g in self.param_groups if g["_n"] > 0]
        k = len(gs)
        n = (ctypes.c_longlong * k)(*[g["_n"] for g in gs])
        tab = lambda base: (ctypes.c_uint64 * k)(*[base.data_ptr() + 4 * g["_off"] for g in gs])
        idx = [self.param_groups.index(g) for g in gs]
        hyper = (ctypes.c_uint64 * k)(*[self.hyper_dev.data_ptr() + 8 * i for i in idx])
        key = (self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.hyper_dev.data_ptr())
        return dict(key=key, k=k, n=n, p=tab(self.flat_param), g=tab(self.flat_grad), m=tab(self.exp_avg), v=tab(self.exp_avg_sq), h=hyper)

    @torch.no_grad()
    def step(self, grad_scale=1.0, groups=None, advance=True, defer_counter=False, leave_room=False):
        """groups: indices of the param groups to sweep (None: all). advance=False: a second call of the same optimizer step (the
        data-parallel path steps the colour hash table while the other gradients are still being all-reduced).
        defer_counter=True (device-resident step count, all groups): ONE launch sweeps every group with step = step_dev + 1 and the
        counter itself is advanced by the caller's psdf_sdf_mlp_pack_advance (Trainer: the re-pack that closes the iteration).
        leave_room: few resident blocks, so that kernels of another stream can run beside the sweep (see csrc/iter_glue.cu)."""
        if self._peer is not None:
            return self._peer_step(grad_scale, advance)
        if advance:
            self.step_count += 1
        b1, b2 = self.betas
        if defer_counter and self.device_step and groups is None and advance and len(self.param_groups) <= 8:
            import ctypes
            if self.step_dev is None:
                self.step_dev = torch.full((1,), self.step_count - 1, dtype=torch.int32, device=self.flat_param.device)
            if self.hyper_dev is None:
                self.sync_hyper()
            mt = getattr(self, "_multi", None)
            if mt is None or mt["key"] != (self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.hyper_dev.data_ptr()):
                mt = self._multi = self._multi_tables()
            call("psdf_adamw_multi_step", mt["k"], ctypes.addressof(mt["n"]), ctypes.addressof(mt["p"]), ctypes.addressof(mt["g"]),
                 ctypes.addressof(mt["m"]), ctypes.addressof(mt["v"]), ctypes.addressof(mt["h"]), b1, b2, self.eps, self.step_dev, 1,
                 float(grad_scale), 1 if leave_room else 0)
            self._clean = True
            return True
        step_dev = None
        if self.device_step:            # CUDA-graph mode: the step counter lives (and is incremented) on the device
            if self.step_dev is None:
                self.step_dev = torch.full((1,), self.step_count - 1, dtype=torch.int32, device=self.flat_param.device)
            if advance:
                self.step_dev.add_(1)
            step_dev = self.step_dev
            if self.hyper_dev is None:
                self.sync_hyper()
        for gi, g in enumerate(self.param_groups):
            off, n = g["_off"], g["_n"]
            if n == 0 or (groups is not None and gi not in groups):
                continue
            hyper = self.hyper_dev[gi] if self.device_step else None
            call("psdf_adamw_step", n, self.flat_param[off:off + n], self.flat_grad[off:off + n], self.exp_avg[off:off + n],
                 self.exp_avg_sq[off:off + n], float(g["lr"]), b1, b2, self.eps, float(g["weight_decay"]), self.step_count, step_dev,
                 hyper, float(grad_scale), 1)
        self._clean = True

    def _gather_peer_state(self):
        """sharded moments -> full (every rank): zero what this rank does not own, sum over the ranks"""
        import torch.distributed as dist
        pe = self._peer
        for t in (self.exp_avg, self.exp_avg_sq):
            keep = torch.zeros_like(t)
            for g, (lo, cnt) in zip(self.param_groups, pe["shards"]):
                a = g["_off"] + lo
                keep[a:a + cnt] = t[a:a + cnt]
            dist.all_reduce(keep, group=pe["group"])
            t.copy_(keep)

    def state_dict(self):
        if self._peer is not None:
            self._gather_peer_state()
        return {"step": self.step_count, "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq,
                "groups": [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]}

    def load_state_dict(self, sd):
        """inverse of state_dict (moments, step count, per-group lr / weight_decay)"""
        if sd["exp_avg"].numel() != self.exp_avg.numel():
            raise RuntimeError("FusedAdamW.load_state_dict: flat size mismatch")
        self.exp_avg.copy_(sd["exp_avg"].to(self.exp_avg.device))
        self.exp_avg_sq.copy_(sd["exp_avg_sq"].to(self.exp_avg.device))
        self.step_count = int(sd["step"])
        if self.step_dev is not None:
            self.step_dev.fill_(self.step_count)
        for g, sg in zip(self.param_groups, sd["groups"]):
            g["lr"], g["weight_decay"] = sg["lr"], sg["weight_decay"]
        self._hyper_cached = None
