"""A/B timing of the value + tangent SDF forward variants (lock-step 128-sample tiles vs two 64-sample groups per CTA) on the GPU.
usage (under gpurun): python tools/ab_forward.py   -> prints us per launch for N = 8192, 65536, 1048576 samples along rays"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "compat")]
import scenes  # noqa: E402


def main():
    from permuto_sdf import Sphere
    from permuto_sdf_b200 import call
    from permuto_sdf_b200.models import SDF
    torch.manual_seed(0)
    m = SDF(3, Sphere(0.5, [0, 0, 0]), 32, 10000, nr_levels=16, capacity=2 ** 18, hidden=64).to("cuda")
    f = m.enable_fused_inference()

    def t(fn, n=30):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / n * 1e3
    for R, S in ((64, 128), (512, 128), (8192, 128)):
        o, d = scenes.make_rays(R, seed=0, miss_fraction=0.0, axis_aligned=0)
        z = np.linspace(0.75, 1.0, S, dtype=np.float32)
        pos = torch.from_numpy((o[:, None, :] + z[None, :, None] * d[:, None, :]).reshape(-1, 3).astype(np.float32)).cuda()
        out = []
        for variant in (0, 1):
            call("psdf_sdf_forward_variant", variant)
            with torch.no_grad():
                out.append(t(lambda: f(pos, 20000, with_gradient=True)))
        call("psdf_sdf_forward_variant", 1)
        print("N=%8d  lock-step %.1f us   dual-group %.1f us   ratio %.2f" % (pos.shape[0], out[0], out[1], out[0] / out[1]))


if __name__ == "__main__":
    main()
