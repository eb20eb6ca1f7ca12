"""'What would this phase cost if it were free' timings of the lock-step value + tangent forward (k_sdf_fused<true>) at 65 536 samples:
PSDF_EXPERIMENT_KNOCKOUT bit 0 skips the encoder, bit 1 the MMAs, bit 2 the GELU arithmetic, bit 3 the operand-tile stores, bit 4 the accumulator loads, bit 5 the output stores (results are
garbage; diagnostics). usage, on the GPU: python tools/knockout_forward.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = r'''
import os, sys, numpy as np, torch
sys.path[:0] = [%r, %r, %r]
import scenes
from permuto_sdf import Sphere
from permuto_sdf_b200 import call
from permuto_sdf_b200.models import SDF
m = SDF(3, Sphere(0.5, [0, 0, 0]), 32, 10000, nr_levels=16, capacity=2 ** 18, hidden=64).to("cuda")
f = m.enable_fused_inference()
call("psdf_sdf_forward_variant", 0)
o, d = scenes.make_rays(512, seed=0, miss_fraction=0.0, axis_aligned=0)
z = np.linspace(0.75, 1.0, 128, dtype=np.float32)
pos = torch.from_numpy((o[:, None, :] + z[None, :, None] * d[:, None, :]).reshape(-1, 3).astype(np.float32)).cuda()
def t(fn, n=30):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n * 1e3
with torch.no_grad():
    print("%%.1f" %% t(lambda: f(pos, 20000, with_gradient=True)))
''' % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "compat"))
NAMES = {0: "everything", 1: "no encoder", 2: "no MMA", 4: "no GELU", 8: "no operand stores", 12: "no GELU, no stores",
         14: "no MMA, GELU, stores", 16: "no accumulator loads", 32: "no output stores", 15: "accumulator loads + barriers + outputs",
         63: "barriers only (sync skeleton)", 191: "skeleton, no fence.proxy.async", 128: "everything but fence.proxy.async (wrong results)"}
for k, name in NAMES.items():
    env = dict(os.environ, PSDF_EXPERIMENT_KNOCKOUT=str(k))
    out = subprocess.run([sys.executable, "-c", CODE], env=env, capture_output=True, text=True)
    print("knockout=%2d  %-36s %s us" % (k, name, out.stdout.strip().splitlines()[-1] if out.stdout.strip() else "ERR " + out.stderr[-300:]))
