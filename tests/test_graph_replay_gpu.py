"""The replay policy of the direct training loops (graphs.run) when the shape alternates: SurfaceFit and Trainer.fit_sphere under
graph replay with shapes A, A, B, A, B, A give the bits of the eager run, and every captured graph holds the workspaces it writes, also
after a run of another shape has replaced the loop's own workspaces."""
import pytest
import torch

from test_sphere_fit_gpu import _fresh_rngs, _trainer, _u01
from test_surface_fit_gpu import draws, sphere_cloud

pytestmark = pytest.mark.gpu

SEQUENCE = "AABABA"


@pytest.fixture(autouse=True)
def _reduction_mode_off_after(cuda):
    """deterministic=True switches the device's mode on; later tests start from the default"""
    yield
    from permuto_sdf_b200 import call
    call("psdf_set_deterministic", 0, 0, 0)


def _check_entry(slot):
    """the captured graph's entry holds the workspace of its own shape, and its loss is that workspace's loss buffer"""
    e = slot["graph"]
    if e is not None:
        assert e["keep"]["key"][0] == e["key"][0], (e["keep"]["key"], e["key"])
        assert e["out"][0].data_ptr() == e["keep"]["loss"].data_ptr()


def _surface_fit(graph):
    from permuto_sdf_b200 import SurfaceFit
    P = 20000
    pts, nrm = sphere_cloud(P)
    f = SurfaceFit(pts, nrm, nr_levels=16, capacity=2 ** 14, nr_iters_for_c2f=100, deterministic=True, seed=9)
    shapes = {"A": (1000, 5000), "B": (600, 3000)}
    fixed = {k: draws(P, Ns, No, seed=5 + i) for i, (k, (Ns, No)) in enumerate(shapes.items())}
    if graph:
        f.enable_cuda_graph()
    losses = []
    for s in SEQUENCE:
        f.fixed_random = fixed[s]
        losses.append(float(f.fit(1, *shapes[s])))
        if graph:
            _check_entry(f._cg["step"])
    captures = f._cg["captures"] if graph else 0
    out = (f.optimizer.flat_param.clone(), f.optimizer.exp_avg_sq.clone(), losses, captures)
    f.disable_cuda_graph()
    return out


def test_surface_fit_replay_with_alternating_shapes_equals_eager(cuda):
    pe, me, le, _ = _surface_fit(False)
    pg, mg, lg, captures = _surface_fit(True)
    assert captures == 2, captures          # A at its second run, B at its second run
    assert le == lg, (le, lg)
    assert torch.equal(pe, pg) and torch.equal(me, mg)


def _sphere_fit(graph):
    _fresh_rngs()
    tr = _trainer(deterministic=True)
    counts = {"A": 30000, "B": 20000}
    u01 = {k: _u01(n, seed=7 + i) for i, (k, n) in enumerate(counts.items())}
    if graph:
        tr.enable_cuda_graph()
    losses = []
    for s in SEQUENCE:
        tr.fixed_random = {"sphere_fit_u01": u01[s]}
        losses.append(float(tr.fit_sphere(1, nr_points=counts[s])))
        if graph:
            _check_entry(tr._fit)
    captures = tr._cg["captures"] if graph else 0
    out = (tr.optimizer.flat_param.clone(), tr.optimizer.exp_avg_sq.clone(), losses, captures)
    if graph:
        tr.disable_cuda_graph()
    _fresh_rngs()
    return out


def test_sphere_fit_replay_with_alternating_point_counts_equals_eager(cuda):
    pe, me, le, _ = _sphere_fit(False)
    pg, mg, lg, captures = _sphere_fit(True)
    assert captures == 2, captures
    assert le == lg, (le, lg)
    assert torch.equal(pe, pg) and torch.equal(me, mg)
