"""Host logic of the sphere-fit phase: the fit count in the trainer state (save / load), how many fit iterations a call runs, and the
refusal under data-parallel training. Trainers are built without models (no device needed); only the methods under test run."""
import pytest
import torch

from permuto_sdf_b200.train import HyperParams, Trainer


class _Opt:
    def __init__(self):
        self.sd = {"step": 0}

    def state_dict(self):
        return dict(self.sd)

    def load_state_dict(self, sd):
        self.sd = dict(sd)


def _bare(fit_iter=0, iter_nr=0):
    tr = Trainer.__new__(Trainer)
    tr.hp = HyperParams()
    tr.optimizer = _Opt()
    tr.iter_nr, tr.sphere_fit_iter, tr.nr_rays_to_create = iter_nr, fit_iter, 512
    tr._dp = None
    return tr


def test_trainer_state_round_trips_the_fit_count(tmp_path):
    a = _bare(fit_iter=1234, iter_nr=0)
    a.optimizer.sd = {"step": 1234}
    torch.save(a._trainer_state(), tmp_path / "trainer_state.pt")
    b = _bare()
    b._restore_trainer_state(torch.load(tmp_path / "trainer_state.pt"))
    assert b.sphere_fit_iter == 1234 and b.iter_nr == 0 and b.optimizer.sd == {"step": 1234}


def test_state_without_fit_count_loads_as_finished(tmp_path):
    old = {"optimizer": {"step": 7}, "iter_nr": 20000, "nr_rays_to_create": 640}      # written before the fit count was recorded
    torch.save(old, tmp_path / "trainer_state.pt")
    b = _bare()
    b._restore_trainer_state(torch.load(tmp_path / "trainer_state.pt"))
    assert b.sphere_fit_iter == b.hp.nr_iter_sphere_fit and b.iter_nr == 20000 and b.nr_rays_to_create == 640
    c = _bare()                           # reference checkpoint: models only, no trainer state
    c._restore_trainer_state(None)
    assert c.sphere_fit_iter == c.hp.nr_iter_sphere_fit and c.iter_nr == 0


def test_fit_sphere_refuses_data_parallel():
    tr = _bare()
    tr._dp = dict(world=2)
    with pytest.raises(RuntimeError, match="one GPU"):
        tr.fit_sphere(1)


class _Model:
    def train(self):
        pass


@pytest.mark.parametrize("done, asked, runs", [(0, None, 4000), (0, 5, 5), (3998, 5, 2), (4000, None, 0), (4000, 3, 0), (10, 0, 0)])
def test_fit_sphere_runs_the_rest_of_the_phase(done, asked, runs):
    tr = _bare(fit_iter=done)
    tr.model_sdf = _Model()
    tr.optimizer.param_groups = [{"name": "model_sdf", "lr": 0.5}, {"name": "model_rgb_only_encoding", "lr": 0.5}]
    tr._direct, tr._direct_why, tr.execution = None, "test", {}
    calls = []

    def fake(gi, n, r, c):
        assert gi == [0] and (n, r, c) == (30000, 0.3, [0.0, 0.0, 0.0])
        calls.append(tr.sphere_fit_iter)
        tr.sphere_fit_iter += 1
        return torch.tensor(float(len(calls)))
    tr._fit_sphere_autograd = fake
    out = tr.fit_sphere(asked)
    assert calls == list(range(done, done + runs))
    assert (out is None) == (runs == 0) and tr.sphere_fit_iter == done + runs
    assert all(g["lr"] == tr.hp.lr for g in tr.optimizer.param_groups)
    assert tr.execution["sphere_fit"].startswith("torch.autograd")
