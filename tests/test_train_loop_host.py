"""The reference's training-loop helpers on the CPU (utils.py:88-385, config.py:234-268, models/flags.py:17-31): signatures, learning-rate
schedules, EMAWarmup, every sigma sample density and ema_update's per-tensor path, against values recorded from the reference by
oracle/make_golden_train_loop.py."""
import inspect
import json
import warnings

import numpy as np
import pytest
import torch

from conftest import GOLDEN

import k_diffusion as K

META = json.loads((GOLDEN / "train_loop.json").read_text())


@pytest.fixture(scope="module")
def npz():
    with np.load(GOLDEN / "train_loop.npz") as z:
        return {k: z[k] for k in z.files}


def _resolve(dotted):
    obj = K
    for part in dotted.split("."):
        obj = getattr(obj, part)
    return obj


def test_signatures_equal_the_references():
    recorded = json.loads((GOLDEN / "train_loop_signatures.json").read_text())
    for name, want in recorded.items():
        got = [[n, p.kind.name, None if p.default is inspect._empty else repr(p.default)]
               for n, p in inspect.signature(_resolve(name)).parameters.items()]
        assert got == want, name


def _scheduler(case, lrs=None):
    name, kwargs, base = META["lr"][case]
    params = [torch.nn.Parameter(torch.zeros(1)) for _ in base]
    opt = torch.optim.SGD([{"params": [p], "lr": lr} for p, lr in zip(params, base)])
    return opt, getattr(K.utils, name)(opt, **kwargs)


@pytest.mark.parametrize("case", sorted(META["lr"]))
def test_lr_schedule_matches_the_reference_bit_for_bit(case, npz):
    opt, sched = _scheduler(case)
    seq, state = [], None
    for i in range(META["lr_steps"]):
        seq.append(sched.get_last_lr())
        opt.step()
        sched.step()
        if i + 1 == META["lr_resume_at"]:
            state = sched.state_dict()
    assert np.array_equal(np.array(seq, dtype=np.float64), npz[f"lr_{case}"])
    opt2, sched2 = _scheduler(case)
    sched2.load_state_dict(state)
    resumed = []
    for _ in range(META["lr_resume_at"], META["lr_steps"]):
        opt2.step()
        sched2.step()
        resumed.append(sched2.get_last_lr())
    assert np.array_equal(np.array(resumed, dtype=np.float64), npz[f"lr_{case}_resumed"])
    assert opt2.param_groups[0]["lr"] == resumed[-1][0]


def test_lr_schedules_reject_a_bad_warmup_and_warn_on_get_lr():
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1e-3)
    for make in (lambda w: K.utils.InverseLR(opt, warmup=w), lambda w: K.utils.ExponentialLR(opt, 10, warmup=w),
                 lambda w: K.utils.ConstantLRWithWarmup(opt, warmup=w)):
        for bad in (-0.1, 1.0):
            with pytest.raises(ValueError, match="Invalid value for warmup"):
                make(bad)
    sched = K.utils.InverseLR(opt, inv_gamma=10.)
    with pytest.warns(UserWarning, match="get_last_lr"):
        sched.get_lr()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        opt.step()
        sched.step()


@pytest.mark.parametrize("case", sorted(META["ema_warmup"]))
def test_ema_warmup_values_and_state(case, npz):
    kwargs, final_state = META["ema_warmup"][case]
    w = K.utils.EMAWarmup(**kwargs)
    vals = []
    for _ in range(META["ema_steps"]):
        vals.append(w.get_value())
        w.step()
    assert np.array_equal(np.array(vals, dtype=np.float64), npz[f"ema_warmup_{case}"])
    assert w.state_dict() == final_state
    w2 = K.utils.EMAWarmup()
    w2.load_state_dict(w.state_dict())
    assert w2.get_value() == w.get_value() and w2.state_dict() == final_state


def test_ema_warmup_clamps_and_holds_before_start_at():
    w = K.utils.EMAWarmup(inv_gamma=1., power=1., min_value=0.3, max_value=0.6, start_at=5)
    got = []
    for _ in range(12):
        got.append(w.get_value())
        w.step()
    assert got[:6] == [0.3] * 6                  # epoch 0 before and at start_at: 0, clamped up to min_value
    assert got[-1] == 0.6 and max(got) == 0.6    # 1 - 1 / (1 + 6) > 0.6: clamped down to max_value


def _density(case, i):
    cfg = META["densities"][case]
    strat = META["strats"][i]
    density = K.config.make_sample_density(cfg)
    torch.manual_seed(1000 + i)
    if strat is None:
        return density([META["n_samples"]], device="cpu")
    with K.utils.enable_stratified(*strat):
        return density([META["n_samples"]], device="cpu")


@pytest.mark.parametrize("case", sorted(META["densities"]))
def test_sample_density_matches_the_reference_bit_for_bit(case, npz):
    for i in range(len(META["strats"])):
        got = _density(case, i)
        want = npz[f"density_{case}_{i}"]
        assert got.dtype == torch.float32 and got.shape == want.shape
        assert np.array_equal(got.numpy(), want), (case, META["strats"][i])


def test_stratification_covers_every_stratum_once():
    groups, n = 4, 8
    u = torch.cat([K.utils.stratified_uniform([n], g, groups, dtype=torch.float64) for g in range(groups)])
    strata = torch.sort((u * n * groups).floor().long()).values
    assert torch.equal(strata, torch.arange(n * groups))
    with pytest.raises(ValueError):
        K.utils.stratified_uniform([2], 0, 0)
    with pytest.raises(ValueError):
        K.utils.stratified_uniform([2], 3, 3)


def test_enable_stratified_is_scoped_and_disable_gives_plain_uniforms():
    with K.utils.enable_stratified(2, 5):
        torch.manual_seed(0)
        a = K.utils.stratified_with_settings([6], dtype=torch.float64)
    with K.utils.enable_stratified(2, 5, disable=True):
        torch.manual_seed(0)
        b = K.utils.stratified_with_settings([6], dtype=torch.float64)
    torch.manual_seed(0)
    c = K.utils.stratified_with_settings([6], dtype=torch.float64)
    torch.manual_seed(0)
    assert torch.equal(a, K.utils.stratified_uniform([6], 2, 5, dtype=torch.float64))
    assert torch.equal(b, c) and not hasattr(K.utils.stratified_settings, "group")


def test_enable_stratified_accelerate_groups_by_process_and_accumulation_step():
    class Acc:
        process_index, num_processes, step = 1, 3, 7

        class gradient_state:
            num_steps = 2
    with K.utils.enable_stratified_accelerate(Acc()):
        s = K.utils.stratified_settings
        assert (s.group, s.groups, s.disable) == (1 * 2 + 7 % 2, 6, False)
    assert not hasattr(K.utils.stratified_settings, "group")


def test_unknown_density_raises_value_error():
    with pytest.raises(ValueError, match="Unknown sample density type"):
        K.config.make_sample_density({"sigma_data": 1., "sigma_sample_density": {"type": "gamma"}})


def test_checkpointing_flag_is_scoped():
    assert K.models.get_checkpointing() is False
    with K.models.checkpointing():
        assert K.models.get_checkpointing() is True
        with K.models.checkpointing(False):
            assert K.models.get_checkpointing() is False
        assert K.models.get_checkpointing() is True
    assert K.models.get_checkpointing() is False


class _Toy(torch.nn.Module):
    """oracle/make_golden_train_loop.py's module"""

    def __init__(self, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.a = torch.nn.Parameter(torch.randn(67, 5, generator=g))
        self.b = torch.nn.Parameter(torch.randn(1, generator=g))
        self.c = torch.nn.Parameter(torch.randn(3, generator=g) * 100)
        self.register_buffer("running", torch.randn(9, generator=g))
        self.register_buffer("count", torch.tensor(seed))


@pytest.mark.parametrize("decay", [0., 0.5, 0.999, 1.])
def test_ema_update_on_cpu_modules_is_the_references(decay, npz):
    model, ema = _Toy(1), _Toy(2)
    K.utils.ema_update(model, ema, decay)
    for k, v in ema.state_dict().items():
        assert np.array_equal(v.numpy(), npz[f"ema_update_{decay}_{k}"]), k
    assert all(p.grad is None for p in ema.parameters())


def test_ema_update_rejects_mismatched_keys():
    a, b = torch.nn.Linear(2, 2), torch.nn.Sequential(torch.nn.Linear(2, 2))
    with pytest.raises(AssertionError):
        K.utils.ema_update(a, b, 0.9)


def test_ema_update_dict():
    d = K.utils.ema_update_dict({}, {"loss": 2.0}, 0.9)
    assert d == {"loss": 2.0}
    K.utils.ema_update_dict(d, {"loss": 1.0, "x": 3.0}, 0.75)
    assert d == {"loss": 2.0 * 0.75 + 0.25 * 1.0, "x": 3.0}
