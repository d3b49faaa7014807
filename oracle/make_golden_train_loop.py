#!/usr/bin/env python
"""Record the pieces of the reference's train.py step that live in its utils and config, from the REAL reference (run by hand, with
$K_DIFFUSION_REFERENCE naming a checkout; k_diffusion.utils and config import with make_golden.py's stubs, train.py's own imports are
not needed):

    python oracle/make_golden_train_loop.py   # -> tests/golden/train_loop_signatures.json, train_loop.npz, train_loop.json

All on the CPU: the signatures of every name, 200 steps of each learning-rate schedule (with a state_dict round trip), EMAWarmup values,
seeded draws of every sigma sample density through make_sample_density (stratification off and on), and ema_update on seeded modules.
The reference's schedulers pass `verbose` to torch's LRScheduler, which torch 2.11 no longer takes; the shim below drops it.
It also checks oracle/train_loop_oracle.py against the reference's densities, bit for bit."""
import inspect
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as G

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import train_loop_oracle as TO

SIGNATURES = ["utils.stratified_uniform", "utils.enable_stratified", "utils.enable_stratified_accelerate", "utils.stratified_with_settings",
              "utils.rand_log_normal", "utils.rand_log_logistic", "utils.rand_log_uniform", "utils.rand_v_diffusion",
              "utils.rand_cosine_interpolated", "utils.rand_split_log_normal", "utils.ema_update", "utils.ema_update_dict",
              "utils.EMAWarmup.__init__", "utils.EMAWarmup.state_dict", "utils.EMAWarmup.load_state_dict", "utils.EMAWarmup.get_value",
              "utils.EMAWarmup.step", "utils.InverseLR.__init__", "utils.ExponentialLR.__init__", "utils.ConstantLRWithWarmup.__init__",
              "utils.InverseLR.get_lr", "utils.InverseLR._get_closed_form_lr", "config.make_sample_density", "models.checkpointing",
              "models.get_checkpointing"]

# (class name, kwargs, base lrs of the param groups)
LR_CASES = {
    "inverse": ("InverseLR", dict(inv_gamma=20000., power=1.), [1e-4]),
    "inverse_warmup": ("InverseLR", dict(inv_gamma=50., power=0.75, warmup=0.99), [5e-4, 2e-4]),
    "inverse_min_lr": ("InverseLR", dict(inv_gamma=10., power=2., warmup=0.9, min_lr=3e-5), [1e-3]),
    "exponential": ("ExponentialLR", dict(num_steps=40, decay=0.3), [1e-3]),
    "exponential_warmup_min_lr": ("ExponentialLR", dict(num_steps=25., warmup=0.95, min_lr=1e-4), [1e-3, 4e-4]),
    "constant": ("ConstantLRWithWarmup", dict(), [2e-4]),
    "constant_warmup": ("ConstantLRWithWarmup", dict(warmup=0.99), [5e-4]),
}
LR_STEPS, LR_RESUME_AT = 200, 100

EMA_CASES = {
    "default": dict(),
    "train_py": dict(power=0.6667, max_value=0.9999),
    "start_at": dict(inv_gamma=10., power=0.75, min_value=0.2, max_value=0.99, start_at=30),
    "resumed": dict(power=2 / 3, last_epoch=1000, max_value=0.999),
}
EMA_STEPS = 300

# model configs after load_config (sigma_data, sigma_min, sigma_max, input_size) with a density each: every type and every key alias
BASE = dict(sigma_data=0.6, sigma_min=1e-2, sigma_max=80., input_size=[28, 28])
DENSITIES = {
    "lognormal_mean_std": dict(type="lognormal", mean=-1.2, std=1.2),
    "lognormal_loc_scale": dict(type="lognormal", loc=-0.5, scale=1.6),
    "loglogistic_default": dict(type="loglogistic"),
    "loglogistic_all": dict(type="loglogistic", loc=0.3, scale=0.7, min_value=1e-2, max_value=80.),
    "loguniform_default": dict(type="loguniform"),
    "loguniform_bounds": dict(type="loguniform", min_value=3e-3, max_value=160.),
    "v-diffusion_default": dict(type="v-diffusion"),
    "cosine_bounds": dict(type="cosine", min_value=1e-2, max_value=80.),
    "split-lognormal_mean_std": dict(type="split-lognormal", mean=-1.2, std_1=1.0, std_2=1.6),
    "split-lognormal_loc_scale": dict(type="split-lognormal", loc=-0.4, scale_1=0.8, scale_2=1.3),
    "cosine-interpolated_default": dict(type="cosine-interpolated"),
    "cosine-interpolated_all": dict(type="cosine-interpolated", min_value=2e-3, max_value=500., image_d=64, noise_d_low=16, noise_d_high=48),
}
STRATS = [None, (0, 1), (1, 4), (3, 4), (2, 7)]
N_SAMPLES = 37


def sig_of(fn):
    return [[name, p.kind.name, None if p.default is inspect._empty else repr(p.default)]
            for name, p in inspect.signature(fn).parameters.items()]


def resolve(K, dotted):
    obj = K
    for part in dotted.split("."):
        obj = getattr(obj, part)
    return obj


def density_configs(K):
    cases = {f"ref_{p.stem}": K.config.load_config(json.loads(p.read_text()))["model"] for p in sorted((G.REF / "configs").glob("*.json"))}
    cases.update({k: dict(BASE, sigma_sample_density=v) for k, v in DENSITIES.items()})
    return cases


def lr_sequences(K, name, kwargs, lrs):
    def make(last_epoch=-1, initial=None):
        params = [torch.nn.Parameter(torch.zeros(1)) for _ in lrs]
        opt = torch.optim.SGD([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)])
        if initial is not None:
            for g, lr in zip(opt.param_groups, initial):
                g["initial_lr"] = lr
        return opt, getattr(K.utils, name)(opt, **kwargs)

    opt, sched = make()
    seq, state = [], None
    for i in range(LR_STEPS):
        seq.append(sched.get_last_lr())
        opt.step()
        sched.step()
        if i + 1 == LR_RESUME_AT:
            state = sched.state_dict()
    opt2, sched2 = make()
    sched2.load_state_dict(state)
    resumed = []
    for _ in range(LR_RESUME_AT, LR_STEPS):
        opt2.step()
        sched2.step()
        resumed.append(sched2.get_last_lr())
    return np.array(seq, dtype=np.float64), np.array(resumed, dtype=np.float64)


class Toy(torch.nn.Module):
    """Parameters of several sizes and alignments, a float buffer and an integer buffer."""

    def __init__(self, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.a = torch.nn.Parameter(torch.randn(67, 5, generator=g))
        self.b = torch.nn.Parameter(torch.randn(1, generator=g))
        self.c = torch.nn.Parameter(torch.randn(3, generator=g) * 100)
        self.register_buffer("running", torch.randn(9, generator=g))
        self.register_buffer("count", torch.tensor(seed))


def main():
    G._stub_missing()
    from torch.optim import lr_scheduler
    lr_scheduler._LRScheduler.__init__ = lambda self, optimizer, last_epoch=-1, verbose=False: \
        lr_scheduler.LRScheduler.__init__(self, optimizer, last_epoch)
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K

    sigs = {name: sig_of(resolve(K, name)) for name in SIGNATURES}
    (G.OUT / "train_loop_signatures.json").write_text(json.dumps(sigs, indent=1))

    arrays, meta = {}, {"lr": {}, "ema_warmup": {}, "densities": {}, "strats": STRATS, "n_samples": N_SAMPLES, "lr_steps": LR_STEPS,
                        "lr_resume_at": LR_RESUME_AT, "ema_steps": EMA_STEPS}
    for case, (name, kwargs, lrs) in LR_CASES.items():
        arrays[f"lr_{case}"], arrays[f"lr_{case}_resumed"] = lr_sequences(K, name, kwargs, lrs)
        meta["lr"][case] = [name, kwargs, lrs]
    for case, kwargs in EMA_CASES.items():
        w = K.utils.EMAWarmup(**kwargs)
        vals = []
        for _ in range(EMA_STEPS):
            vals.append(w.get_value())
            w.step()
        arrays[f"ema_warmup_{case}"] = np.array(vals, dtype=np.float64)
        meta["ema_warmup"][case] = [kwargs, w.state_dict()]
    for case, cfg in density_configs(K).items():
        meta["densities"][case] = {k: cfg[k] for k in ("sigma_data", "sigma_min", "sigma_max", "input_size", "sigma_sample_density")}
        density = K.config.make_sample_density(cfg)
        for i, strat in enumerate(STRATS):
            torch.manual_seed(1000 + i)
            if strat is None:
                got = density([N_SAMPLES], device="cpu")
            else:
                with K.utils.enable_stratified(*strat):
                    got = density([N_SAMPLES], device="cpu")
            torch.manual_seed(1000 + i)
            want = TO.sample_density(cfg, [N_SAMPLES], "cpu", strat)
            assert got.dtype == want.dtype and torch.equal(got, want), (case, strat)
            arrays[f"density_{case}_{i}"] = got.numpy()
    for decay in (0., 0.5, 0.999, 1.):
        model, ema = Toy(1), Toy(2)
        K.utils.ema_update(model, ema, decay)
        for k, v in ema.state_dict().items():
            arrays[f"ema_update_{decay}_{k}"] = v.numpy()
    np.savez(G.OUT / "train_loop.npz", **arrays)
    (G.OUT / "train_loop.json").write_text(json.dumps(meta, indent=1))
    print("wrote", G.OUT / "train_loop_signatures.json", G.OUT / "train_loop.npz", len(arrays), "arrays")


if __name__ == "__main__":
    main()
