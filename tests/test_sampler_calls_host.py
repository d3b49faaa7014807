"""Call trace of the fixed-schedule samplers, CPU only: with the native primitives replaced by the torch one-liners of
test_host_fuzz.py, every solver-kernel call (its float32 scalars, how many tensors it reads, whether `noise` / `old` is None), every
noise-sampler call (arguments and their Python types), every global-RNG draw, every callback payload, what is handed to the graph
runner and the bits of the result are compared with tests/golden/sampler_calls.json.  The golden was recorded from the hand-written
Euler / Euler-ancestral / Heun / DPM++(2M) loops before those samplers moved onto the op-plan executor: a change of launch order,
of a scalar a kernel receives, of the noise-sampler calling convention or of the graph-capture decision shows up here."""
import inspect
import json

import numpy as np
import torch

import k_diffusion as K
from conftest import GOLDEN, bits
from test_host_fuzz import _stub, toy2

S = K.sampling
GOLDEN_FILE = GOLDEN / "sampler_calls.json"
_LOGGED = ("euler_step", "heun_correct", "dpmpp_2m_step", "lincomb", "noise_brownian")


def _value(v):
    if isinstance(v, torch.Tensor):
        return "tensor"
    if v is None or isinstance(v, (bool, int, str)):
        return v
    if isinstance(v, (list, tuple)):
        return [_value(e) for e in v]
    return float(np.float32(v))                  # the kernels take float32 scalars


def _install(monkeypatch, log):
    """Stubbed primitives that append what they were called with to `log`."""
    from k_diffusion import _native
    _stub(monkeypatch)
    g = torch.Generator().manual_seed(7)
    monkeypatch.setattr(_native, "noise_brownian", lambda like, seeds, t_min, t_max, t0, t1, depth=24, out=None:
                        torch.randn(like.shape, generator=g))
    for name in _LOGGED:
        fn = getattr(_native, name)
        sig = inspect.signature(fn)

        def logged(*a, _fn=fn, _sig=sig, _name=name, **kw):
            b = _sig.bind(*a, **kw)
            b.apply_defaults()
            log.append([_name, {k: _value(v) for k, v in b.arguments.items() if k != "out"}])
            return _fn(*a, **kw)
        monkeypatch.setattr(_native, name, logged)

    def randn_like(t, *a, **kw):
        log.append(["randn_like", list(t.shape)])
        return torch.randn(t.shape, generator=g)
    monkeypatch.setattr(torch, "randn_like", randn_like)

    def args_of(a):
        return [[type(v).__name__, str(v.dtype) if isinstance(v, torch.Tensor) else None, float(v)] for v in a]

    brownian_call = S.BrownianTreeNoiseSampler.__call__

    def brownian(self, *a):
        log.append(["noise_sampler", "brownian", args_of(a)])
        return brownian_call(self, *a)
    monkeypatch.setattr(S.BrownianTreeNoiseSampler, "__call__", brownian)
    default = S.default_noise_sampler

    def default_noise_sampler(x):
        inner = default(x)
        return lambda *a: log.append(["noise_sampler", "default", args_of(a)]) or inner(*a)
    monkeypatch.setattr(S, "default_noise_sampler", default_noise_sampler)
    run = S._run

    def run_logged(name, body, ev, x, sig, params, callback, noise_sampler=None):
        marker = "global_rng" if noise_sampler is S._GLOBAL_RNG else S._noise_kind(noise_sampler)
        log.append(["run", name, repr(params), marker, callback is not None])
        return run(name, body, ev, x, sig, params, callback, noise_sampler)
    monkeypatch.setattr(S, "_run", run_logged)

    def foreign():
        return lambda *a: log.append(["noise_sampler", "foreign", args_of(a)]) or torch.randn([2, 1, 4, 4], generator=g)

    def callback(d):
        log.append(["callback", d["i"], float(d["sigma"]), float(d["sigma_hat"]), sorted(d)])
    return foreign, callback


def _cases(foreign):
    sig = S.get_sigmas_karras(5, 0.05, 40.)
    nz = sig[:-1]                                # no trailing zero
    window = dict(s_churn=3., s_tmin=0.1, s_tmax=30., s_noise=1.1)
    cases = {}
    for tag, s in (("zero", sig), ("nozero", nz)):
        cases[f"euler_{tag}"] = lambda s=s: (S.sample_euler, s, {})
        cases[f"heun_{tag}"] = lambda s=s: (S.sample_heun, s, {})
        cases[f"dpmpp_2m_{tag}"] = lambda s=s: (S.sample_dpmpp_2m, s, {})
        cases[f"euler_a_foreign_{tag}"] = lambda s=s: (S.sample_euler_ancestral, s, dict(noise_sampler=foreign()))
    cases.update({
        "euler_churn": lambda: (S.sample_euler, sig, dict(s_churn=20., s_noise=0.9)),
        "euler_churn_window": lambda: (S.sample_euler, sig, window),
        "heun_churn": lambda: (S.sample_heun, sig, dict(s_churn=20.)),
        "heun_churn_window": lambda: (S.sample_heun, sig, window),
        "euler_a_default": lambda: (S.sample_euler_ancestral, sig, dict(eta=0.5, s_noise=0.9)),
        "euler_a_eta0": lambda: (S.sample_euler_ancestral, sig, dict(eta=0., noise_sampler=foreign())),
        "euler_a_brownian": lambda: (S.sample_euler_ancestral, sig, dict(noise_sampler=S.BrownianTreeNoiseSampler(
            torch.zeros(2, 1, 4, 4), 0.05, 40., seed=[11, 12]))),
        "dpm_2_churn_window": lambda: (S.sample_dpm_2, sig, window),
        "dpm_2_ancestral_foreign": lambda: (S.sample_dpm_2_ancestral, sig, dict(noise_sampler=foreign())),
        "dpmpp_2m_sde_brownian": lambda: (S.sample_dpmpp_2m_sde, sig, {}),
    })
    return cases


def trace_samplers(monkeypatch):
    """{case: [call, ...]} of every case, each ending with the bits of the sample."""
    log = []
    foreign, callback = _install(monkeypatch, log)
    out = {}
    for name, make in _cases(foreign).items():
        torch.manual_seed(0)
        fn, sig, kw = make()
        x = torch.randn(2, 1, 4, 4, generator=torch.Generator().manual_seed(3)) * float(sig[0])
        del log[:]
        y = fn(toy2, x, sig, disable=True, callback=callback, **kw)
        out[name] = log[:] + [["result", bits(y)]]
    return out


def test_sampler_call_sequences_match_golden(monkeypatch):
    want = json.loads(GOLDEN_FILE.read_text())
    got = json.loads(json.dumps(trace_samplers(monkeypatch)))
    assert sorted(got) == sorted(want)
    for name in want:
        for j, (g, w) in enumerate(zip(got[name], want[name])):
            assert g == w, (name, j, g, w)
        assert len(got[name]) == len(want[name]), name
