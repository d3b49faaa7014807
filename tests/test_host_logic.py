"""Host-side logic of the product package, CPU only: schedules (bit-exact), DiscreteSchedule
(bit-exact integer indices), step plans, config/state-dict compatibility, sharding helpers."""
import json

import numpy as np
import pytest
import torch

import k_diffusion as K
from conftest import GOLDEN, assert_close, bits, load_fixture, load_npz, synth_sd, unhex
from oracle import kdiff_oracle as O

S = K.sampling


def test_schedules_bit_exact(kat):
    fns = dict(karras=S.get_sigmas_karras, exponential=S.get_sigmas_exponential, polyexponential=S.get_sigmas_polyexponential, vp=S.get_sigmas_vp)
    for e in kat["schedules"]:
        assert bits(fns[e["fn"]](*e["args"])) == e["hex"], e


def test_discrete_schedule_bit_exact(kat):
    d = kat["discrete"]
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000) ** 2
    ac = torch.cumprod(1 - betas, 0)
    ds = K.external.DiscreteSchedule(((1 - ac) / ac) ** 0.5, True)
    assert float(ds.sigma_min) == d["sigma_min"] and float(ds.sigma_max) == d["sigma_max"]
    assert bits(ds.get_sigmas(10)) == d["get_sigmas_10"] and bits(ds.get_sigmas(37)) == d["get_sigmas_37"]
    assert len(ds.get_sigmas()) == 1001 and bits(ds.get_sigmas()[:5]) == d["get_sigmas_all_head"]
    t = ds.sigma_to_t(ds.get_sigmas(10)[:-1])
    assert t.dtype == torch.int64 and t.tolist() == d["roundtrip_t"]
    q = unhex(d["query"])
    assert ds.sigma_to_t(q).tolist() == d["t_quant"]
    assert bits(ds.sigma_to_t(q, quantize=False)) == d["t_interp"]
    assert bits(ds.t_to_sigma(torch.tensor([0.0, 0.5, 17.25, 998.9, 999.0]))) == d["t_to_sigma"]
    assert set(ds.state_dict()) == {"sigmas", "log_sigmas"}


def test_ancestral_step_and_scalings(kat):
    for e in kat["ancestral"]:
        d, u = S.get_ancestral_step(unhex([e["sigma_from"]])[0], unhex([e["sigma_to"]])[0], eta=e["eta"])
        assert float(d) == e["down"] and float(u) == e["up"]
    s = kat["scalings"]
    cs, co, ci = K.Denoiser(None, sigma_data=s["sigma_data"]).get_scalings(torch.tensor(s["sigma"]))
    for got, want in ((cs, s["c_skip"]), (co, s["c_out"]), (ci, s["c_in"])):
        assert_close(got, unhex(want), rtol=2e-7, atol=0)


def _exec_ops(plan, model, x, noise=None):
    """CPU interpreter of the op plans (what the solver kernels and the evaluator do), for plan verification only."""
    f = np.float32
    T = {"x": x.clone()}
    B = x.shape[0]
    it = iter(noise) if noise is not None else None
    for st in plan:
        k = 0
        for op in st["ops"]:
            if op[0] == "eval":
                T[op[1]] = model(T[op[2]], torch.full([B], st["evals"][k]))
                k += 1
            elif op[0] == "lin":
                T[op[1]] = sum(f(c) * T[n] for n, c in op[2])
            elif op[0] == "euler":
                _, out, xn, dn, r, nn, cn = op
                T[out] = T[xn] + (T[xn] - T[dn]) * f(r) + (0 if nn is None else T[nn] * f(cn))
            elif op[0] == "heun":
                _, out, xn, dn, x2, d2, a1, a2 = op
                T[out] = T[xn] + ((T[xn] - T[dn]) * f(a1) + (T[x2] - T[d2]) * f(a2))
            elif op[0] == "dpmpp_2m":
                _, out, xn, dn, old, a, b, k1, k0 = op
                T[out] = f(a) * T[xn] - f(b) * (f(k1) * T[dn] + (f(k0) * T[old] if k0 != 0 else 0))
            elif op[0] == "noise":
                T[op[1]] = next(it)
            elif op[0] == "keep":
                T[op[1]] = T[op[2]]
            else:
                raise AssertionError(op)
        assert k == len(st["evals"])
    return T["x"]


def test_fused_step_plans_reproduce_reference_trajectories():
    """Euler / Heun / DPM++(2M) / Euler-ancestral op plans (fused step kinds) vs trajectories recorded from the reference
    (oracle/make_golden.py), through the same op interpreter as the other samplers' plans."""
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    z = load_npz("toy_samplers.npz")
    sig = S.host_sigmas(z["sigmas"])
    for key, plan, noise in [("sample_euler", S.plan_euler(sig), None), ("sample_heun", S.plan_heun(sig), None),
                             ("sample_dpmpp_2m", S.plan_dpmpp_2m(sig), None),
                             ("sample_euler_ancestral", S.plan_euler_ancestral(sig), z["noise"]),
                             ("sample_euler_ancestral_eta05", S.plan_euler_ancestral(sig, eta=0.5, s_noise=0.9), z["noise"])]:
        assert_close(_exec_ops(plan, toy2, z["x"], noise), z[key], rtol=1e-4, atol=1e-5, what=key)


def test_generic_op_plans_reproduce_reference_trajectories():
    """SURVEY 8f.1 samplers: host plans vs trajectories recorded from the reference (oracle/make_golden_next.py)."""
    z = load_npz("toy_next_samplers.npz")
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    sig = S.host_sigmas(z["sigmas"])
    x, nz = z["x"], z["noise"]
    cases = [
        ("sample_dpm_2", S.plan_dpm_2(sig), None),
        ("sample_lms", S.plan_lms(sig), None),
        ("sample_lms_order2", S.plan_lms(sig, order=2), None),
        ("sample_dpm_2_ancestral", S.plan_dpm_2_ancestral(sig), nz),
        ("sample_dpm_2_ancestral_eta05", S.plan_dpm_2_ancestral(sig, eta=0.5, s_noise=0.9), nz),
        ("sample_dpmpp_2s_ancestral", S.plan_dpmpp_2s_ancestral(sig), nz),
        ("sample_dpmpp_2s_ancestral_eta0", S.plan_dpmpp_2s_ancestral(sig, eta=0.), nz),
        ("sample_dpmpp_sde", S.plan_dpmpp_sde(sig), nz),
        ("sample_dpmpp_sde_r03", S.plan_dpmpp_sde(sig, eta=0.7, s_noise=0.9, r=0.3), nz),
        ("sample_dpmpp_2m_sde", S.plan_dpmpp_2m_sde(sig), nz),
        ("sample_dpmpp_2m_sde_heun", S.plan_dpmpp_2m_sde(sig, eta=0.6, solver_type="heun"), nz),
        ("sample_dpmpp_2m_sde_eta0", S.plan_dpmpp_2m_sde(sig, eta=0.), nz),
        ("sample_dpmpp_3m_sde", S.plan_dpmpp_3m_sde(sig), nz),
        ("sample_dpmpp_3m_sde_eta05", S.plan_dpmpp_3m_sde(sig, eta=0.5, s_noise=0.8), nz),
    ]
    for key, plan, noise in cases:
        assert_close(_exec_ops(plan, toy2, x, noise), z[key], rtol=1e-4, atol=2e-5, what=key)
        assert all(len(terms) <= 6 for st in plan for op in st["ops"] if op[0] == "lin" for terms in [op[2]])   # one lincomb launch each
    assert sum(len(st["evals"]) for st in S.plan_dpm_2(sig)) == 19 and sum(len(st["evals"]) for st in S.plan_lms(sig)) == 10
    with pytest.raises(ValueError):
        S.plan_dpmpp_2m_sde(sig, solver_type="euler")
    with pytest.raises(ValueError):
        S.plan_lms(sig, order=0)
    assert max(len(op[2]) for st in S.plan_lms(sig, order=5) for op in st["ops"] if op[0] == "lin") == 6     # x + five derivative buffers


def test_generic_sampler_entry_points_with_stubbed_kernels(monkeypatch):
    """The executor behind sample_dpm_2 / lms / dpmpp_*_sde, driven end to end on the CPU by replacing the three native
    primitives it touches with torch one-liners (test-only stubs; the product has no CPU path).  Checks op interpretation,
    evaluation order, callback payloads and the noise-sampler calling convention against the reference trajectories."""
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())
    monkeypatch.setattr(_native, "lincomb", lambda ts, cs, out=None: sum(np.float32(c) * t for t, c in zip(ts, cs)))
    z = load_npz("toy_next_samplers.npz")
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    x, sig, nz = z["x"], z["sigmas"], z["noise"]

    def ns():
        it = iter(nz)
        return lambda a, b: next(it)

    runs = {
        "sample_dpm_2": lambda: S.sample_dpm_2(toy2, x, sig, disable=True),
        "sample_lms": lambda: S.sample_lms(toy2, x, sig, disable=True),
        "sample_dpm_2_ancestral_eta05": lambda: S.sample_dpm_2_ancestral(toy2, x, sig, disable=True, eta=0.5, s_noise=0.9, noise_sampler=ns()),
        "sample_dpmpp_2s_ancestral": lambda: S.sample_dpmpp_2s_ancestral(toy2, x, sig, disable=True, noise_sampler=ns()),
        "sample_dpmpp_sde_r03": lambda: S.sample_dpmpp_sde(toy2, x, sig, disable=True, eta=0.7, s_noise=0.9, r=0.3, noise_sampler=ns()),
        "sample_dpmpp_2m_sde_heun": lambda: S.sample_dpmpp_2m_sde(toy2, x, sig, disable=True, eta=0.6, solver_type="heun", noise_sampler=ns()),
        "sample_dpmpp_3m_sde": lambda: S.sample_dpmpp_3m_sde(toy2, x, sig, disable=True, noise_sampler=ns()),
    }
    for key, run in runs.items():
        assert_close(run(), z[key], rtol=1e-4, atol=2e-5, what=key)
    zh = load_npz("toy_lms_high_order.npz")          # any order: x + more than five derivative buffers = chained lincomb launches
    for o in (5, 6, 7, 10):
        assert_close(S.sample_lms(toy2, zh["x"], zh["sigmas"], disable=True, order=o), zh[f"sample_lms_order{o}"], rtol=1e-5, atol=5e-6, what=f"lms {o}")
    assert max(len(op[2]) for st in S.plan_lms(S.host_sigmas(zh["sigmas"]), 10) for op in st["ops"] if op[0] == "lin") == 11
    with pytest.raises(ValueError):
        S.sample_lms(toy2, x, sig, disable=True, order=0)
    seen = []
    S.sample_dpmpp_2m_sde(toy2, x, sig, disable=True, noise_sampler=ns(), callback=seen.append)
    assert [c["i"] for c in seen] == list(range(10)) and set(seen[0]) == {"x", "i", "sigma", "sigma_hat", "denoised"}
    assert torch.equal(seen[0]["x"], x) and float(seen[3]["sigma"]) == float(sig[3])
    calls = []
    S.sample_dpmpp_sde(toy2, x, sig, disable=True, noise_sampler=lambda a, b: calls.append((float(a), float(b))) or nz[0])
    assert len(calls) == 18 and all(a > b for a, b in calls)        # two draws per step except the final Euler step, sigma decreasing
    with pytest.raises(ValueError):
        S.sample_dpmpp_2m_sde(toy2, x, sig, solver_type="euler")


def test_op_plan_details():
    sig = S.host_sigmas(S.get_sigmas_karras(50, 1e-2, 160))
    kinds = lambda st: [op[0] for op in st["ops"]]
    heun = S.plan_heun(sig)
    assert sum(len(st["evals"]) for st in heun) == 99                       # NFE of Heun-50 (SURVEY 3.2)
    assert kinds(heun[-1]) == ["eval", "euler"] and heun[-1]["ops"][-1][4] == -1.0      # final Euler step lands on denoised
    assert sum(len(st["evals"]) for st in S.plan_dpmpp_2m(S.host_sigmas(S.get_sigmas_karras(25, 1e-2, 160)))) == 25
    d = [[op for op in st["ops"] if op[0] == "dpmpp_2m"][0] for st in S.plan_dpmpp_2m(sig)]     # (kind, out, x, den, old, a, b, k1, k0)
    assert d[0][8] == 0 and d[-1][5] == 0 and d[-1][6] == -1 and d[-1][8] == 0
    ch = S.plan_heun(sig, s_churn=40, s_tmin=0.05, s_tmax=50)
    on = [st for st in ch if st["gamma"] > 0]
    assert on and all(0.05 <= sig[st["i"]] <= 50 for st in on) and all(abs(st["gamma"] - (2 ** 0.5 - 1)) < 1e-12 for st in on)
    assert all(kinds(st)[:3] == ["randn", "lin", "eval"] if st["gamma"] > 0 else "randn" not in kinds(st) for st in ch)   # draw before the step
    ea = S.plan_euler_ancestral(sig)
    assert "noise" not in kinds(ea[-1]) and ea[-1]["ops"][-1][4] == -1.0 and all("noise" in kinds(st) for st in ea[:-1])
    with pytest.raises(ValueError):
        S.host_sigmas(torch.zeros(1))


@pytest.mark.parametrize("stem", ["cfg1_mnist", "sw64", "cfg2_sw256"])
def test_config_and_state_dict_match_reference(stem):
    meta = json.loads((GOLDEN / f"{stem}_shapes.json").read_text())
    raw = {"model": {k: v for k, v in meta["config"]["model"].items()}, "dataset": meta["config"]["dataset"]}
    cfg = K.config.load_config(raw)
    assert cfg["model"] == meta["config"]["model"]
    model = K.config.make_model(cfg)
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == meta["shapes"]
    den = K.config.make_denoiser_wrapper(cfg)(model)
    assert den.sigma_data == cfg["model"]["sigma_data"] and den.inner_model is model


def test_config_defaults_from_minimal_json():
    cfg = K.config.load_config({"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [64, 64], "patch_size": [4, 4],
                                          "depths": [2, 2], "widths": [128, 256]}})
    ref = json.loads((GOLDEN / "cfg3_na256_config.json").read_text())["config"]
    assert cfg["model"]["self_attns"] == [{"type": "neighborhood", "d_head": 64, "kernel_size": 7}, {"type": "global", "d_head": 64}]
    assert cfg["model"]["d_ffs"] == [384, 768] and cfg["model"]["mapping_d_ff"] == 768 and cfg["model"]["dropout_rate"] == [0.0, 0.0]
    assert set(cfg) == set(ref)
    with pytest.raises(ValueError):
        K.config.load_config({"model": {"type": "image_v1"}})


def test_fresh_model_init_matches_reference_distribution():
    torch.manual_seed(0)
    cfg = K.config.load_config(json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"])
    sd = K.config.make_model(cfg).state_dict()
    for k, v in sd.items():
        if k.endswith(("out_proj.weight", "down_proj.weight", "norm.linear.weight", "patch_out.proj.weight")):
            assert not v.any(), k                                           # zero-initialised in the reference
    assert torch.all(sd["mid_level.0.self_attn.scale"] == 10) and float(sd["out_norm.scale"].mean()) == 1
    w = sd["mid_level.0.self_attn.qkv_proj.weight"]
    assert abs(float(w.std()) - (1 / 256 ** 0.5) / 3 ** 0.5) < 2e-3 and float(w.abs().max()) <= 1 / 16
    assert bits(sd["mid_level.3.self_attn.pos_emb.freqs"]) == bits(O.rope_freqs(64, 4))


def test_cpu_tensors_are_rejected_not_emulated():
    cfg = K.config.load_config(json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"])
    model = K.Denoiser(K.config.make_model(cfg), sigma_data=0.6162)
    x = torch.zeros(1, 1, 28, 28)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(x, torch.ones(1), class_cond=torch.zeros(1, dtype=torch.long))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.sample_heun(lambda x, s: x, x, S.get_sigmas_karras(3, 0.1, 10))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.to_d(x, torch.ones(()), x)


def test_synth_weights_are_order_independent():
    a = K.synth.synth_tensor("mid_level.0.ff.up_proj.weight", (8, 4), seed=1)
    b = K.synth.synth_tensor("mid_level.0.ff.up_proj.weight", (8, 4), seed=1)
    c = K.synth.synth_tensor("mid_level.0.ff.up_proj.weight", (8, 4), seed=2)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert float(K.synth.synth_tensor("x.out_proj.weight", (64, 64), 0).std()) < 0.03


def test_shard_helpers():
    P = K.parallel
    for n, w in [(256, 8), (10, 4), (3, 8), (128, 1)]:
        spans = [P.shard_range(n, r, w) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == n and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        assert max(b - a for a, b in spans) - min(b - a for a, b in spans) <= 1
    full = P.sample_seeds(7, 0, 16)
    assert len(set(full)) == 16 and all(0 <= s < 2 ** 63 for s in full)
    assert P.sample_seeds(7, 4, 9) == full[4:9] and P.sample_seeds(8, 0, 16) != full


def test_dpm_solver_plans_and_entry_points_with_stubbed_kernels(monkeypatch):
    """SURVEY 8(f) row 4: sample_dpm_fast (an op plan like the other fixed-schedule samplers) and sample_dpm_adaptive (host PID loop
    around the same lincomb / evaluation / error-norm primitives) against outputs recorded from the reference
    (oracle/make_golden_dpm.py), step and rejection counts included.  Native primitives replaced by torch one-liners (test-only)."""
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())
    monkeypatch.setattr(_native, "lincomb", lambda ts, cs, out=None: sum(np.float32(c) * t for t, c in zip(ts, cs)))

    def dpm_error(lo, hi, prev, atol, rtol):
        delta = torch.maximum(torch.tensor(atol), torch.tensor(rtol) * torch.maximum(lo.abs(), prev.abs()))
        return float(torch.linalg.norm((lo - hi) / delta) / lo.numel() ** 0.5)

    monkeypatch.setattr(_native, "dpm_error", dpm_error)
    monkeypatch.setattr(S, "_on_x_device", lambda fn: fn, raising=False)
    z = load_npz("toy_dpm_solvers.npz")
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    x = z["x"]

    def ns():
        it = iter(z["noise"])
        return lambda a, b: next(it)

    fast = S.sample_dpm_fast.__wrapped__ if hasattr(S.sample_dpm_fast, "__wrapped__") else S.sample_dpm_fast
    adaptive = S.sample_dpm_adaptive.__wrapped__ if hasattr(S.sample_dpm_adaptive, "__wrapped__") else S.sample_dpm_adaptive
    for n in (4, 5, 6, 9, 10):
        plan, ts = S.plan_dpm_fast(1e-2, 80., n)
        assert sum(len(st["evals"]) for st in plan) == n                       # the NFE budget is met exactly (sampling.py:409-417)
        assert all(len(op[2]) <= 6 for st in plan for op in st["ops"] if op[0] == "lin")
        assert_close(fast(toy2, x, 1e-2, 80., n, disable=True), z[f"dpm_fast_n{n}"], rtol=1e-4, atol=2e-5, what=f"dpm_fast n={n}")
    assert_close(fast(toy2, x, 1e-2, 80., 7, disable=True, eta=0.5, s_noise=0.9, noise_sampler=ns()), z["dpm_fast_n7_eta05"], rtol=1e-4, atol=2e-5)
    # eta = 1 from sigma 80 (|x| up to 250, step coefficients ~20) is ill-conditioned in fp32: a 1e-7 relative change of any step
    # coefficient moves the result by 2e-4, and the reference's own fp32 run sits 3.6e-4 from the float64 evaluation of the same formulas
    # (the plan: 5.0e-4; in float64 with float64 coefficients plan and reference formulas agree to 1e-12).  North-star rtol with an
    # absolute floor at that noise:
    assert_close(fast(toy2, x, 1e-2, 80., 6, disable=True, eta=1.0, noise_sampler=ns()), z["dpm_fast_n6_eta1"], rtol=1e-3, atol=1e-3)
    cases = {"dpm_adaptive_o3": dict(), "dpm_adaptive_o2": dict(order=2), "dpm_adaptive_o3_tight": dict(rtol=0.01, atol=0.002, h_init=0.1),
             "dpm_adaptive_o3_pid": dict(pcoeff=0.2, icoeff=0.7, dcoeff=0.1, accept_safety=0.9), "dpm_adaptive_o3_eta05": dict(eta=0.5, s_noise=0.9)}
    for name, kw in cases.items():
        got, info = adaptive(toy2, x, 1e-2, 80., disable=True, return_info=True, noise_sampler=ns() if kw.get("eta") else None, **kw)
        assert [info[k] for k in ("steps", "nfe", "n_accept", "n_reject")] == [int(v) for v in z[name + "_info"]], name
        # the step sizes feed back through the error norm: coefficient differences of 1e-7 grow like in the eta = 1 case above;
        # same accept / reject sequence, result within the north-star rtol of the signal's scale
        assert float((got - z[name]).abs().max()) <= 1e-3 * float(z[name].abs().max()), (name, float((got - z[name]).abs().max()))
    seen = []
    fast(toy2, x, 1e-2, 80., 6, disable=True, callback=seen.append)
    assert [c["i"] for c in seen] == [0, 1, 2] and {"x", "i", "sigma", "sigma_hat", "denoised", "t", "t_up"} <= set(seen[0])
    with pytest.raises(ValueError):
        adaptive(toy2, x, 1e-2, 80., order=4)
    with pytest.raises(ValueError):
        fast(toy2, x, 0., 80., 6)
    # the reference's driver object (sampling.py:333-488): same numbers through DPMSolver, callbacks at the reference's cadence
    evals, infos = [], []
    solver = S.DPMSolver(toy2, eps_callback=lambda: evals.append(1), info_callback=infos.append)
    t_start, t_end = solver.t(torch.tensor(80.)), solver.t(torch.tensor(1e-2))
    assert float(solver.sigma(t_start)) == pytest.approx(80.)
    assert_close(solver.dpm_solver_fast(x, t_start, t_end, 10), z["dpm_fast_n10"], rtol=1e-4, atol=2e-5, what="DPMSolver.dpm_solver_fast")
    assert len(evals) == 10 and [c["i"] for c in infos] == [0, 1, 2, 3] and {"x", "t", "t_up", "denoised"} <= set(infos[0])
    evals.clear()
    got, info = solver.dpm_solver_adaptive(x, t_start, t_end)
    assert [info[k] for k in ("steps", "nfe", "n_accept", "n_reject")] == [int(v) for v in z["dpm_adaptive_o3_info"]] and len(evals) == info["nfe"]
    assert float((got - z["dpm_adaptive_o3"]).abs().max()) <= 1e-3 * float(z["dpm_adaptive_o3"].abs().max())
    with pytest.raises(NotImplementedError):
        solver.dpm_solver_fast(x, t_end, t_start, 10)
    with pytest.raises(ValueError):
        solver.dpm_solver_adaptive(x, t_end, t_start, eta=0.5)
    assert S.linear_multistep_coeff is S.lms_coefficient


def test_log_likelihood_host_logic_with_stubbed_kernels(monkeypatch):
    """SURVEY 8(f) row 4, log_likelihood: the product's dopri5 host loop (lincomb launches + one error-ratio read per step) against the
    values recorded from the reference (oracle/make_golden_ll.py) through the autograd branch, and the native branch -- 4th-order
    central difference of the engine's fp32 evaluations instead of a VJP -- against the oracle's autograd evaluation of the same
    quadratic form on the cfg1 model.  Native primitives replaced by torch one-liners (test-only stubs)."""
    import k_diffusion as K
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())
    monkeypatch.setattr(_native, "lincomb", lambda ts, cs, out=None: sum(np.float32(c) * t for t, c in zip(ts, cs)))
    monkeypatch.setattr(_native, "rk_error", lambda err, y0, y1, atol, rtol:
                        float((err / (atol + rtol * torch.maximum(y0.abs(), y1.abs()))).pow(2).mean().sqrt()))
    ll_fn = S.log_likelihood
    while hasattr(ll_fn, "__wrapped__"):
        ll_fn = ll_fn.__wrapped__                      # below the device guard (no CUDA here)
    z = load_npz("toy_log_likelihood.npz")
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    gauss = lambda x, s, **kw: x * (0.49 / (0.49 + s[:, None, None, None] ** 2))
    for name, model, kw in (("toy", toy2, {}), ("gauss", gauss, {}), ("toy_tight", toy2, dict(atol=1e-6, rtol=1e-6))):
        with torch.no_grad():
            ll, info = ll_fn(model, z["x"], 1e-2, 80., v=z[name + "_v"], **kw)
        # the first error estimates are differences of nearly equal stages (fp32 round-off level), so the two evaluation orders may
        # pick slightly different early steps: same step count within two, values within the integration tolerance
        assert abs(info["fevals"] - int(z[name + "_fevals"])) <= 12 and info["fevals"] == 2 + 6 * (info["n_accept"] + info["n_reject"]), (name, info)
        tol = kw.get("rtol", 1e-4)
        assert float((ll - z[name + "_ll"]).abs().max()) <= 3 * tol * float(z[name + "_ll"].abs().max()), (name, ll, z[name + "_ll"])
    with torch.no_grad(), pytest.raises(RuntimeError):                         # a model autograd cannot see through fails loudly
        ll_fn(lambda x, s: x.detach() * 0.5, z["x"], 1e-2, 80.)
    assert len(S._DP5_BETA[-1]) == 6 and S._DP5_C_ERR[1] == 0 and S._DP5_C_MID[1] == 0      # every stage fits one 6-input lincomb
    assert [tuple(r) for r in S._DP5_BETA] == [tuple(r) for r in O.DOPRI5_BETA] and S._DP5_C_ERR == O.DOPRI5_C_ERR and S._DP5_C_MID == O.DOPRI5_C_MID

    # native branch: right-hand side by finite differences of (stubbed) engine evaluations vs autograd through the oracle model
    cfg, shapes, _ = load_fixture("cfg1_mnist")
    omodel = O.make_denoiser(synth_sd(shapes, 1), cfg["model"])
    den = K.config.make_denoiser_wrapper(cfg)(K.config.make_model(cfg))
    assert den.is_native()
    seen = []

    class StubEvaluator:                                # stands in for the engine: evaluates the oracle model, records what was asked
        def __init__(self, model, x, extra_args, sigmas):
            self.sig, self.ea = sigmas, extra_args
            seen.append(self)

        def __call__(self, k, x):
            with torch.no_grad():
                return omodel(x, torch.full((x.shape[0],), self.sig[k]), **self.ea)

    monkeypatch.setattr(S, "_Evaluator", StubEvaluator)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 1, 28, 28, generator=g) * 0.4 + 0.1
    v = torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1
    ea = {"class_cond": torch.tensor([1, 9])}
    rhs, count = S._likelihood_rhs(den, x, ea, v, 1e-2)
    for sigma in (0.02, 0.7, 30.0):
        xs = x * (1 + sigma)
        with torch.no_grad():
            d, d_ll = rhs(sigma, (xs, torch.zeros(2)))
        assert seen[-1].precision == _native.PREC_FP32 and len(seen[-1].sig) == 5
        with torch.enable_grad():
            xg = xs.clone().requires_grad_()
            dd = (xg - omodel(xg, torch.full((2,), sigma), **ea)) / sigma
            want = (v * torch.autograd.grad((dd * v).sum(), xg)[0]).flatten(1).sum(1)
        assert_close(d, dd.detach(), rtol=1e-5, atol=1e-6 * float(xs.abs().max()) / sigma, what=f"d at sigma {sigma}")     # (x - D) / sigma cancels
        assert float((d_ll - want).abs().max()) <= 2e-3 / sigma + 1e-4 * float(want.abs().max()), (sigma, d_ll, want)
    assert count[0] == 3
    with torch.no_grad():
        ll, info = ll_fn(den, x, 1e-2, 80., extra_args=ea, v=v)
    ll_o, info_o = O.log_likelihood(omodel, x, 1e-2, 80., extra_args=ea, v=v)
    # at the default tolerances two correct integrations differ by a few rtol * |ll| (measured: the tight-tolerance value lies between)
    assert float((ll - ll_o).abs().max()) <= 1e-3 * float(ll_o.abs().max()) and abs(info["fevals"] - info_o["fevals"]) <= 18


def test_public_api_matches_reference_signatures():
    """SURVEY 8(b): every public name of the reference's API for the path exists here and is callable with the reference's arguments --
    same parameter names, order, kinds and defaults (tests/golden/api_signatures.json, recorded by oracle/make_golden_api.py from the real
    reference).  Extra parameters are allowed only AFTER the reference's, keyword-only or with a default."""
    import inspect
    from k_diffusion.models import image_transformer_v2 as itv2
    ref = json.loads((GOLDEN / "api_signatures.json").read_text())
    roots = {"sampling": S, "layers": K.layers, "external": K.external, "config": K.config, "utils": K.utils, "models": itv2}

    def same_default(ours, theirs):
        if ours == theirs:
            return True
        if theirs.startswith("<function"):                       # e.g. transform=lambda x: x
            return ours.startswith("<function")
        try:
            return float(eval(ours)) == float(eval(theirs))      # 1.0 / 1. / 1, inf
        except Exception:
            return False

    assert len(ref) >= 45
    for label, want in ref.items():
        obj = roots[label.split(".")[0]]
        for part in label.split(".")[1:]:
            assert hasattr(obj, part), f"{label}: missing"
            obj = getattr(obj, part)
        got = [[n, p.kind.name, None if p.default is inspect._empty else repr(p.default)] for n, p in inspect.signature(obj).parameters.items()]
        if any(w[1] == "VAR_KEYWORD" for w in want):             # **kwargs stays last; named extras may sit in front of it
            assert any(g[1] == "VAR_KEYWORD" for g in got), f"{label}: **kwargs dropped"
            want, got = [w for w in want if w[1] != "VAR_KEYWORD"], [g for g in got if g[1] != "VAR_KEYWORD"]
        head, extra = got[:len(want)], got[len(want):]
        for g, w in zip(head, want):
            assert g[0] == w[0] and g[1] == w[1], f"{label}: parameter {g} vs reference {w}"
            if w[2] is None:
                assert g[2] is None, f"{label}: {g[0]} gained a default"
            else:
                assert g[2] is not None and same_default(g[2], w[2]), f"{label}: default of {g[0]} is {g[2]}, reference {w[2]}"
        assert len(head) == len(want), f"{label}: parameters missing: {want[len(head):]}"
        for g in extra:
            assert g[1] in ("KEYWORD_ONLY", "VAR_KEYWORD") or g[2] is not None, f"{label}: extra required parameter {g}"


def test_denoiser_wrapper_variants_follow_reference_config():
    """config.py:216-232: 'karras' (+ has_variance) and 'simple' loss configs select wrappers that differ in the training loss only."""
    base = json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"]
    mk = lambda **kw: K.config.make_denoiser_wrapper({"model": {**base["model"], **kw}})
    assert mk().func is K.layers.Denoiser and mk().keywords["sigma_data"] == base["model"]["sigma_data"]
    assert mk(has_variance=True).func is K.layers.DenoiserWithVariance and "scales" not in mk(has_variance=True).keywords
    assert mk(loss_config="simple").func is K.layers.SimpleLossDenoiser and set(mk(loss_config="simple").keywords) == {"sigma_data"}
    assert issubclass(K.layers.SimpleLossDenoiser, K.Denoiser) and K.layers.SimpleLossDenoiser.forward is K.Denoiser.forward
    with pytest.raises(ValueError):
        mk(loss_config="simple", has_variance=True)
    with pytest.raises(ValueError):
        mk(loss_config="vp")


def test_sample_script_command_line_matches_reference():
    """sample.py (reference sample.py:17-31): same flags and defaults; the additions are optional."""
    import runpy
    from conftest import ROOT
    mod = runpy.run_path(str(ROOT / "k-diffusion_b200" / "sample.py"), run_name="sample_script")
    a = mod["cli"](["--checkpoint", "m.safetensors"])
    assert (a.batch_size, a.n, a.steps, a.prefix, a.config) == (64, 64, 50, "out", None) and str(a.checkpoint) == "m.safetensors"
    assert (a.seed, a.precision, a.sampler) == (None, "fp32", "sample_lms")
    with pytest.raises(SystemExit):
        mod["cli"]([])                                                       # --checkpoint is required
    assert mod["image_shape"]({"input_size": [32, 32], "input_channels": 3}) == (3, 32, 32)
    with pytest.raises(SystemExit):
        mod["image_shape"]({"input_size": [32, 64], "input_channels": 3})


def test_karras_churn_entry_points_with_stubbed_kernels(monkeypatch):
    """s_churn > 0 through the product's plans (sample_euler / sample_heun fused-step kernels, sample_dpm_2 op plan) against the reference
    outputs of oracle/make_golden_churn.py.  The product draws noise only on steps with gamma > 0 (quirk Q1): it is fed the reference's
    draws of exactly those steps.  Native primitives replaced by torch one-liners (test-only stubs)."""
    from k_diffusion import _native
    f = np.float32
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "f32c", lambda t: t.to(torch.float32).contiguous())
    monkeypatch.setattr(_native, "lincomb", lambda ts, cs, out=None: sum(f(c) * t for t, c in zip(ts, cs)))
    monkeypatch.setattr(_native, "euler_step", lambda x, den, r, noise=None, cn=0.0, out=None: x + (x - den) * f(r) + (0 if noise is None else noise * f(cn)))
    monkeypatch.setattr(_native, "heun_correct", lambda x, d1, x2, d2, a1, a2, out=None: x + ((x - d1) * f(a1) + (x2 - d2) * f(a2)))
    z = load_npz("toy_churn.npz")
    toy2 = lambda x, s, **kw: x / (1 + s[:, None, None, None] ** 2) + 0.1 * torch.tanh(x)
    sig = S.host_sigmas(z["sigmas"])
    cases = {"euler_churn20": (S.sample_euler, S.plan_euler, dict(s_churn=20.)),
             "heun_churn3_window": (S.sample_heun, S.plan_heun, dict(s_churn=3., s_tmin=0.1, s_tmax=30., s_noise=1.1)),
             "dpm_2_churn2": (S.sample_dpm_2, S.plan_dpm_2, dict(s_churn=2.))}
    for name, (fn, plan_fn, kw) in cases.items():
        plan = plan_fn(sig, **{k: v for k, v in kw.items() if k != "s_noise"})
        active = [st["i"] for st in plan if st.get("gamma", 0) > 0]
        assert active and (name != "heun_churn3_window" or len(active) < len(plan))           # the window case skips steps
        it = iter([z[name + "_eps"][i] for i in active])
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: next(it))
        assert_close(fn(toy2, z["x"], z["sigmas"], disable=True, **kw), z[name], rtol=1e-4, atol=2e-5, what=name)
        assert next(it, None) is None                                                          # every recorded draw of an active step was used
