"""Forward-mode derivative (JVP) of the native denoiser on the GPU.

The engine's J_D v (kdb_model_forward_jvp, fp32) against torch.func.jvp of the oracle's denoiser on every attention kind and both
conditioning routes, per stage through the debug taps, the exact properties of the tangent pass (bit-identical primal, exact
linearity, CUDA-graph replay) and log_likelihood(jvp=True).

Bound (tests/test_jvp_bound.py shows it separates the right derivative from near misses): rel-L2 <= 1e-4, and elementwise the fp32
gate |got - want| <= 1e-3 |want| + 1e-5 max|want|.
"""
import ctypes

import pytest
import torch

import k_diffusion as K
from k_diffusion import _native
from oracle import kdiff_oracle as O
from test_gpu_parity import build
from test_jvp_bound import NA3, check_tangent

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
S = K.sampling
DEV = "cuda"

NONSQUARE = {"model": {"type": "image_transformer_v2", "input_channels": 2, "input_size": [32, 64], "patch_size": [2, 4],
                       "depths": [1, 2], "widths": [64, 128], "mapping_cond_dim": 5, "sigma_data": 1.0,
                       "self_attns": [{"type": "shifted-window", "d_head": 32, "window_size": 4}, {"type": "global", "d_head": 64}]},
             "dataset": {"type": "x", "num_classes": 3}}


def inputs(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*shape, generator=g) * scale
    v = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
    return x, v


def oracle_jvp(om, x, v, sig, **kw):
    return torch.func.jvp(lambda xx: om(xx, sig, **kw), (x,), (v,))


# ------------------------------------------------------------------------------------------
# whole denoiser against the oracle
# ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("aug", [False, True])
def test_cfg1_per_sample_rows_vs_oracle(aug):
    """global attention, per-sample class rows, three different sigmas"""
    cfg, sd, inner, model, _ = build("cfg1_mnist")
    x, v = inputs((3, 1, 28, 28), 11, 0.8)
    sig = torch.tensor([0.05, 1.3, 20.0])
    kw = dict(class_cond=torch.tensor([1, 9, 4]))
    if aug:
        kw["aug_cond"] = torch.randn(3, 9, generator=torch.Generator().manual_seed(2))
    d, jv = model.jvp(x.to(DEV), sig.to(DEV), v.to(DEV), **{k: t.to(DEV) for k, t in kw.items()})
    want_d, want_jv = oracle_jvp(O.make_denoiser(sd, cfg["model"]), x, v, sig, **kw)
    check_tangent(d, want_d, "cfg1 D")
    check_tangent(jv, want_jv, "cfg1 J_D v")


@pytest.mark.parametrize("name", ["sw64", "na3", "nonsquare"])
def test_models_vs_oracle_both_routes(name):
    """sw64 (shift 0 and 4 at every level), [neighbourhood, none, global], and a non-square grid with mapping / class / aug
    conditioning.  The shared-row route (cond_batch_stride 0, one sigma) runs through the sampler's evaluator; the per-sample route
    through Denoiser.jvp."""
    raw = {"sw64": "sw64", "na3": NA3, "nonsquare": NONSQUARE}[name]
    cfg, sd, inner, model, _ = build(raw)
    mcfg = cfg["model"]
    C, (H, W) = mcfg["input_channels"], mcfg["input_size"]
    x, v = inputs((2, C, H, W), 21, 1.5)
    om = O.make_denoiser(sd, mcfg)
    kw = {}
    if name == "nonsquare":
        g = torch.Generator().manual_seed(6)
        kw = dict(class_cond=torch.tensor([0, 2]), mapping_cond=torch.randn(2, 5, generator=g), aug_cond=torch.randn(2, 9, generator=g))
    sig = torch.tensor([0.4, 7.0])
    d, jv = model.jvp(x.to(DEV), sig.to(DEV), v.to(DEV), **{k: t.to(DEV) for k, t in kw.items()})
    want_d, want_jv = oracle_jvp(om, x, v, sig, **kw)
    check_tangent(d, want_d, f"{name} per-sample D")
    check_tangent(jv, want_jv, f"{name} per-sample J_D v")
    if not kw:
        ev = S._Evaluator(model, x.to(DEV), {}, [1.1])
        assert not ev.per_sample
        d, jv = ev.jvp(0, x.to(DEV), v.to(DEV))
        want_d, want_jv = oracle_jvp(om, x, v, torch.full((2,), 1.1))
        check_tangent(d, want_d, f"{name} shared-row D")
        check_tangent(jv, want_jv, f"{name} shared-row J_D v")


def test_raw_inner_model_vs_oracle():
    """sigma_data <= 0: the tangent of F itself"""
    cfg, sd, inner, model, _ = build("sw64")
    x, v = inputs((2, 3, 64, 64), 31, 0.5)
    sig = torch.tensor([0.3, 3.0])
    f, jf = inner.jvp(x.to(DEV), sig.to(DEV), v.to(DEV))
    want_f, want_jf = torch.func.jvp(lambda xx: O.model_forward(sd, cfg["model"], xx, sig), (x,), (v,))
    check_tangent(f, want_f, "F")
    check_tangent(jf, want_jf, "J_F v")


# ------------------------------------------------------------------------------------------
# per stage, through the taps (primal rows followed by tangent rows)
# ------------------------------------------------------------------------------------------

def oracle_cond(sd, sigma, class_cond=None):
    emb = O.fourier_features((torch.log(sigma) / 4)[..., None], sd["time_emb.weight"]) @ sd["time_in_proj.weight"].T
    emb = emb + O.fourier_features(sigma.new_zeros(sigma.shape[0], 9), sd["aug_emb.weight"]) @ sd["aug_in_proj.weight"].T
    if "class_emb.weight" in sd:
        emb = emb + sd["class_emb.weight"][class_cond]
    return O.mapping_network(sd, emb)


def tap_jvp(inner, name, x, v, sig, kw):
    eng = inner.engine()
    buf = eng.arm_tap(name, 1 << 24, DEV)
    inner.denoise_jvp(x, sig, v, 1.0, **kw)
    n = eng.tap_count()
    assert n > 0, name
    half = buf[:n].view(2, -1)
    return half[0].cpu(), half[1].cpu()


@pytest.mark.parametrize("name,layer", [("cfg1_mnist", 0), ("cfg1_mnist", 3), ("sw64", 0), ("sw64", 1), ("na3", 0)])
def test_stage_taps_vs_oracle(name, layer):
    """.ao (norm, qkv, cosine-sim + RoPE, attention) and .geglu (norm, up_proj, GEGLU) of one layer: the tangent half of the tap
    against the oracle's JVP of that stage alone, fed with the primal and tangent halves of the previous tap"""
    raw = NA3 if name == "na3" else name
    cfg, sd, inner, model, _ = build(raw)
    mcfg = cfg["model"]
    C_in, (H, W) = mcfg["input_channels"], mcfg["input_size"]
    B = 2
    x, v = inputs((B, C_in, H, W), 41, 1.0)
    sig = torch.tensor([0.6, 5.0])
    kw = dict(class_cond=torch.tensor([2, 7])) if name == "cfg1_mnist" else {}
    x, v, sig_d = x.to(DEV), v.to(DEV), sig.to(DEV)
    kwd = {k: t.to(DEV) for k, t in kw.items()}
    cond = oracle_cond(sd, sig, kw.get("class_cond"))
    ph, pw = mcfg["patch_size"]
    h, w, C = H // ph, W // pw, mcfg["widths"][0]
    attn = mcfg["self_attns"][0]
    p = f"down_levels.0.{layer}." if len(mcfg["widths"]) > 1 else f"mid_level.{layer}."
    shape = (B, h, w, C)

    xin, tin = tap_jvp(inner, "patch_in" if layer == 0 else f"layer{layer - 1}.ff", x, v, sig_d, kwd)
    ao_p, ao_t = tap_jvp(inner, f"layer{layer}.ao", x, v, sig_d, kwd)

    def ao_stage(t):
        a = p + "self_attn."
        xn = O.rms_norm(t, (cond @ sd[a + "norm.linear.weight"].T)[:, None, None, :] + 1)
        e = attn.get("d_head", 64)
        q, k, vv = (xn @ sd[a + "qkv_proj.weight"].T).view(B, h, w, 3, C // e, e).unbind(3)
        q, k = O.cosine_sim_scale(q, k, sd[a + "scale"])
        theta = O.rope_theta(O.make_axial_pos(h, w), sd[a + "pos_emb.freqs"])
        q, k = O.apply_rope(q, theta), O.apply_rope(k, theta)
        if attn["type"] == "global":
            o = O.global_attention(q, k, vv)
        elif attn["type"] == "shifted-window":
            ws = attn["window_size"]
            o = O.shifted_window_attention(q, k, vv, ws, ws // 2 if layer % 2 == 1 else 0)
        else:
            o = O.neighborhood_attention(q, k, vv, attn.get("kernel_size", 7))
        return o.reshape(B, h, w, C)

    _, want = torch.func.jvp(ao_stage, (xin.view(shape),), (tin.view(shape),))
    check_tangent(ao_t.view(shape), want, f"{name} layer{layer}.ao tangent")

    xin, tin = tap_jvp(inner, f"layer{layer}.attn", x, v, sig_d, kwd)
    _, gg_t = tap_jvp(inner, f"layer{layer}.geglu", x, v, sig_d, kwd)

    def geglu_stage(t):
        xn = O.rms_norm(t, (cond @ sd[p + "ff.norm.linear.weight"].T)[:, None, None, :] + 1)
        return O.linear_geglu(xn, sd[p + "ff.up_proj.weight"])

    _, want = torch.func.jvp(geglu_stage, (xin.view(shape),), (tin.view(shape),))
    check_tangent(gg_t.view(want.shape), want, f"{name} layer{layer}.geglu tangent")


# ------------------------------------------------------------------------------------------
# exact properties
# ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["cfg1_mnist", "sw64"])
def test_exact_properties(name):
    cfg, sd, inner, model, _ = build(name)
    mcfg = cfg["model"]
    C, (H, W) = mcfg["input_channels"], mcfg["input_size"]
    x, v = inputs((2, C, H, W), 51, 2.0)
    x, v = x.to(DEV), v.to(DEV)
    sig = torch.tensor([0.8, 14.0], device=DEV)
    kw = dict(class_cond=torch.tensor([5, 0], device=DEV)) if name == "cfg1_mnist" else {}
    inner.set_precision("bf16")                                   # jvp always takes the fp32 path
    d, jv = model.jvp(x, sig, v, **kw)
    inner.set_precision("fp32")
    assert torch.equal(d, model(x, sig, **kw)), "primal differs from the fp32 forward"
    _, jv2 = model.jvp(x, sig, 2 * v, **kw)
    assert torch.equal(jv2, 2 * jv), "tangent is not exactly linear"
    _, j0 = model.jvp(x, sig, torch.zeros_like(v), **kw)
    assert torch.equal(j0, torch.zeros_like(j0))
    assert float(jv.abs().max()) > 0

    # CUDA graph: one forward_jvp captured (the grid's position tables exist) and replayed equals eager
    eng = inner.engine()
    ev = S._Evaluator(model, x, kw, [0.8])
    cond, stride = ev._rows(0)
    sig_b = ev.sigma_rows[0]
    out, tan = torch.empty_like(x), torch.empty_like(x)
    xs, vs = x.clone(), v.clone()
    eager = eng.forward_jvp(xs, vs, sig_b, cond, stride, ev.sigma_data)
    eager = tuple(t.clone() for t in eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.forward_jvp(xs, vs, sig_b, cond, stride, ev.sigma_data, out=out, out_tangent=tan)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.forward_jvp(xs, vs, sig_b, cond, stride, ev.sigma_data, out=out, out_tangent=tan)
    out.zero_()
    tan.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager[0]) and torch.equal(tan, eager[1])

    # bf16 at the C entry point is refused with KDB_ERR_UNSUPPORTED
    ws = torch.empty(int(_native.lib().kdb_model_workspace_bytes(eng._h, _native.PREC_FP32, 4, H, W)), dtype=torch.uint8, device=DEV)
    rc = _native.lib().kdb_model_forward_jvp(eng._h, _native.PREC_BF16, 2, H, W, _native.ptr(xs), _native.ptr(vs), _native.ptr(sig_b),
                                             ctypes.c_float(ev.sigma_data), _native.ptr(cond), stride, _native.ptr(out), _native.ptr(tan),
                                             _native.ptr(ws), ws.numel(), _native.stream())
    assert rc == -2 and b"fp32" in _native.lib().kdb_last_error()
    # the workspace is sized for 2B images
    rc = _native.lib().kdb_model_forward_jvp(eng._h, _native.PREC_FP32, 2, H, W, _native.ptr(xs), _native.ptr(vs), _native.ptr(sig_b),
                                             ctypes.c_float(ev.sigma_data), _native.ptr(cond), stride, _native.ptr(out), _native.ptr(tan),
                                             _native.ptr(ws), int(_native.lib().kdb_model_workspace_bytes(eng._h, 0, 2, H, W)), _native.stream())
    assert rc == -5


# ------------------------------------------------------------------------------------------
# log_likelihood(jvp=True)
# ------------------------------------------------------------------------------------------

def test_log_likelihood_jvp_cfg1(monkeypatch):
    cfg, sd, inner, model, z = build("cfg1_mnist")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 1, 28, 28, generator=g) * 0.4 + 0.1
    v = torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1
    cc = torch.tensor([1, 9])
    ea = dict(class_cond=cc.to(DEV))
    om = O.make_denoiser(sd, cfg["model"])
    calls = {"forward": 0, "forward_jvp": 0}
    for fn in calls:
        orig = getattr(_native.Engine, fn)

        def counted(self, *a, _orig=orig, _fn=fn, **k):
            calls[_fn] += 1
            return _orig(self, *a, **k)
        monkeypatch.setattr(_native.Engine, fn, counted)
    rhs, count = S._likelihood_rhs(model, x.to(DEV), ea, v.to(DEV), 1e-2, jvp=True)
    for sigma in (0.02, 0.7, 30.0):
        xs = x * (1 + sigma)
        d, d_ll = rhs(sigma, (xs.to(DEV), torch.zeros(2, device=DEV)))
        with torch.enable_grad():
            xg = xs.clone().requires_grad_()
            dd = (xg - om(xg, torch.full((2,), sigma), class_cond=cc)) / sigma
            want = (v * torch.autograd.grad((dd * v).sum(), xg)[0]).flatten(1).sum(1)
        assert float((d.cpu() - dd.detach()).abs().max()) <= 1e-3 * float(dd.abs().max()) + 1e-4 * float(xs.abs().max()) / sigma
        assert float((d_ll.cpu() - want).abs().max()) <= 1e-3 * float(want.abs().max()), (sigma, d_ll, want)
    assert count[0] == 3 and calls == {"forward": 0, "forward_jvp": 3}, calls
    ll, info = S.log_likelihood(model, x.to(DEV), 1e-2, 80., extra_args=ea, v=v.to(DEV), atol=1e-6, rtol=1e-6, jvp=True)
    assert calls["forward_jvp"] == 3 + info["fevals"] and calls["forward"] == 0
    ll_o, info_o = O.log_likelihood(om, x, 1e-2, 80., extra_args=dict(class_cond=cc), v=v, atol=1e-6, rtol=1e-6)
    # fp32 integrations of this ODE scatter by ~1.5e-5 relative at these tolerances (measured on one H100 and two CPUs: the fp32 oracle
    # lies 0.6e-5..1.3e-5 from a float64 oracle and differs between CPUs; this path gave 1.4e-5 from float64; the finite-difference
    # path moves by 1.3e-5 between rtol 1e-6 and 1e-7)
    assert float((ll.cpu() - ll_o).abs().max()) <= 2.5e-5 * float(ll_o.abs().max()), (ll, ll_o, info, info_o)
