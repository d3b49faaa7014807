"""The image_v1 U-Net at the tf32 precision on the H100: kdb_unet_conv_tf32 (every convolution of the engine on the tensor cores) and the
whole denoiser with it.

- The convolution bit for bit against float64 torch conv2d on dyadic operands, which are exact in tf32 and whose every partial sum is exact
  in fp32, over the shape matrix of the fp32 convolution's test plus 7x7 grids: one wrong tap, channel, source offset, residual column,
  pixel or output row fails.  On normal operands within the error bound of tf32 operands and fp32 accumulation.
- The attention (kdb_attention at tf32) against float64 softmax attention at 49, 64, 256 and 1024 keys, 1 to 8 heads, within the bound
  of its tf32 operands; a head size other than 64 takes attn_generic.
- Every stage of mnist and cifar10 against the float64 oracle stage, with the engine's tf32 operand rounding, fed the engine's own input.
- The whole denoiser of the four reference configs and the six edge configs, and the mnist Heun-10 trajectory, against the reference's
  fp32 recordings within twice the reference's own tf32 deviation (tests/golden/tf32_budget.json, oracle/make_golden_tf32.py).
- Routes (every convolution launches as unet_conv_tf32 and every d_head-64 attention as unet_attn_tf32), determinism, batch independence,
  separate CUDA graphs for fp32 and tf32 calls on one model, and the refusals of the tf32 precision outside the U-Net.
"""
import json

import pytest
import torch
from torch.nn import functional as F

import k_diffusion as K
from conftest import GOLDEN, load_npz
from oracle import kdiff_oracle as O
from oracle import unet_oracle as U
from oracle.make_golden_tf32 import tf32_round, tf32_sdpa, tf32_trunc
from test_gpu_unet import META, build, oracle_mapping_cond, unet_engine
from test_gpu_unet_kernels import CONV_CASES, GUARD, conv_ref, device_kwargs, dyadic, edge
from test_unet_edges_host import VARIANTS, variant_kwargs

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
BUDGET = json.loads((GOLDEN / "tf32_budget.json").read_text())
DEV = "cuda"
N = K._native


# ------------------------------------------------------------------------------------------------------------------------------
# tf32 arithmetic of the engine, restated
# ------------------------------------------------------------------------------------------------------------------------------

class Tf32Functional:
    """torch.nn.functional for the oracle with the engine's tf32 arithmetic: every dense conv2d but the listed fp32 ones takes its input
    truncated and its weight rounded to tf32 (the depthwise resampling filters stay exact); the attention truncates q, k, v and P."""

    def __init__(self, fp32_weights):
        self._keep = {id(w) for w in fp32_weights}

    def __getattr__(self, name):
        return getattr(F, name)

    def conv2d(self, x, w, *args, **kwargs):
        if id(w) in self._keep or kwargs.get("groups", 1) != 1:
            return F.conv2d(x, w, *args, **kwargs)
        return F.conv2d(tf32_trunc(x), tf32_round(w), *args, **kwargs)

    @staticmethod
    def scaled_dot_product_attention(q, k, v, *args, **kwargs):
        return tf32_sdpa(q, k, v, *args, **kwargs)


def rel_l2(a, b):
    a, b = a.cpu().double(), b.cpu().double()
    return float((a - b).norm() / b.norm())


def tf32_oracle(monkeypatch, sd64):
    """the oracle's functional model with the engine's tf32 arithmetic (proj_in / proj_out stay fp32, as in the engine)"""
    monkeypatch.setattr(U, "F", Tf32Functional([sd64["proj_in.weight"], sd64["proj_out.weight"]]))


# ------------------------------------------------------------------------------------------------------------------------------
# kdb_unet_conv_tf32
# ------------------------------------------------------------------------------------------------------------------------------

TF32_CASES = CONV_CASES + [
    (3, 7, 7, 36, 0, 68, 3, "r1"),            # 7x7 grids: two images and a padded row and column per M tile
    (2, 7, 7, 68, 36, 36, 1, 12),             # 7x7, two sources with c1 % 32 == 4 (a channel block holds both), residual split at 12
]


def run_conv_tf32(x1, w, ks, x2=None, bias=None, r1=None, r2=None):
    """kdb_unet_conv_tf32 into a NaN-filled buffer GUARD floats longer than the output: -> output; asserts it fully written, the guard untouched"""
    B, h, wd, _ = x1.shape
    n = B * h * wd * w.shape[0]
    buf = torch.full((n + GUARD,), float("nan"), device=DEV)
    out = N.unet_conv_tf32(x1, w, ks, x2=x2, bias=bias, r1=r1, r2=r2, out=buf[:n].view(B, h, wd, w.shape[0]))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all(), "an output element was not written"
    assert torch.isnan(buf[n:]).all(), "the kernel wrote past the end of its output"
    return out


def operands(case, make):
    B, H, W, c1, c2, Nn, ks, res = case
    x1 = make((B, H, W, c1), 4)
    x2 = make((B, H, W, c2), 4) if c2 else None
    w = make((Nn, ks * ks, c1 + c2), 8)
    r1 = r2 = None
    if res == "r1":
        r1 = make((B, H, W, Nn), 2)
    elif res is not None:
        r1, r2 = make((B, H, W, res), 2), make((B, H, W, Nn - res), 2)
    return x1, x2, w, r1, r2


def cpu(t):
    return None if t is None else t.cpu()


@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("case", TF32_CASES, ids=lambda c: "B{}_{}x{}_c{}+{}_N{}_k{}_r{}".format(*c))
def test_conv_tf32_exact_on_dyadic_operands(case, with_bias):
    g = torch.Generator().manual_seed(TF32_CASES.index(case))
    x1, x2, w, r1, r2 = operands(case, lambda shape, den: dyadic(g, shape, den))
    bias = dyadic(g, (case[5],), 4, -8, 8) if with_bias else None
    for t in (x1, x2, w):
        assert t is None or torch.equal(tf32_trunc(t), t), "operand not exact in tf32"
    got = run_conv_tf32(x1, w, case[6], x2, bias, r1, r2)
    want = conv_ref(cpu(x1), cpu(x2), cpu(w), case[6], cpu(bias), cpu(r1), cpu(r2))
    assert torch.equal(want.float().double(), want), "operands too large for an exact fp32 sum"
    bad = got.cpu().double() != want
    assert not bad.any(), f"{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()} (b, y, x, n)"


@pytest.mark.parametrize("case", [(3, 5, 9, 36, 0, 68, 3, 28), (2, 12, 20, 64, 32, 96, 3, None), (3, 6, 10, 20, 12, 36, 1, "r1"),
                                  (2, 16, 16, 128, 128, 256, 3, None)],
                         ids=lambda c: "B{}_{}x{}_c{}+{}_N{}_k{}_r{}".format(*c))
def test_conv_tf32_random_operands_within_the_tf32_error_bound(case):
    """Inputs and weights both truncated to tf32 (relative error < 2^-10 each), fp32 accumulation of K products:
    |got - exact| <= (2^-9 + 4 (K + 2) 2^-24) (|A| conv |W| + |bias| + |residual|) element by element.  Against the operands the tensor
    cores see (both truncated, float64 conv) the error is the accumulation's alone: <= 4 (K + 2) 2^-24 of the same magnitude."""
    B, H, W, c1, c2, Nn, ks, res = case
    g = torch.Generator().manual_seed(12)
    x1, x2, w, r1, r2 = operands(case, lambda shape, den: torch.randn(*shape, generator=g).to(DEV) / den * 2)
    bias = torch.randn(Nn, generator=g).to(DEV)
    got = run_conv_tf32(x1, w, ks, x2, bias, r1, r2).cpu().double()
    want = conv_ref(cpu(x1), cpu(x2), cpu(w), ks, cpu(bias), cpu(r1), cpu(r2))
    mag = conv_ref(cpu(x1).abs(), cpu(x2).abs() if x2 is not None else None, cpu(w).abs(), ks, cpu(bias).abs(),
                   None if r1 is None else cpu(r1).abs(), None if r2 is None else cpu(r2).abs())
    K_ = ks * ks * (c1 + c2)
    acc_bound = 4 * (K_ + 2) * 2.0 ** -24 * mag
    err = (got - want).abs()
    assert (err <= 2.0 ** -9 * mag + acc_bound).all(), f"max err / bound {float((err / (2.0 ** -9 * mag + acc_bound)).max()):.3f}"
    seen = conv_ref(tf32_trunc(cpu(x1)), None if x2 is None else tf32_trunc(cpu(x2)), tf32_trunc(cpu(w)), ks, cpu(bias), cpu(r1), cpu(r2))
    err_seen = (got - seen).abs()
    assert (err_seen <= acc_bound).all(), f"vs truncated operands: max err / bound {float((err_seen / acc_bound).max()):.3f}"
    assert float(err.max()) > 4 * float(err_seen.max()), "no tf32 rounding visible: did the fp32 kernel run?"


def test_conv_tf32_refusals():
    L, p = N.lib(), N.ptr
    x = torch.zeros(1, 4, 4, 8, device=DEV)
    w = torch.zeros(8, 9, 8, device=DEV)
    out = torch.empty(1, 4, 4, 8, device=DEV)
    call = lambda c1, ks, rc1=0, r1=None: L.kdb_unet_conv_tf32(p(x), c1, None, 0, p(w), None, r1, rc1, None, p(out), 1, 4, 4, 8, ks, N.stream())
    assert call(8, 2) == -1
    assert call(6, 3) == -4
    assert call(8, 3, 4, p(x)) == -1          # a split residual without r2
    assert call(8, 3) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------
# the engine at tf32
# ------------------------------------------------------------------------------------------------------------------------------

def at_tf32(model):
    model.set_precision("tf32")
    assert model.resolved_precision() == N.PREC_TF32
    return model


@pytest.mark.parametrize("name", sorted(META))
def test_denoiser_within_the_tf32_budget(name):
    """B = 3 at (sigma_min, 1, sigma_max), with and without aug_cond, against the reference's fp32 recording"""
    _, _, model, den = build(name)
    at_tf32(model)
    z = load_npz(f"unet_{name}.npz")
    x, sig, aug = z["x"].to(DEV), z["sigma"].to(DEV), z["aug_cond"].to(DEV)
    for key, kw in (("denoised", {}), ("denoised_aug", dict(aug_cond=aug))):
        err, budget = rel_l2(den(x, sig, **kw), z[key]), BUDGET[f"{name}.{key}"]
        assert 0 < err <= 2 * budget, f"{name} {key}: rel_l2 {err:.3e} vs 2 x the reference's tf32 deviation {budget:.3e}"


@pytest.mark.parametrize("name", sorted(EDGES))
def test_edge_denoiser_within_the_tf32_budget(name):
    _, _, model, den, z = edge(name)
    at_tf32(model)
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    for key in (k for k in VARIANTS if k in z):
        err, budget = rel_l2(den(x, sig, **device_kwargs(z, key)), z[key]), BUDGET[f"edge_{name}.{key}"]
        assert err <= 2 * budget, f"{name} {key}: rel_l2 {err:.3e} vs 2 x the reference's tf32 deviation {budget:.3e}"


def test_heun_trajectory_within_the_tf32_budget():
    _, _, model, den = build("mnist")
    at_tf32(model)
    z = load_npz("unet_mnist.npz")
    got = K.sampling.sample_heun(den, z["heun_x"].to(DEV), z["heun_sigmas"].to(DEV), disable=True)
    err, budget = rel_l2(got, z["heun"]), BUDGET["mnist.heun10"]
    assert err <= 2 * budget, f"heun-10: rel_l2 {err:.3e} vs 2 x the reference's tf32 deviation {budget:.3e}"


# ------------------------------------------------------------------------------------------------------------------------------
# the attention
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,h,w,nh", [(3, 7, 7, 1), (2, 8, 8, 8), (1, 16, 16, 4), (3, 16, 16, 2), (2, 32, 32, 3), (1, 5, 13, 1)],
                         ids=lambda v: str(v))
def test_attention_tf32_against_float64(B, h, w, nh):
    """|got - exact| <= (2 (2^-9 max_j sum_d |q_d k_jd| + 2^-10) + 2^-10) max_j |v_jd| + 2^-20, element by element: q and k truncated
    move each logit by at most 2^-9 sum |q k|, truncated P moves each probability by 2^-10 relative, truncated v by 2^-10 relative."""
    T, C = h * w, nh * 64
    g = torch.Generator().manual_seed(T + nh)
    qkv = torch.randn(B, T, 3 * C, generator=g)
    qkv[..., :C] *= 0.25                                # logits of a few units
    got = N.unet_attention_tf32(qkv.to(DEV), h, w, nh).cpu().double()
    q, k, v = (qkv.double()[..., i * C:(i + 1) * C].view(B, T, nh, 64).transpose(1, 2) for i in range(3))
    want = torch.softmax(q @ k.transpose(-2, -1), dim=-1) @ v
    qk = q.abs() @ k.abs().transpose(-2, -1)
    vmax = v.abs().amax(dim=-2, keepdim=True)
    bound = (2 * (2.0 ** -9 * qk.amax(-1, keepdim=True) + 2.0 ** -10) + 2.0 ** -10) * vmax + 2.0 ** -20
    err = (got.view(B, T, nh, 64).transpose(1, 2) - want).abs()
    assert (err <= bound).all(), f"max err / bound {float((err / bound).max()):.3f}"
    assert float(err.max()) > 1e-6, "no tf32 rounding visible"


def test_attention_tf32_refusals():
    L, p = N.lib(), N.ptr
    qkv = torch.zeros(1, 16, 3 * 64, device=DEV)
    out = torch.empty(1, 16, 64, device=DEV)
    for code, e, fast in ((N.ATTN_SHIFTED_WINDOW, 64, 0), (N.ATTN_NEIGHBORHOOD, 64, 0), (N.ATTN_GLOBAL, 32, 0), (N.ATTN_GLOBAL, 64, 1)):
        assert L.kdb_attention(N.PREC_TF32, fast, p(qkv), p(out), 1, 4, 4, 64 // e, e, code, 0, 0, None, N.stream()) == -2
    assert L.kdb_attention(N.PREC_TF32, 0, p(qkv), p(out), 1, 4, 4, 1, 64, N.ATTN_GLOBAL, 0, 0, None, N.stream()) == 0
    torch.cuda.synchronize()


def test_other_head_sizes_keep_attn_generic():
    """odd_nonsquare attends at d_head 68, 96 and 36: at tf32 its attention runs on attn_generic, its convolutions on the tensor cores"""
    _, _, model, den, z = edge("odd_nonsquare")
    at_tf32(model)
    with N.profile() as p:
        den(z["x"].to(DEV), z["sigma"].to(DEV))
    assert "unet_attn_tf32" not in p.by_family and p.by_family["attn_generic"][0] > 0
    assert "unet_conv" not in p.by_family and p.by_family["unet_conv_tf32"][0] > 0


# ------------------------------------------------------------------------------------------------------------------------------
# every stage
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["mnist", "cifar10"])
def test_every_stage_against_the_tf32_oracle(name, monkeypatch):
    """Each debug tap at tf32 against the oracle's float64 stage with the engine's tf32 operand rounding, fed the engine's own tapped input:
    rel_l2 <= 2^-9 (the two can differ where a value lies within float64-vs-fp32 noise of a tf32 boundary, and in the attention where the
    engine truncates P against the running rather than the final maximum -- each a change of at most one tf32 ulp, 2^-10 relative)"""
    cfg, sd, model, _ = build(name)
    at_tf32(model)
    mcfg = cfg["model"]
    B, (H, W) = 2, mcfg["input_size"]
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, mcfg["input_channels"], H, W, generator=g).to(DEV)
    sig = torch.tensor([0.7, 9.0], device=DEV)
    aug = (torch.randn(B, 9, generator=g) * 0.5).to(DEV)
    eng = unet_engine(model, mcfg)
    cond = eng.conditioning(sig, aug)
    sd64 = {k: v.double() for k, v in sd.items()}
    c64 = U.mapping(sd64, sig.cpu().double(), oracle_mapping_cond(mcfg, B, aug.cpu().double()))
    tf32_oracle(monkeypatch, sd64)

    def run_tap(tap, level, c):
        buf = eng.arm_tap(tap, 1 << 24, x.device)
        eng.forward(x, sig, cond, eng.cond_stride, 0.0, N.PREC_TF32)
        h, w = U.level_hw(mcfg, H, W, level)
        assert eng.tap_count() == B * h * w * c, (tap, eng.tap_count())
        return buf[: B * h * w * c].view(B, h, w, c).permute(0, 3, 1, 2).cpu().double()

    outs = {"patch_in": run_tap("patch_in", 0, mcfg["channels"][0])}
    for tap, (src, op, skip, level) in U.stage_plan(mcfg).items():
        inp = outs[src] if skip is None else torch.cat([outs[src], outs[skip]], dim=1)
        want = U.stage_op(sd64, op, inp, c64)
        got = run_tap(tap, level, want.shape[1])
        assert rel_l2(got, want) <= 2.0 ** -9, f"{name} stage {tap}: rel_l2 {rel_l2(got, want):.3e}"
        outs[tap] = got


def test_routes_and_fp32_untouched():
    """At tf32 every convolution launches as unet_conv_tf32 and every attention as unet_attn_tf32, none as unet_conv or attn_generic; at
    fp32 the reverse, and the fp32 output is the same bits before and after tf32 calls on the same model"""
    _, _, model, den = build("cifar10")
    g = torch.Generator().manual_seed(4)
    x = (torch.randn(2, 3, 32, 32, generator=g) * 5).to(DEV)
    sig = torch.tensor([0.5, 20.0], device=DEV)
    model.set_precision("fp32")
    a = den(x, sig)
    with N.profile() as p32:
        den(x, sig)
    at_tf32(model)
    with N.profile() as p:
        t = den(x, sig)
    model.set_precision("fp32")
    b = den(x, sig)
    assert torch.equal(a, b), "a tf32 call changed the fp32 route"
    assert "unet_conv" not in p.by_family and p.by_family["unet_conv_tf32"][0] == p32.by_family["unet_conv"][0]
    assert "attn_generic" not in p.by_family and p.by_family["unet_attn_tf32"][0] == p32.by_family["attn_generic"][0]
    assert "unet_conv_tf32" not in p32.by_family and "unet_attn_tf32" not in p32.by_family
    tf32_names = {"unet_conv_tf32", "unet_attn_tf32"}
    assert {f: c for f, (c, _) in p.by_family.items() if f not in tf32_names} == \
        {f: c for f, (c, _) in p32.by_family.items() if f not in ("unet_conv", "attn_generic")}
    assert not torch.equal(a, t)


def test_deterministic_and_batch_independent_at_tf32():
    """B = 3 mnist (784 pixels per image: the 7x7 level packs two images per M tile) and B = 4 cifar10"""
    for name, B in (("mnist", 3), ("cifar10", 4)):
        _, _, model, den = build(name)
        at_tf32(model)
        H, W = META[name]["config"]["model"]["input_size"]
        g = torch.Generator().manual_seed(9)
        x = (torch.randn(B, META[name]["config"]["model"]["input_channels"], H, W, generator=g) * 5).to(DEV)
        sig = torch.linspace(0.1, 40.0, B, device=DEV)
        aug = (torch.randn(B, 9, generator=g) * 0.5).to(DEV)
        a, b = den(x, sig, aug_cond=aug), den(x, sig, aug_cond=aug)
        assert torch.equal(a, b), f"{name}: two calls differ"
        for i in range(B):
            assert torch.equal(den(x[i:i + 1], sig[i:i + 1], aug_cond=aug[i:i + 1]), a[i:i + 1]), f"{name}: image {i} depends on its batch"


def test_fp32_and_tf32_calls_get_separate_graphs():
    _, _, model, den = build("mnist")
    z = load_npz("unet_mnist.npz")
    S = K.sampling
    S.clear_graph_cache()
    x, sigmas = z["heun_x"].to(DEV), z["heun_sigmas"].to(DEV)
    model.set_precision("fp32")
    a = S.sample_heun(den, x, sigmas, disable=True)
    assert len(S._graph_cache) == 1
    at_tf32(model)
    t = S.sample_heun(den, x, sigmas, disable=True)
    assert len(S._graph_cache) == 2, "the tf32 call replayed the fp32 graph"
    model.set_precision("fp32")
    assert torch.equal(S.sample_heun(den, x, sigmas, disable=True), a)
    assert len(S._graph_cache) == 2
    assert not torch.equal(a, t)


def test_tf32_refused_outside_the_unet():
    _, _, model, _ = build("mnist")
    eng = model.inner_model.engine(augment=True)
    L, p = N.lib(), N.ptr
    assert L.kdb_unet_workspace_bytes(eng._h, N.PREC_TF32, 2, 28, 28) == L.kdb_unet_workspace_bytes(eng._h, N.PREC_FP32, 2, 28, 28) > 0
    meta = json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())
    cfg = K.config.load_config(meta["config"])
    from oracle.fixtures import synth_sd
    inner = K.config.make_model(cfg)
    inner.load_state_dict(synth_sd(meta["shapes"], 1))
    inner = inner.to(DEV).eval()
    teng = inner.engine()
    assert L.kdb_model_workspace_bytes(teng._h, N.PREC_TF32, 1, 28, 28) == 0
    ws = torch.empty(teng.workspace_bytes(N.PREC_FP32, 1, 28, 28), dtype=torch.uint8, device=DEV)
    xm = torch.zeros(1, 1, 28, 28, device=DEV)
    sig = torch.ones(1, device=DEV)
    cond = teng.conditioning(sig, class_cond=torch.zeros(1, dtype=torch.long, device=DEV))
    assert L.kdb_model_forward(teng._h, N.PREC_TF32, 1, 28, 28, p(xm), p(sig), 1.0, p(cond), 0, p(torch.empty_like(xm)), p(ws), ws.numel(),
                               N.stream()) == -2
    torch.cuda.synchronize()
