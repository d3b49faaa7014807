"""The image_v1 U-Net at the fp16 precision on the H100: kdb_unet_conv_fp16 (every convolution of the engine with fp16 operands), the
fp16 global attention, and the whole denoiser with them.

- The convolution bit for bit against float64 torch conv2d on dyadic operands, which are exact in fp16 and whose every partial sum is exact
  in fp32, over the shape matrix of the tf32 convolution's test; on normal operands within the bound of fp16 operands and fp32
  accumulation; an operand past fp16's range becomes inf.
- The attention (kdb_attention at fp16) against float64 softmax attention, within the bound of its fp16 operands.
- Every stage of mnist and cifar10 against the float64 oracle stage with the engine's fp16 operand rounding, fed the engine's own input,
  with the workspace NaN-filled before each forward.
- The whole denoiser of the four reference configs and the six edge configs, and the mnist Heun-10 trajectory, against the reference's
  fp32 recordings within twice the reference's own fp16 deviation (tests/golden/fp16_budget.json, oracle/make_golden_fp16.py).
- The fp32 and tf32 outputs keep the bits they had before fp16 existed (tests/golden/unet_route_digests.json), before and after fp16
  calls on the same model; routes, determinism, batch independence, separate CUDA graphs per precision, and the refusals.
"""
import hashlib
import json

import pytest
import torch
from torch.nn import functional as F

import k_diffusion as K
from conftest import GOLDEN, load_npz
from oracle import unet_oracle as U
from oracle.make_golden_fp16 import f16_round, f16_sdpa
from test_gpu_unet import META, build, oracle_mapping_cond, unet_engine
from test_gpu_unet_kernels import GUARD, conv_ref, device_kwargs, dyadic, edge
from test_gpu_unet_tf32 import TF32_CASES, cpu, operands, rel_l2
from test_unet_edges_host import VARIANTS

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
BUDGET = json.loads((GOLDEN / "fp16_budget.json").read_text())
DEV = "cuda"
N = K._native


class F16Functional:
    """torch.nn.functional for the oracle with the engine's fp16 arithmetic: every dense conv2d but the listed fp32 ones takes its input
    and weight rounded to fp16 (the depthwise resampling filters stay exact); the attention rounds q, k, v and P."""

    def __init__(self, fp32_weights):
        self._keep = {id(w) for w in fp32_weights}

    def __getattr__(self, name):
        return getattr(F, name)

    def conv2d(self, x, w, *args, **kwargs):
        if id(w) in self._keep or kwargs.get("groups", 1) != 1:
            return F.conv2d(x, w, *args, **kwargs)
        return F.conv2d(f16_round(x), f16_round(w), *args, **kwargs)

    @staticmethod
    def scaled_dot_product_attention(q, k, v, *args, **kwargs):
        return f16_sdpa(q, k, v, *args, **kwargs)


# ------------------------------------------------------------------------------------------------------------------------------
# kdb_unet_conv_fp16
# ------------------------------------------------------------------------------------------------------------------------------

def run_conv_fp16(x1, w, ks, x2=None, bias=None, r1=None, r2=None, finite=True):
    """kdb_unet_conv_fp16 into a NaN-filled buffer GUARD floats longer than the output: -> output; asserts it fully written (finite), the
    guard untouched"""
    B, h, wd, _ = x1.shape
    n = B * h * wd * w.shape[0]
    buf = torch.full((n + GUARD,), float("nan"), device=DEV)
    out = N.unet_conv_fp16(x1, w, ks, x2=x2, bias=bias, r1=r1, r2=r2, out=buf[:n].view(B, h, wd, w.shape[0]))
    torch.cuda.synchronize()
    if finite:
        assert torch.isfinite(out).all(), "an output element was not written"
    assert torch.isnan(buf[n:]).all(), "the kernel wrote past the end of its output"
    return out


@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("case", TF32_CASES, ids=lambda c: "B{}_{}x{}_c{}+{}_N{}_k{}_r{}".format(*c))
def test_conv_fp16_exact_on_dyadic_operands(case, with_bias):
    g = torch.Generator().manual_seed(TF32_CASES.index(case))
    x1, x2, w, r1, r2 = operands(case, lambda shape, den: dyadic(g, shape, den))
    bias = dyadic(g, (case[5],), 4, -8, 8) if with_bias else None
    for t in (x1, x2, w):
        assert t is None or torch.equal(f16_round(t), t), "operand not exact in fp16"
    got = run_conv_fp16(x1, w, case[6], x2, bias, r1, r2)
    want = conv_ref(cpu(x1), cpu(x2), cpu(w), case[6], cpu(bias), cpu(r1), cpu(r2))
    assert torch.equal(want.float().double(), want), "operands too large for an exact fp32 sum"
    bad = got.cpu().double() != want
    assert not bad.any(), f"{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()} (b, y, x, n)"


@pytest.mark.parametrize("case", [(3, 5, 9, 36, 0, 68, 3, 28), (2, 12, 20, 64, 32, 96, 3, None), (3, 6, 10, 20, 12, 36, 1, "r1"),
                                  (2, 16, 16, 128, 128, 256, 3, None), (2, 7, 7, 68, 36, 36, 1, 12)],
                         ids=lambda c: "B{}_{}x{}_c{}+{}_N{}_k{}_r{}".format(*c))
def test_conv_fp16_random_operands_within_the_fp16_error_bound(case):
    """Inputs and weights both rounded to nearest fp16 (relative error <= 2^-11 each, absolute <= 2^-25 in fp16's subnormal range), fp32
    accumulation of K products: |got - exact| <= (2^-10 + 4 (K + 2) 2^-24) (|A| conv |W| + |bias| + |residual|) + 2^-24 (1 conv |W|
    + |A| conv 1).  Against the operands the tensor cores see (both rounded, float64 conv) the error is the accumulation's alone."""
    B, H, W, c1, c2, Nn, ks, res = case
    g = torch.Generator().manual_seed(12)
    x1, x2, w, r1, r2 = operands(case, lambda shape, den: torch.randn(*shape, generator=g).to(DEV) / den * 2)
    bias = torch.randn(Nn, generator=g).to(DEV)
    got = run_conv_fp16(x1, w, ks, x2, bias, r1, r2).cpu().double()
    want = conv_ref(cpu(x1), cpu(x2), cpu(w), ks, cpu(bias), cpu(r1), cpu(r2))
    ab = lambda t: None if t is None else cpu(t).abs()
    mag = conv_ref(ab(x1), ab(x2), ab(w), ks, ab(bias), ab(r1), ab(r2))
    one = lambda t: None if t is None else torch.ones_like(cpu(t))
    sub = conv_ref(one(x1), one(x2), ab(w), ks, None, None, None) + conv_ref(ab(x1), ab(x2), one(w), ks, None, None, None)
    K_ = ks * ks * (c1 + c2)
    acc_bound = 4 * (K_ + 2) * 2.0 ** -24 * mag
    bound = 2.0 ** -10 * mag + acc_bound + 2.0 ** -24 * sub
    err = (got - want).abs()
    assert (err <= bound).all(), f"max err / bound {float((err / bound).max()):.3f}"
    r = lambda t: None if t is None else f16_round(cpu(t))
    seen = conv_ref(r(x1), r(x2), r(w), ks, cpu(bias), cpu(r1), cpu(r2))
    err_seen = (got - seen).abs()
    assert (err_seen <= acc_bound).all(), f"vs rounded operands: max err / bound {float((err_seen / acc_bound).max()):.3f}"
    assert float(err.max()) > 4 * float(err_seen.max()), "no fp16 rounding visible: did the fp32 kernel run?"


def test_conv_fp16_operands_past_the_fp16_range_become_inf():
    """Rounding does not saturate: 65519 rounds to 65504 (the largest fp16), 65520 and beyond to inf, -65520 to -inf"""
    x = torch.zeros(1, 2, 2, 8, device=DEV)
    x[0, 0, 0, 0], x[0, 0, 1, 0], x[0, 1, 0, 3], x[0, 1, 1, 5] = 65519.0, 65520.0, -1e6, 1.0
    w = torch.ones(8, 1, 8, device=DEV)
    out = run_conv_fp16(x, w, 1, finite=False).cpu()
    assert torch.equal(out[0, 0, 0], torch.full((8,), 65504.0))
    assert torch.equal(out[0, 0, 1], torch.full((8,), float("inf")))
    assert torch.equal(out[0, 1, 0], torch.full((8,), float("-inf")))
    assert torch.equal(out[0, 1, 1], torch.ones(8))


def test_conv_fp16_refusals():
    L, p = N.lib(), N.ptr
    x = torch.zeros(1, 4, 4, 8, device=DEV)
    w = torch.zeros(8, 9, 8, dtype=torch.float16, device=DEV)
    out = torch.empty(1, 4, 4, 8, device=DEV)
    call = lambda c1, ks, rc1=0, r1=None, wp=p(w): L.kdb_unet_conv_fp16(p(x), c1, None, 0, wp, None, r1, rc1, None, p(out), 1, 4, 4, 8, ks,
                                                                         N.stream())
    assert call(8, 2) == -1
    assert call(6, 3) == -4
    assert call(8, 3, 4, p(x)) == -1          # a split residual without r2
    assert call(8, 3, wp=None) == -1
    assert call(8, 3) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------
# the attention
# ------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,h,w,nh", [(3, 7, 7, 1), (2, 8, 8, 8), (1, 16, 16, 4), (3, 16, 16, 2), (2, 32, 32, 3), (1, 5, 13, 1)],
                         ids=lambda v: str(v))
def test_attention_fp16_against_float64(B, h, w, nh):
    """|got - exact| <= (2 (2^-10 max_j sum_d |q_d k_jd| + 2^-11) + 2^-11) max_j |v_jd| + T 2^-25 max_j |v_jd| + 2^-20, element by element:
    q and k rounded move each logit by at most 2^-10 sum |q k|, rounded P moves each probability by 2^-11 relative (2^-25 absolute in
    fp16's subnormal range), rounded v by 2^-11 relative.  49, 64, 65, 256 and 1024 keys: 49 and 65 are not multiples of the key block."""
    T, C = h * w, nh * 64
    g = torch.Generator().manual_seed(T + nh)
    qkv = torch.randn(B, T, 3 * C, generator=g)
    qkv[..., :C] *= 0.25                                # logits of a few units
    got = N.unet_attention_fp16(qkv.to(DEV), h, w, nh).cpu().double()
    q, k, v = (qkv.double()[..., i * C:(i + 1) * C].view(B, T, nh, 64).transpose(1, 2) for i in range(3))
    want = torch.softmax(q @ k.transpose(-2, -1), dim=-1) @ v
    qk = q.abs() @ k.abs().transpose(-2, -1)
    vmax = v.abs().amax(dim=-2, keepdim=True)
    bound = (2 * (2.0 ** -10 * qk.amax(-1, keepdim=True) + 2.0 ** -11) + 2.0 ** -11 + T * 2.0 ** -25) * vmax + 2.0 ** -20
    err = (got.view(B, T, nh, 64).transpose(1, 2) - want).abs()
    assert (err <= bound).all(), f"max err / bound {float((err / bound).max()):.3f}"
    assert float(err.max()) > 1e-6, "no fp16 rounding visible"
    # against the float64 attention of the fp16-rounded q, k, v only P's rounding (2^-11 relative on P and on l) and the fp32 sums remain
    q16, k16, v16 = (f16_round(t) for t in (q, k, v))
    want16 = torch.softmax(q16 @ k16.transpose(-2, -1), dim=-1) @ v16
    err16 = (got.view(B, T, nh, 64).transpose(1, 2) - want16).abs()
    bound16 = (2.0 ** -10 + T * 2.0 ** -24) * v16.abs().amax(dim=-2, keepdim=True) + 2.0 ** -20
    assert (err16 <= bound16).all(), f"vs rounded q, k, v: max err / bound {float((err16 / bound16).max()):.3f}"


def test_attention_fp16_refusals():
    L, p = N.lib(), N.ptr
    qkv = torch.zeros(1, 16, 3 * 64, device=DEV)
    out = torch.empty(1, 16, 64, device=DEV)
    for code, e, fast in ((N.ATTN_SHIFTED_WINDOW, 64, 0), (N.ATTN_NEIGHBORHOOD, 64, 0), (N.ATTN_GLOBAL, 32, 0), (N.ATTN_GLOBAL, 64, 1)):
        assert L.kdb_attention(N.PREC_FP16, fast, p(qkv), p(out), 1, 4, 4, 64 // e, e, code, 0, 0, None, N.stream()) == -2
    assert L.kdb_attention(N.PREC_FP16, 0, p(qkv), p(out), 1, 4, 4, 1, 64, N.ATTN_GLOBAL, 0, 0, None, N.stream()) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------
# the engine at fp16
# ------------------------------------------------------------------------------------------------------------------------------

def at_fp16(model):
    model.set_precision("fp16")
    assert model.resolved_precision() == N.PREC_FP16
    return model


@pytest.mark.parametrize("name", sorted(META))
def test_denoiser_within_the_fp16_budget(name):
    """B = 3 at (sigma_min, 1, sigma_max), with and without aug_cond, against the reference's fp32 recording"""
    _, _, model, den = build(name)
    at_fp16(model)
    z = load_npz(f"unet_{name}.npz")
    x, sig, aug = z["x"].to(DEV), z["sigma"].to(DEV), z["aug_cond"].to(DEV)
    for key, kw in (("denoised", {}), ("denoised_aug", dict(aug_cond=aug))):
        err, budget = rel_l2(den(x, sig, **kw), z[key]), BUDGET[f"{name}.{key}"]
        assert 0 < err <= 2 * budget, f"{name} {key}: rel_l2 {err:.3e} vs 2 x the reference's fp16 deviation {budget:.3e}"


@pytest.mark.parametrize("name", sorted(EDGES))
def test_edge_denoiser_within_the_fp16_budget(name):
    _, _, model, den, z = edge(name)
    at_fp16(model)
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    for key in (k for k in VARIANTS if k in z):
        err, budget = rel_l2(den(x, sig, **device_kwargs(z, key)), z[key]), BUDGET[f"edge_{name}.{key}"]
        assert err <= 2 * budget, f"{name} {key}: rel_l2 {err:.3e} vs 2 x the reference's fp16 deviation {budget:.3e}"


def test_heun_trajectory_within_the_fp16_budget():
    _, _, model, den = build("mnist")
    at_fp16(model)
    z = load_npz("unet_mnist.npz")
    got = K.sampling.sample_heun(den, z["heun_x"].to(DEV), z["heun_sigmas"].to(DEV), disable=True)
    err, budget = rel_l2(got, z["heun"]), BUDGET["mnist.heun10"]
    assert err <= 2 * budget, f"heun-10: rel_l2 {err:.3e} vs 2 x the reference's fp16 deviation {budget:.3e}"


@pytest.mark.parametrize("name", ["mnist", "cifar10"])
def test_every_stage_against_the_fp16_oracle(name, monkeypatch):
    """Each debug tap at fp16 against the oracle's float64 stage with the engine's fp16 operand rounding, fed the engine's own tapped input,
    the workspace NaN-filled before every forward (a stage that reads a buffer nothing wrote fails): rel_l2 <= 2^-10 (the two can differ
    where a value lies within float64-vs-fp32 noise of an fp16 rounding boundary, and in the attention where the engine rounds P against
    the running rather than the final maximum -- each a change of at most one fp16 ulp, 2^-11 relative)"""
    cfg, sd, model, _ = build(name)
    at_fp16(model)
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
    monkeypatch.setattr(U, "F", F16Functional([sd64["proj_in.weight"], sd64["proj_out.weight"]]))

    def run_tap(tap, level, c):
        eng._workspace(N.PREC_FP16, B, H, W, x.device).fill_(0xFF)       # every float of it a NaN
        buf = eng.arm_tap(tap, 1 << 24, x.device)
        eng.forward(x, sig, cond, eng.cond_stride, 0.0, N.PREC_FP16)
        h, w = U.level_hw(mcfg, H, W, level)
        assert eng.tap_count() == B * h * w * c, (tap, eng.tap_count())
        return buf[: B * h * w * c].view(B, h, w, c).permute(0, 3, 1, 2).cpu().double()

    outs = {"patch_in": run_tap("patch_in", 0, mcfg["channels"][0])}
    assert torch.isfinite(outs["patch_in"]).all()
    for tap, (src, op, skip, level) in U.stage_plan(mcfg).items():
        inp = outs[src] if skip is None else torch.cat([outs[src], outs[skip]], dim=1)
        want = U.stage_op(sd64, op, inp, c64)
        got = run_tap(tap, level, want.shape[1])
        assert torch.isfinite(got).all(), f"{name} stage {tap}: non-finite output"
        assert rel_l2(got, want) <= 2.0 ** -10, f"{name} stage {tap}: rel_l2 {rel_l2(got, want):.3e}"
        outs[tap] = got


def test_routes():
    """At fp16 every convolution launches as unet_conv_fp16 and every d_head-64 attention as unet_attn_fp16, as many as the tf32 route
    launches of its own; every other kernel family runs as at tf32.  odd_nonsquare (d_head 68, 96 and 36) keeps attn_generic."""
    _, _, model, den = build("cifar10")
    g = torch.Generator().manual_seed(4)
    x = (torch.randn(2, 3, 32, 32, generator=g) * 5).to(DEV)
    sig = torch.tensor([0.5, 20.0], device=DEV)
    model.set_precision("tf32")
    den(x, sig)
    with N.profile() as p32:
        den(x, sig)
    at_fp16(model)
    den(x, sig)
    with N.profile() as p:
        den(x, sig)
    assert p.by_family["unet_conv_fp16"][0] == p32.by_family["unet_conv_tf32"][0] > 0
    assert p.by_family["unet_attn_fp16"][0] == p32.by_family["unet_attn_tf32"][0] > 0
    swap = {"unet_conv_fp16": "unet_conv_tf32", "unet_attn_fp16": "unet_attn_tf32"}
    assert {swap.get(f, f): c for f, (c, _) in p.by_family.items()} == {f: c for f, (c, _) in p32.by_family.items()}
    _, _, model, den, z = edge("odd_nonsquare")
    at_fp16(model)
    with N.profile() as p:
        den(z["x"].to(DEV), z["sigma"].to(DEV))
    assert "unet_attn_fp16" not in p.by_family and p.by_family["attn_generic"][0] > 0
    assert "unet_conv" not in p.by_family and p.by_family["unet_conv_fp16"][0] > 0


def test_deterministic_and_batch_independent_at_fp16():
    """B = 3 mnist (784 pixels per image: the 7x7 level packs two images per M tile) and B = 4 cifar10"""
    for name, B in (("mnist", 3), ("cifar10", 4)):
        _, _, model, den = build(name)
        at_fp16(model)
        H, W = META[name]["config"]["model"]["input_size"]
        g = torch.Generator().manual_seed(9)
        x = (torch.randn(B, META[name]["config"]["model"]["input_channels"], H, W, generator=g) * 5).to(DEV)
        sig = torch.linspace(0.1, 40.0, B, device=DEV)
        aug = (torch.randn(B, 9, generator=g) * 0.5).to(DEV)
        a, b = den(x, sig, aug_cond=aug), den(x, sig, aug_cond=aug)
        assert torch.equal(a, b), f"{name}: two calls differ"
        for i in range(B):
            assert torch.equal(den(x[i:i + 1], sig[i:i + 1], aug_cond=aug[i:i + 1]), a[i:i + 1]), f"{name}: image {i} depends on its batch"


# ------------------------------------------------------------------------------------------------------------------------------
# the fp32 and tf32 routes keep their bits
# ------------------------------------------------------------------------------------------------------------------------------

def sha256(t):
    return hashlib.sha256(t.detach().float().contiguous().cpu().numpy().tobytes()).hexdigest()


def route_digests(precisions=("fp32", "tf32")):
    """SHA-256 of the float32 output bytes of the cifar10 denoiser (its recorded x, sigma and aug_cond) and of the odd_nonsquare edge
    denoiser (its recorded x and sigma), one model of each called at the precisions in turn -> {"<config>.<precision>": [digest of each
    call at that precision]}"""
    out = {}
    _, _, model, den = build("cifar10")
    z = load_npz("unet_cifar10.npz")
    for prec in precisions:
        model.set_precision(prec)
        out.setdefault(f"cifar10.{prec}", []).append(sha256(den(z["x"].to(DEV), z["sigma"].to(DEV), aug_cond=z["aug_cond"].to(DEV))))
    _, _, model, den, z = edge("odd_nonsquare")
    for prec in precisions:
        model.set_precision(prec)
        out.setdefault(f"edge_odd_nonsquare.{prec}", []).append(sha256(den(z["x"].to(DEV), z["sigma"].to(DEV))))
    return out


def test_fp32_and_tf32_outputs_keep_the_bits_recorded_before_fp16():
    """The digests in tests/golden/unet_route_digests.json were recorded on the build before the fp16 precision was added.  Each model runs
    fp32 and tf32, then fp16, then fp32 and tf32 again: every one of those fp32 and tf32 outputs keeps the recorded bits (a tf32 kernel
    instantiation that changed, or an fp16 call that disturbed shared state, fails)."""
    want = json.loads((GOLDEN / "unet_route_digests.json").read_text())["digests"]
    got = route_digests(("fp32", "tf32", "fp16", "fp32", "tf32"))
    for key, digest in want.items():
        assert got[key] == [digest, digest], key
    assert len(set(got["cifar10.fp16"])) == 1 and got["cifar10.fp16"][0] not in want.values()


def test_fp16_calls_interleaved_with_fp32_and_tf32_keep_their_bits():
    _, _, model, den = build("cifar10")
    z = load_npz("unet_cifar10.npz")
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    outs = {}
    for prec in ("fp32", "tf32", "fp16"):
        model.set_precision(prec)
        outs[prec] = den(x, sig)
    for prec in ("fp16", "tf32", "fp32", "fp16"):
        model.set_precision(prec)
        assert torch.equal(den(x, sig), outs[prec]), prec
    assert not torch.equal(outs["fp16"], outs["tf32"]) and not torch.equal(outs["fp16"], outs["fp32"])


# ------------------------------------------------------------------------------------------------------------------------------
# graphs and refusals
# ------------------------------------------------------------------------------------------------------------------------------

def test_fp16_and_tf32_calls_get_separate_graphs():
    _, _, model, den = build("mnist")
    z = load_npz("unet_mnist.npz")
    S = K.sampling
    S.clear_graph_cache()
    x, sigmas = z["heun_x"].to(DEV), z["heun_sigmas"].to(DEV)
    model.set_precision("tf32")
    t = S.sample_heun(den, x, sigmas, disable=True)
    assert len(S._graph_cache) == 1
    at_fp16(model)
    h = S.sample_heun(den, x, sigmas, disable=True)
    assert len(S._graph_cache) == 2, "the fp16 call replayed the tf32 graph"
    model.set_precision("fp32")
    f = S.sample_heun(den, x, sigmas, disable=True)
    assert len(S._graph_cache) == 3
    model.set_precision("tf32")
    assert torch.equal(S.sample_heun(den, x, sigmas, disable=True), t)
    at_fp16(model)
    assert torch.equal(S.sample_heun(den, x, sigmas, disable=True), h)
    assert len(S._graph_cache) == 3
    assert not torch.equal(h, t) and not torch.equal(h, f)


def test_fp16_refused_outside_the_unet():
    _, _, model, _ = build("mnist")
    eng = model.inner_model.engine(augment=True)
    L, p = N.lib(), N.ptr
    assert L.kdb_unet_workspace_bytes(eng._h, N.PREC_FP16, 2, 28, 28) == L.kdb_unet_workspace_bytes(eng._h, N.PREC_FP32, 2, 28, 28) > 0
    assert L.kdb_unet_workspace_bytes(eng._h, N.PREC_FP16, 2, 28, 28) == L.kdb_unet_workspace_bytes(eng._h, N.PREC_TF32, 2, 28, 28)
    assert L.kdb_unet_workspace_bytes(eng._h, N.PREC_BF16, 2, 28, 28) == -2
    meta = json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())
    cfg = K.config.load_config(meta["config"])
    from oracle.fixtures import synth_sd
    inner = K.config.make_model(cfg)
    inner.load_state_dict(synth_sd(meta["shapes"], 1))
    inner = inner.to(DEV).eval()
    teng = inner.engine()
    assert L.kdb_model_workspace_bytes(teng._h, N.PREC_FP16, 1, 28, 28) == 0
    ws = torch.empty(teng.workspace_bytes(N.PREC_FP32, 1, 28, 28), dtype=torch.uint8, device=DEV)
    xm = torch.zeros(1, 1, 28, 28, device=DEV)
    sig = torch.ones(1, device=DEV)
    cond = teng.conditioning(sig, class_cond=torch.zeros(1, dtype=torch.long, device=DEV))
    assert L.kdb_model_forward(teng._h, N.PREC_FP16, 1, 28, 28, p(xm), p(sig), 1.0, p(cond), 0, p(torch.empty_like(xm)), p(ws), ws.numel(),
                               N.stream()) == -2
    torch.cuda.synchronize()
