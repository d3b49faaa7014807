"""The image_v1 U-Net kernels past the four reference configs, on the H100.

- kdb_unet_conv, the engine's convolution on its own: bit for bit against float64 torch conv2d on dyadic operands (every partial sum is
  exact in any order, so one wrong tap, channel, row or column fails), at shapes with N and M tails, nearly all-padding images, two
  sources and the split residual; element by element within an error bound on normal operands; the grid-row limit refused.
- The edge configs of oracle/make_golden_unet.py (odd widths, GroupNorm groups of 34 and 36, d_head 36 / 68 / 96, non-square and odd grids,
  patch_size 2 with skip_stages 1, mapping_cond with and without the augment wrapper, the identity skip over a concat, the variance
  channel): the whole conditioning row, every stage, the whole denoiser against the reference's recording and the oracle.
- Determinism and batch independence where conv tiles straddle images; the refusals of widths and grids the kernels cannot run.
"""
import json

import pytest
import torch
from torch.nn import functional as F

import k_diffusion as K
from conftest import GOLDEN, assert_close, load_npz
from oracle import unet_oracle as U
from oracle.fixtures import synth_sd
from test_gpu_unet import build, check_every_stage, oracle_mapping_cond, unet_engine
from test_unet_edges_host import VARIANTS, variant_kwargs

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
EDGES = json.loads((GOLDEN / "unet_edges.json").read_text())
NAMES = sorted(EDGES)
DEV = "cuda"
N = K._native
GUARD = 64          # NaN floats past the end of every conv output, which the kernel must leave alone


# ------------------------------------------------------------------------------------------------------------------------------
# kdb_unet_conv
# ------------------------------------------------------------------------------------------------------------------------------

def conv_ref(x1, x2, w, ks, bias, r1, r2):
    """float64 restatement of kdb_unet_conv on token-major operands: torch conv2d (zero padding ks // 2) on the channel concatenation"""
    x = x1 if x2 is None else torch.cat([x1, x2], dim=-1)
    Nn, Ct = w.shape[0], x.shape[-1]
    wt = w.double().view(Nn, ks, ks, Ct).permute(0, 3, 1, 2)                 # tap-major [N, ks*ks, C] -> [N, C, ks, ks]
    y = F.conv2d(x.double().permute(0, 3, 1, 2), wt, None if bias is None else bias.double(), padding=ks // 2).permute(0, 2, 3, 1)
    if r1 is not None:
        y = y + (r1 if r2 is None else torch.cat([r1, r2], dim=-1)).double()
    return y


def run_conv(x1, w, ks, x2=None, bias=None, r1=None, r2=None):
    """kdb_unet_conv into a NaN-filled buffer GUARD floats longer than the output: -> output; asserts it fully written, the guard untouched"""
    B, h, wd, _ = x1.shape
    n = B * h * wd * w.shape[0]
    buf = torch.full((n + GUARD,), float("nan"), device=DEV)
    out = N.unet_conv(x1, w, ks, x2=x2, bias=bias, r1=r1, r2=r2, out=buf[:n].view(B, h, wd, w.shape[0]))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all(), "an output element was not written"
    assert torch.isnan(buf[n:]).all(), "the kernel wrote past the end of its output"
    return out


def dyadic(g, shape, den, lo=-3, hi=3):
    return (torch.randint(lo, hi + 1, shape, generator=g).float() / den).to(DEV)


# (B, H, W, c1, c2, N, ks, residual): residual None, "r1" (rc1 = N) or an int rc1 (r1 with rc1 channels, r2 with the rest)
CONV_CASES = [
    (2, 1, 1, 8, 0, 16, 3, None),              # every neighbour of the single pixel is padding
    (3, 2, 7, 12, 0, 20, 3, "r1"),            # two rows: each pixel has a padded row above or below
    (3, 5, 9, 36, 0, 68, 3, "r1"),            # N tail (68 = 64 + 4), M tail (135 = 2 * 64 + 7), K-blocks straddling taps (Ct = 36)
    (3, 6, 10, 20, 12, 36, 1, None),          # two sources with c1 % 16 == 4: a k-block holds channels of both
    (2, 8, 8, 68, 68, 64, 3, 28),             # two sources under a 3x3 kernel, the split residual at rc1 = 28
    (1, 33, 65, 16, 0, 130, 3, None),         # N = 130 (three column tiles, the last of two), 33 x 65 grid, M = 2145
    (4, 7, 3, 4, 0, 4, 3, "r1"),              # the narrowest operands: Ct = N = 4
]


@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "B{}_{}x{}_c{}+{}_N{}_k{}_r{}".format(*c))
def test_conv_exact_on_dyadic_operands(case, with_bias):
    B, H, W, c1, c2, Nn, ks, res = case
    g = torch.Generator().manual_seed(CONV_CASES.index(case))
    x1 = dyadic(g, (B, H, W, c1), 4)
    x2 = dyadic(g, (B, H, W, c2), 4) if c2 else None
    w = dyadic(g, (Nn, ks * ks, c1 + c2), 8)
    bias = dyadic(g, (Nn,), 4, -8, 8) if with_bias else None
    r1 = r2 = None
    if res == "r1":
        r1 = dyadic(g, (B, H, W, Nn), 2)
    elif res is not None:
        r1, r2 = dyadic(g, (B, H, W, res), 2), dyadic(g, (B, H, W, Nn - res), 2)
    got = run_conv(x1, w, ks, x2, bias, r1, r2)
    want = conv_ref(x1.cpu(), None if x2 is None else x2.cpu(), w.cpu(), ks, None if bias is None else bias.cpu(),
                    None if r1 is None else r1.cpu(), None if r2 is None else r2.cpu())
    assert torch.equal(want.float().double(), want), "operands too large for an exact fp32 sum"
    bad = got.cpu().double() != want
    assert not bad.any(), f"{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()} (b, y, x, n)"


@pytest.mark.parametrize("case", [(3, 5, 9, 36, 0, 68, 3, 28), (2, 12, 20, 64, 32, 96, 3, None), (3, 6, 10, 20, 12, 36, 1, "r1")],
                         ids=lambda c: "B{}_{}x{}_c{}+{}_N{}_k{}_r{}".format(*c))
def test_conv_random_operands_within_the_fp32_error_bound(case):
    """|got - exact| <= 4 (K + 2) 2^-24 (|A| conv |W| + |bias| + |residual|) element by element"""
    B, H, W, c1, c2, Nn, ks, res = case
    g = torch.Generator().manual_seed(11)
    rn = lambda *s: torch.randn(*s, generator=g).to(DEV)
    x1, x2, w, bias = rn(B, H, W, c1), rn(B, H, W, c2) if c2 else None, rn(Nn, ks * ks, c1 + c2) * 0.2, rn(Nn)
    r1 = r2 = None
    if res == "r1":
        r1 = rn(B, H, W, Nn)
    elif res is not None:
        r1, r2 = rn(B, H, W, res), rn(B, H, W, Nn - res)
    got = run_conv(x1, w, ks, x2, bias, r1, r2).cpu().double()
    cpu = lambda t: None if t is None else t.cpu()
    want = conv_ref(cpu(x1), cpu(x2), cpu(w), ks, cpu(bias), cpu(r1), cpu(r2))
    mag = conv_ref(cpu(x1).abs(), cpu(x2).abs() if x2 is not None else None, cpu(w).abs(), ks, cpu(bias).abs(),
                   None if r1 is None else cpu(r1).abs(), None if r2 is None else cpu(r2).abs())
    K_ = ks * ks * (c1 + c2)
    bound = 4 * (K_ + 2) * 2.0 ** -24 * mag
    err = (got - want).abs()
    assert (err <= bound).all(), f"max err / bound {float((err / bound).max()):.3f}"
    assert float((err / bound).max()) > 0, "suspiciously exact"


def test_conv_grid_row_limit():
    """B * H * W = 65535 * 64 pixels (960 x 4369) runs and is checked exactly on dyadic operands; 960 x 4370 is KDB_ERR_BAD_SHAPE, with
    real buffers of that size behind every pointer"""
    L = N.lib()
    g = torch.Generator().manual_seed(3)
    w = dyadic(g, (4, 1, 4), 8)
    x = torch.randint(-3, 4, (1, 960, 4370, 4), device=DEV).float() / 4
    out = torch.full_like(x, float("nan"))
    p = N.ptr
    assert L.kdb_unet_conv(p(x), 4, None, 0, p(w), None, None, 0, None, p(out), 1, 960, 4370, 4, 1, N.stream()) == -4
    assert b"grid" in L.kdb_last_error()
    assert torch.isnan(out).all()
    xs, outs = x.view(-1, 4)[: 960 * 4369].view(1, 960, 4369, 4), out.view(-1, 4)[: 960 * 4369].view(1, 960, 4369, 4)
    assert (960 * 4369) == 65535 * 64
    N.unet_conv(xs, w, 1, out=outs)
    assert torch.equal(outs.double(), xs.double() @ w[:, 0].double().T)
    assert torch.isnan(out.view(-1, 4)[960 * 4369:]).all()


# ------------------------------------------------------------------------------------------------------------------------------
# edge configs
# ------------------------------------------------------------------------------------------------------------------------------

def edge(name):
    cfg, sd, model, den = build(name, EDGES)
    return cfg, sd, model, den, load_npz(f"unet_edge_{name}.npz")


def device_kwargs(z, key):
    return {k: v.to(DEV) for k, v in variant_kwargs(z, key).items()}


def ada_segments(mcfg):
    """(state-dict prefix of the AdaGN mapper, channels) of every AdaGN in execution order: the layout of the conditioning row"""
    segs = []
    for op in (op for _, op, _, _ in U.stage_plan(mcfg).values() if isinstance(op, tuple)):
        kind, p, c_in, c_mid, c_out = op
        segs += [(p + "main.0.", c_in), (p + "main.4.", c_mid)] if kind == "res" else [(p + "norm_in.", c_out)]
    return segs


@pytest.mark.parametrize("name", NAMES)
def test_conditioning_row_against_float64(name):
    """The whole cond row: the mapping net's output against the float64 oracle, and every AdaGN (weight, bias) pair at its offset against
    the float64 mapper of the engine's own mapping output, within the fp32 bound of a length-mapping_out dot product"""
    cfg, sd, model, _, z = edge(name)
    mcfg = cfg["model"]
    eng = unet_engine(model, mcfg)
    mw = mcfg["mapping_out"]
    segs = ada_segments(mcfg)
    ada_total = sum(2 * c for _, c in segs)
    assert eng.cond_stride == (ada_total + mw + 3) // 4 * 4
    sd64 = {k: v.double() for k, v in sd.items()}
    sig = z["sigma"].to(DEV)
    for key in (k for k in VARIANTS if k in z):
        kw = device_kwargs(z, key)
        cond = eng.conditioning(sig, kw.get("aug_cond"), mapping_cond=kw.get("mapping_cond")).cpu().double()
        mc = oracle_mapping_cond(mcfg, 3, *(None if k not in kw else kw[k].cpu().double() for k in ("aug_cond", "mapping_cond")))
        c64 = U.mapping(sd64, sig.cpu().double(), mc)
        assert_close(cond[:, ada_total:ada_total + mw], c64, rtol=1e-4, atol=1e-5, what=f"{name} {key}: mapping net")
        h = cond[:, ada_total:ada_total + mw]
        off = 0
        for p, c in segs:
            W, b = sd64[p + "mapper.weight"], sd64[p + "mapper.bias"]
            want, mag = h @ W.T + b, h.abs() @ W.abs().T + b.abs()
            got = cond[:, off:off + 2 * c]
            err, bound = (got - want).abs(), 2 * (mw + 1) * 2.0 ** -24 * mag
            assert (err <= bound).all(), f"{name} {key}: {p}mapper at offset {off}, max err / bound {float((err / bound).max()):.2f}"
            off += 2 * c


@pytest.mark.parametrize("name", NAMES)
def test_every_stage_of_the_edge_configs(name):
    """every debug tap against the oracle's stage fed the engine's own input, on the recorded inputs with aug_cond and mapping_cond
    wherever the config takes them"""
    cfg, sd, model, _, z = edge(name)
    key = [k for k in VARIANTS if k in z][-1]
    kw = device_kwargs(z, key)
    n = check_every_stage(name, cfg, sd, model, z["x"].to(DEV), z["sigma"].to(DEV), kw.get("aug_cond"), kw.get("mapping_cond"))
    assert n == 1 + len(U.stage_plan(cfg["model"]))


@pytest.mark.parametrize("name", NAMES)
def test_edge_denoiser_matches_reference_and_oracle(name):
    cfg, sd, _, den, z = edge(name)
    oden = U.make_denoiser(sd, cfg["model"])
    x, sig = z["x"].to(DEV), z["sigma"].to(DEV)
    for key in (k for k in VARIANTS if k in z):
        got = den(x, sig, **device_kwargs(z, key))
        assert got.shape == z["x"].shape
        assert_close(got, z[key], what=f"{name} {key} vs reference")
        assert_close(got, oden(z["x"], z["sigma"], **variant_kwargs(z, key)), what=f"{name} {key} vs oracle")


@pytest.mark.parametrize("name", ["odd_nonsquare", "mnist"])
def test_deterministic_and_batch_independent_across_straddling_tiles(name):
    """B = 3 with 720 (20x36) or 784 (28x28) pixels per image: conv row tiles of 64 straddle images.  Two calls are byte-equal and each
    image alone equals its slice of the batch bit for bit."""
    if name == "mnist":
        _, _, _, den = build(name)
        z = load_npz("unet_mnist.npz")
    else:
        _, _, _, den, z = edge(name)
    x, sig, aug = z["x"].to(DEV), z["sigma"].to(DEV), z["aug_cond"].to(DEV)
    assert x.shape[0] == 3 and (x.shape[2] * x.shape[3]) % 64 != 0
    a, b = den(x, sig, aug_cond=aug), den(x, sig, aug_cond=aug)
    assert torch.equal(a, b), "two calls differ"
    for i in range(3):
        alone = den(x[i:i + 1], sig[i:i + 1], aug_cond=aug[i:i + 1])
        assert torch.equal(alone, a[i:i + 1]), f"image {i} depends on its batch"


# ------------------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------------------

def tiny(channels, self_attn, size):
    """a one-level U-Net with synth weights on the GPU: (engine, inputs of one image, Denoiser)"""
    over = dict(input_size=list(size), depths=[1], channels=list(channels), self_attn_depths=list(self_attn), mapping_out=32)
    meta = json.loads(json.dumps(EDGES["variance"]))
    meta["config"]["model"].update(over, has_variance=False)
    cfg = K.config.load_config(meta["config"])
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    model.load_state_dict(synth_sd({k: list(v.shape) for k, v in model.state_dict().items()}, 1))
    model = model.to(DEV)
    eng = model.inner_model.engine(augment=True)
    x = torch.randn(1, 3, *size, generator=torch.Generator().manual_seed(1)).to(DEV)
    return eng, x, K.config.make_denoiser_wrapper(cfg)(model)


def raw_forward(eng, x):
    """kdb_unet_forward through the C ABI -> return code"""
    B, _, H, W = x.shape
    sig = torch.ones(B, device=DEV)
    cond = eng.conditioning(sig)
    need = eng.workspace_bytes(N.PREC_FP32, B, H, W)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.full_like(x, float("nan"))
    p = N.ptr
    rc = N.lib().kdb_unet_forward(eng._h, N.PREC_FP32, B, H, W, p(x), p(sig), 1.0, p(cond), 0, p(out), p(ws), need, N.stream())
    torch.cuda.synchronize()
    return rc


def test_group_norm_indivisible_width_is_refused_by_the_forward():
    """100 channels make 3 AdaGN groups: the reference builds the model and fails at its first group_norm; the engine returns
    KDB_ERR_BAD_SHAPE from the forward and the Python call raises"""
    eng, x, den = tiny([100], [False], (8, 8))
    assert raw_forward(eng, x) == -4
    assert b"3 groups" in N.lib().kdb_last_error()
    with pytest.raises(RuntimeError, match="3 groups"):
        den(x, torch.ones(1, device=DEV))


def test_attention_past_the_shared_memory_budget_is_refused():
    """self-attention over 82 x 82 = 6724 keys at d_head 64 needs more shared memory than attn_generic has: KDB_ERR_UNSUPPORTED where the
    attention would launch, and the same engine still runs a grid that fits"""
    eng, x, den = tiny([64], [True], (82, 82))
    assert raw_forward(eng, x) == -2
    assert b"6724 keys" in N.lib().kdb_last_error()
    small = x[:, :, :8, :8].contiguous()
    assert raw_forward(eng, small) == 0
    assert torch.isfinite(den(small, torch.ones(1, device=DEV))).all()
