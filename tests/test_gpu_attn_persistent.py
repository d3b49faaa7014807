"""The persistent, warp-specialized tensor-core attention kernel (attn_ws_kernel: the shifted-window and global modes of kdb_attention's
bf16 fast path) against an fp32 reference built from the oracle on the same bf16 inputs, with P rounded to bf16 where the kernel rounds
it: p = exp(s - shift) -> bf16, out = (p v) / sum(p), shift = the logit bound when one is given, else the row maximum.

Every case also checks that the NaN-prefilled output is written everywhere, that two runs are byte-equal, and that an image alone and the
same image inside the batch give bit-identical outputs (no work item depends on which CTA runs it, or on its neighbours)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALE = 10.0            # cosine-similarity scale of the test data: |q . k| <= SCALE


def _qkv(B, h, w, nh, seed):
    """qkv [B, h*w, 3*nh*64] bf16 with cosine-normalised q, k (|q| = |k| = sqrt(SCALE)) like the real layer input."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = torch.randn(B, h * w, 3, nh, 64, device=DEV, generator=g)
    t[:, :, :2] = t[:, :, :2] / t[:, :, :2].norm(dim=-1, keepdim=True) * SCALE ** 0.5
    return t.to(torch.bfloat16).reshape(B, h * w, 3 * nh * 64).contiguous()


def _reference(monkeypatch, qkv, h, w, nh, kind, shift, bound):
    """the oracle's window / global attention with its softmax replaced by the kernel's rounding of P"""
    from oracle import kdiff_oracle as O

    def softmax_av_bf16_p(q, k, v, allow=None):
        logits = q @ k.transpose(-1, -2)
        if allow is not None:
            logits = logits.masked_fill(~allow, float("-inf"))
        if bound is None:
            shift_ = logits.amax(-1, keepdim=True)
        else:              # q, k, v here are [B, nh, ...]: the bound of head n on dimension 1
            shift_ = bound.cpu().view(1, nh, *([1] * (logits.dim() - 2)))
        p = torch.exp(logits - shift_).to(torch.bfloat16).float()
        return (p @ v) / p.sum(-1, keepdim=True)

    monkeypatch.setattr(O, "_softmax_av", softmax_av_bf16_p)
    B = qkv.shape[0]
    q, k, v = qkv.float().cpu().view(B, h, w, 3, nh, 64).unbind(3)
    o = O.global_attention(q, k, v) if kind == "global" else O.shifted_window_attention(q, k, v, 8, shift)
    return o.reshape(B, h * w, nh * 64)


def _run(qkv, h, w, nh, kind, shift, bound):
    from k_diffusion import _native as N_
    B = qkv.shape[0]
    out = torch.full((B, h * w, nh * 64), float("nan"), dtype=torch.bfloat16, device=DEV)
    N_.check(N_.lib().kdb_attention(N_.PREC_BF16, 1, N_.ptr(qkv), N_.ptr(out), B, h, w, nh, 64, N_._ATTN_CODE[kind],
                                    8 if kind == "shifted-window" else 0, shift, N_.ptr(bound), N_.stream()))
    torch.cuda.synchronize()
    return out


CASES = [
    # shifted window: B, h, w, nh, shift
    (1, 8, 8, 2, "shifted-window", 0),          # one window
    (1, 8, 8, 2, "shifted-window", 4),          # one window, both seams
    (1, 8, 24, 2, "shifted-window", 4),         # odd window count, h != w
    (2, 24, 8, 4, "shifted-window", 0),
    (1, 16, 16, 2, "shifted-window", 4),        # fewer tiles than SMs
    (3, 48, 40, 4, "shifted-window", 0),        # 180 tiles: an uneven number per CTA
    (3, 48, 40, 4, "shifted-window", 4),
    (32, 32, 32, 4, "shifted-window", 0),       # the cfg2 level-1 shape (256x256 model, batch 32)
    (32, 32, 32, 4, "shifted-window", 4),
    # global: B, h, w, nh (shift 0)
    (1, 8, 16, 2, "global", 0),                 # S = 128: one key block
    (2, 16, 16, 8, "global", 0),                # S = 256
    (32, 16, 16, 8, "global", 0),               # the cfg2 middle-level shape
    (3, 16, 32, 3, "global", 0),                # S = 512, odd head count, 36 tiles
    (1, 32, 64, 1, "global", 0),                # S = 2048: 16 key blocks through the ring of stages
    (16, 32, 32, 16, "global", 0),              # the cfg5 middle-level shape (512x512 model, widths 256/512/1024, batch 16)
    (64, 16, 16, 8, "global", 0),               # the cfg3 middle-level shape (256x256 neighbourhood model, batch 64)
]


@pytest.mark.parametrize("bounded", [True, False], ids=["bounded", "row-max"])
@pytest.mark.parametrize("B,h,w,nh,kind,shift", CASES)
def test_attention_persistent_vs_reference(monkeypatch, B, h, w, nh, kind, shift, bounded):
    qkv = _qkv(B, h, w, nh, seed=B * 1000 + h * w + nh + shift)
    bound = torch.full([nh], SCALE, device=DEV) if bounded else None
    got = _run(qkv, h, w, nh, kind, shift, bound)
    assert not bool(torch.isnan(got).any()), "an output element was not written"
    want = _reference(monkeypatch, qkv, h, w, nh, kind, shift, bound)
    err = (got.float().cpu() - want).abs()
    # bf16 output (2^-9 relative), the summation order of l and P V, and a p whose bf16 rounding flips on the last bit of its logit
    # (2^-8 of its share of the row: visible in the seam windows' 16-key rows)
    tol = 8e-3 * want.abs() + 8e-3
    assert bool((err <= tol).all()), f"max err {float(err.max()):.4g} at {int(err.argmax())}, want {float(want.flatten()[err.argmax()]):.4g}"
    assert float(err.mean()) < 2.5e-3 * float(want.abs().mean()), f"mean err {float(err.mean()):.3g}"   # ~ the bf16 rounding alone
    again = _run(qkv, h, w, nh, kind, shift, bound)
    assert torch.equal(got.view(torch.int16), again.view(torch.int16)), "two runs differ"
    b = B - 1
    alone = _run(qkv[b:b + 1].contiguous(), h, w, nh, kind, shift, bound)
    assert torch.equal(got[b:b + 1].view(torch.int16), alone.view(torch.int16)), "an image alone differs from the same image in the batch"
