"""The fused attention block of a 128-wide shifted-window level (csrc/tc_attn_block.cuh) against an fp32 torch reference built from the
oracle, and the launch accounting that matches a profile's GEMM launches to shapes."""
import json

import pytest
import torch

from conftest import ROOT

DEV = "cuda"


def _cfg2():
    import k_diffusion as K
    return K.config.load_config(json.loads((ROOT / "tests/golden/cfg2_sw256_shapes.json").read_text())["config"])["model"]


def test_launch_layers_cfg2_counts_each_level0_attention_block_as_one_launch():
    from k_diffusion.models import flops
    mcfg = _cfg2()
    seq = flops.launch_layers(mcfg, 32)
    assert len(seq) == 44                       # 48 with the level-0 qkv and out_proj as separate launches (four blocks)
    assert sum(m for *_, m in seq) == flops.linear_macs(mcfg, 32)
    fused = [s for s in seq if "attn (" in s[0]]
    assert len(fused) == 4 and all(M == 32 * 64 * 64 and N == 384 and K == 128 for _, M, N, K, _ in fused)
    # attention_macs: only the levels whose attention still runs in the stand-alone kernel (level 1 and the middle level)
    assert flops.fused_attention_levels(mcfg) == {0}
    full = sum(d * (1 if l == 2 else 2) * (C // 64) * (64 >> l) ** 2 * (64 if l < 2 else (16 * 16)) * 2 * 64
               for l, (d, C) in enumerate(zip(mcfg["depths"], mcfg["widths"])))
    level0 = 2 * 2 * 2 * 64 * 64 * 64 * 2 * 64
    assert flops.attention_macs(mcfg, 1) == full - level0


def _reference(x, w_qkv, w_out, theta, scale, shift, ss):
    """fp32 torch: x + out_proj(shifted_window_attention(rope(cos_sim(q, k)), v)), q k v = (x / rms) Wqkv^T; q, k, v and the attention
    output rounded to bf16 where the kernel rounds them."""
    from oracle import kdiff_oracle as O
    B, h, w, C = x.shape
    xf = x.float().cpu()
    xn = xf * torch.rsqrt(ss.cpu()[:, :1].view(B, h, w, 1) / C + 1e-6)
    qkv = (xn @ w_qkv.float().cpu().T).view(B, h, w, 3, 2, 64)
    q, k, v = qkv.unbind(3)
    q, k = O.cosine_sim_scale(q, k, scale.cpu())
    th = theta.cpu()
    q, k = O.apply_rope(q, th), O.apply_rope(k, th)
    bf = lambda t: t.to(torch.bfloat16).float()
    o = O.shifted_window_attention(bf(q), bf(k), bf(v), 8, shift)
    return xf + bf(o.reshape(B, h, w, C)) @ w_out.float().cpu().T


@pytest.mark.gpu
@pytest.mark.parametrize("B,h,w,shift", [
    (1, 8, 8, 0), (1, 8, 8, 4),                  # one window: the second warpgroup of the only tile idles
    (3, 8, 8, 4),                                # odd number of windows
    (2, 16, 24, 0), (2, 16, 24, 4),              # h != w, even
    (1, 24, 16, 4), (3, 16, 40, 0),              # h != w, odd (3 x 10 windows = 15 tiles)
    (32, 64, 64, 0), (32, 64, 64, 4)])           # the level-0 shape of the 256x256 model at batch 32
def test_attn_block_matches_reference(B, h, w, shift):
    from k_diffusion import _native as N_
    from oracle import kdiff_oracle as O
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + h * 10 + w + shift)
    C = 128
    x = (torch.randn(B, h, w, C, device=DEV, generator=g) * (0.5 + torch.rand(B, h, w, 1, device=DEV, generator=g) * 3)).to(torch.bfloat16)
    w_qkv = (torch.randn(3 * C, C, device=DEV, generator=g) / C ** 0.5).to(torch.bfloat16)
    w_out = (torch.randn(C, C, device=DEV, generator=g) / C ** 0.5).to(torch.bfloat16)
    scale = torch.tensor([10.0, 6.5], device=DEV)
    theta = O.rope_theta(O.make_axial_pos(h, w), O.rope_freqs(64, 2)).to(DEV)
    M = B * h * w
    ss = torch.zeros(M, 8, device=DEV)
    ss[:, 0] = x.float().pow(2).sum(-1).flatten()
    ss[:, 1:] = float("nan")                     # only slot 0 belongs to a 128-wide level: the others must never be read
    ss_out = torch.full((M, 8), -1.0, device=DEV)
    n = min(B, 4)                                # images compared with the CPU reference
    want = _reference(x[:n], w_qkv, w_out, theta, scale, shift, ss[: n * h * w])
    got = N_.attn_block_bf16(x.clone(), w_qkv, w_out, theta, scale, shift, ss, ss_out)
    torch.cuda.synchronize()
    err = (got[:n].float().cpu() - want).abs()
    tol = 1.5e-2 * want.abs() + 3e-2
    assert bool((err <= tol).all()), f"max err {float(err.max()):.4f} (want {float(want.flatten()[err.argmax()]):.4f})"
    # every window of every image was written (the tail of the batch is not compared with the reference)
    assert bool(torch.isfinite(got.float()).all()) and float((got.float() - x.float()).abs().mean()) > 1e-2
    # row statistics of the new stream for the fused RMSNorm after it: slot 0 only
    want_ss = got.float().pow(2).sum(-1).flatten()
    assert torch.allclose(ss_out[:, 0], want_ss, rtol=2e-2, atol=1e-2)
    assert bool((ss_out[:, 1:] == -1.0).all())
    # in place with the statistics aliased, as the engine runs it
    ss2 = ss.clone()
    x2 = x.clone()
    N_.attn_block_bf16(x2, w_qkv, w_out, theta, scale, shift, ss2, ss2)
    torch.cuda.synchronize()
    assert torch.equal(x2, got)
    assert torch.equal(ss2[:, 0], ss_out[:, 0])
