"""The persistent token-stream GEMM (gemm_wg_kernel): one CTA per SM walks the output tiles and its two MMA warpgroups take alternate
tiles, so a tile's CTA, warpgroup and ring phase depend on M.  A row block must come out bit-identical whatever M it is computed
inside, for every epilogue; tile counts around multiples of the SM count, fewer k-blocks than ring stages, long K and M tails
exercise the schedule's edges."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(M, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
    return a, w


def _placement(M, N, K, block, sms):
    """Where gemm_wg_kernel computes the tiles of 128-row block `block` of an [M, N] x K problem: [(CTA, warpgroup, ring position of
    the tile's first k-block)] over its n-tiles.  Tile t = block * n_tiles + n (N-fastest), grid = min(tiles, SMs), CTA t % grid takes
    it as its local tile t // grid, warpgroup = local % 2, and the CTA's ring has carried local * K / 64 k-blocks before it."""
    bn = 128 if N % 128 == 0 else 64
    n_tiles = N // bn
    tiles = -(-M // 128) * n_tiles
    grid = min(tiles, sms)
    return [((block * n_tiles + n) % grid, (block * n_tiles + n) // grid % 2, (block * n_tiles + n) // grid * (K // 64)) for n in range(n_tiles)]


def _blocks_to_compare(M, N, K, sms):
    """Row blocks 0 and last (tail), and the first block with a tile on warpgroup 1 of its CTA when the problem has one"""
    nb = -(-M // 128)
    picks = [0, nb - 1]
    odd = [b for b in range(nb) if any(wg == 1 for _, wg, _ in _placement(M, N, K, b, sms))]
    if odd:
        picks.append(odd[0])
    return sorted(set(picks)), bool(odd)


# (tiles of 128 rows as a function of the SM count S, K): fewer tiles than SMs, exactly S and 2 S, 2 S +- 1, with K = 64 (one k-block,
# fewer than the ring's stages), 128, 256 and 1536; the -37 makes the last row block a tail
@pytest.mark.parametrize("tiles,K", [(lambda S: 7, 64), (lambda S: S, 256), (lambda S: 2 * S, 128), (lambda S: 2 * S - 1, 64),
                                     (lambda S: 2 * S + 1, 1536), (lambda S: 3 * S + 1, 256)])
@pytest.mark.parametrize("N", [128, 64])
def test_store_tile_counts_and_row_blocks(tiles, K, N):
    from k_diffusion import _native as N_
    S = _sms()
    M = 128 * tiles(S) - 37
    a, w = _operands(M, N, K, M + K)
    got = N_.gemm_bf16(a, w)
    want = a.float() @ w.float().T
    err = (got.float() - want).abs()
    assert bool((err <= 1e-2 * want.abs() + 2e-2).all()), f"max err {float(err.max()):.4f}"
    # a row block alone is one tile row: CTAs 0.., warpgroup 0, ring position 0.  Inside the full problem the compared blocks include the
    # tail and, whenever a CTA gets more than one tile, a block on warpgroup 1 further along the ring
    blocks, has_wg1 = _blocks_to_compare(M, N, K, S)
    assert has_wg1 == (-(-M // 128) * (N // (128 if N % 128 == 0 else 64)) > S)
    for b in blocks:
        r0 = 128 * b
        rows = min(128, M - r0)
        alone = N_.gemm_bf16(a[r0:r0 + rows].contiguous(), w)
        assert torch.equal(alone, got[r0:r0 + rows]), f"row block {b}, placed at {_placement(M, N, K, b, S)}"


# M: 133 row blocks of N2 = 1536 (12 n-tiles each) with a 123-row tail, 265 row blocks with a one-row tail, 3 row blocks (fewer tiles
# than SMs: every tile on warpgroup 0)
@pytest.mark.parametrize("M,K", [(128 * 133 - 5, 256), (128 * 264 + 1, 512), (300, 1024)])
def test_geglu_with_row_statistics_row_blocks(M, K):
    from k_diffusion import _native as N_
    S = _sms()
    N2 = 1536
    a, w = _operands(M, N2, K, M)
    parts = torch.zeros(M, 8, device=DEV)
    xs = a.float().view(M, K // 128, 128)
    parts[:, :K // 128] = (xs * xs).sum(-1)
    got = N_.gemm_bf16_geglu(a, w, parts)
    assert bool(torch.isfinite(got.float()).all()) and float(got.float().abs().mean()) > 0
    blocks, has_wg1 = _blocks_to_compare(M, N2, K, S)
    assert has_wg1 == (-(-M // 128) * (N2 // 128) > S)
    for b in blocks:
        r0 = 128 * b
        rows = min(128, M - r0)
        part = N_.gemm_bf16_geglu(a[r0:r0 + rows].contiguous(), w, parts[r0:r0 + rows].contiguous())
        assert torch.equal(part, got[r0:r0 + rows]), f"row block {b}, placed at {_placement(M, N2, K, b, S)}"


def test_engine_stages_independent_of_batch():
    """The last image of a batch of 17 through the cfg2 model (256 x 256), and the same image alone: every GEMM stage outside level 0 --
    qkv with cos-sim + RoPE, out_proj and down_proj with the residual and row statistics, up_proj + GEGLU with the fused norm, the
    TokenMerge gathers, the TokenSplit lerps -- and the denoised image are bit-identical.  Alone, every tile of the image is the first
    tile of its CTA (warpgroup 0, ring position 0); in the batch, each of its tiles is on another CTA or further along the ring, and every
    generic GEMM puts some of them on warpgroup 1 (asserted below from the launch shapes)."""
    from test_gpu_bf16_stages import cfg2_raw, latent, make
    import k_diffusion as K
    from k_diffusion import _native as N_
    H = W = 256
    B = 17
    S = _sms()
    inner, P = make(cfg2_raw(H, W), H, W)
    launches = [(lbl, M, N, Kd) for lbl, M, N, Kd, _ in K.models.flops.launch_layers(P.mcfg, B) if "fused" not in lbl]
    assert launches
    for lbl, M, N, Kd in launches:
        per = M // B // 128                              # row blocks per image
        batched = [t for b in range((B - 1) * per, B * per) for t in _placement(M, N, Kd, b, S)]
        alone = [t for b in range(per) for t in _placement(M // B, N, Kd, b, S)]
        assert all(wg == 0 and ring == 0 for _, wg, ring in alone), lbl
        assert any(wg == 1 for _, wg, _ in batched) and all(x != y for x, y in zip(batched, alone)), (lbl, batched)

    inner = inner.to(DEV).eval().set_precision("bf16")
    eng = inner.engine()
    names = []
    for L in P.layers:
        if L.level == 0:
            continue
        if L.kind != "none":
            names += [f"layer{L.k}.qkv", f"layer{L.k}.ao"]
        names += [f"layer{L.k}.geglu", f"layer{L.k}.ff"]
    names += [f"L{l}.merge" for l in range(P.n - 1)] + [f"L{l}.split" for l in range(P.n - 1)]
    sigma = torch.tensor([0.3, 2.5, 40.0] * 6)[:B]
    img = latent(5, B, H, W, sigma)
    table = eng.conditioning(sigma[-1:].to(DEV))         # one shared conditioning row for both runs

    def last_image(Bn):
        x, s = img[B - Bn:].to(DEV), sigma[B - Bn:].to(DEV)
        res = {}
        for name in names + [None]:
            buf = eng.arm_tap(name, Bn * H * W * 16, DEV) if name else None
            out = eng.forward(x, s, table, 0, P.sigma_data, N_.PREC_BF16)
            torch.cuda.synchronize()
            if name:
                n = eng.tap_count()
                assert n > 0 and n % Bn == 0, f"tap {name}: {n} elements"
                res[name] = buf[n - n // Bn:n].cpu()
            else:
                res["out"] = out[-1:].cpu()
        return res

    alone, batched = last_image(1), last_image(B)
    bad = [k for k in alone if not torch.equal(alone[k], batched[k])]
    assert not bad, f"stages that depend on the batch: {bad}"
