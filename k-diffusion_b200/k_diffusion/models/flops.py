"""Algorithmic work of the image_transformer_v2 forward pass (same accounting as the reference's
models/flops.py:40-54: one MAC per weight per token; attention = q k^T and a v).

`linear_layers` lists every nn.Linear on the token stream in execution order -- the order the engine
launches its GEMMs -- so a per-launch profile can be matched to shapes."""


def token_grid(mcfg):
    ph, pw = mcfg["patch_size"]
    return mcfg["input_size"][0] // ph, mcfg["input_size"][1] // pw


def linear_layers(mcfg, batch=1):
    """[(label, M, N, K)] for batch `batch`, in execution order."""
    widths, depths, d_ffs, attns = mcfg["widths"], mcfg["depths"], mcfg["d_ffs"], mcfg["self_attns"]
    h, w = token_grid(mcfg)
    t0, n = h * w, len(widths)
    seq = []

    def layer(l, tag):
        M, C, F = batch * (t0 >> (2 * l)), widths[l], d_ffs[l]
        if attns[l]["type"] != "none":
            seq.append((f"{tag} qkv", M, 3 * C, C))
            seq.append((f"{tag} out+res", M, C, C))
        seq.append((f"{tag} up+geglu", M, 2 * F, C))
        seq.append((f"{tag} down+res", M, C, F))

    for l in range(n - 1):
        for i in range(depths[l]):
            layer(l, f"L{l}.down{i}")
        seq.append((f"merge{l}", batch * (t0 >> (2 * l + 2)), widths[l + 1], 4 * widths[l]))
    for i in range(depths[-1]):
        layer(n - 1, f"mid{i}")
    for l in reversed(range(n - 1)):
        seq.append((f"split{l}", batch * (t0 >> (2 * l + 2)), 4 * widths[l], widths[l + 1]))
        for i in range(depths[l]):
            layer(l, f"L{l}.up{i}")
    return seq


FUSED_FFN_WIDTHS = (128,)      # level widths whose feed-forward block runs as ONE kernel (csrc/tc_ffn_fused.cuh)
FUSED_ATTN_WIDTHS = (128,)     # level widths whose shifted-window attention block runs as ONE kernel (csrc/tc_attn_block.cuh)


def fused_attention_levels(mcfg):
    """Levels whose whole attention block (qkv, window attention, out_proj) is one kernel on the bf16 path: 128 wide, two heads of 64,
    8x8 shifted windows, token grid a multiple of 8."""
    h, w = token_grid(mcfg)
    out = set()
    for l, (C, a) in enumerate(zip(mcfg["widths"], mcfg["self_attns"])):
        if (C in FUSED_ATTN_WIDTHS and a["type"] == "shifted-window" and a.get("window_size") == 8 and a.get("d_head", 64) == 64
                and (h >> l) % 8 == 0 and (w >> l) % 8 == 0):
            out.add(l)
    return out


def launch_layers(mcfg, batch=1, fused_ffn=True):
    """[(label, M, N, K, macs)] per tensor-core GEMM LAUNCH in execution order: like `linear_layers`, but an up_proj + down_proj pair of a
    128-wide level is one launch when the fused feed-forward kernel is active (N, K are then the up projection's; macs covers both), and
    the qkv + out_proj pair of a level in `fused_attention_levels` is one launch (N, K are the qkv projection's; macs covers both, the
    window attention inside that kernel is not a Linear and is not counted)."""
    fused_attn_C = {mcfg["widths"][l] for l in fused_attention_levels(mcfg)}
    out, seq, i = [], linear_layers(mcfg, batch), 0
    while i < len(seq):
        label, M, N, K = seq[i]
        if label.endswith(" qkv") and K in fused_attn_C and i + 1 < len(seq):
            _, M2, N2, K2 = seq[i + 1]
            out.append((label.replace(" qkv", " attn (qkv+window attention+out+res, fused)"), M, N, K, M * N * K + M2 * N2 * K2))
            i += 2
        elif fused_ffn and label.endswith("up+geglu") and K in FUSED_FFN_WIDTHS and i + 1 < len(seq):
            _, M2, N2, K2 = seq[i + 1]
            out.append((label.replace("up+geglu", "ffn (up+geglu+down+res, fused)"), M, N, K, M * N * K + M2 * N2 * K2))
            i += 2
        else:
            out.append((label, M, N, K, M * N * K))
            i += 1
    return out


def linear_macs(mcfg, batch=1):
    return sum(M * N * K for _, M, N, K in linear_layers(mcfg, batch))


def attention_macs(mcfg, batch=1):
    """q k^T and a v MACs of the attention that runs in the stand-alone attention kernels (attn_ws_kernel, attn_na_kernel), i.e. of every level except
    the `fused_attention_levels`, whose attention runs inside the fused attention-block kernel."""
    widths, depths, attns = mcfg["widths"], mcfg["depths"], mcfg["self_attns"]
    h, w = token_grid(mcfg)
    total, n = 0, len(widths)
    fused = fused_attention_levels(mcfg)
    for l in range(n):
        a = attns[l]
        if a["type"] == "none" or l in fused:
            continue
        t = (h >> l) * (w >> l)
        e = a.get("d_head", 64)
        keys = t if a["type"] == "global" else (a["window_size"] ** 2 if a["type"] == "shifted-window" else a.get("kernel_size", 7) ** 2)
        total += depths[l] * (1 if l == n - 1 else 2) * (widths[l] // e) * t * keys * 2 * e
    return total * batch
