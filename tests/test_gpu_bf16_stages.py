"""Every stage of the bf16 forward against an fp32 reference of that one stage.

The whole-image parity tests (test_gpu_bf16_parity.py) compare the final output with a rel-L2 budget: an error confined to one
TokenMerge quadrant, one tail tile, one head or one row-statistics slot moves that number by a fraction.  Here the engine is driven
on the route the sampler takes and every stage is read back through the debug taps (one tap per forward; the forward is
deterministic).  Each stage's reference is the oracle's fp32 restatement of that stage, fed with the PREVIOUS stage's tap (teacher
forcing) and rounded to bf16 where the kernels round.  So a failing stage names itself, and the comparison is tight enough that a
near miss -- a transposed quadrant, the other shift, swapped head scales, a statistics slot that covers half the row -- is rejected.

Routes:
  shared      one conditioning row for the batch (stride 0): folded weights bf16(bf16(W) * g), fused RMSNorm from the row statistics
              the previous GEMM left, attn_block / ffn_fused at 128-wide levels (what the sampler's graph runs)
  per_sample  one conditioning row per image: the stand-alone RMSNorm writes xn = bf16(x * g * rstd); the qkv (QKV_ROPE epilogue)
              and GEGLU GEMMs read xn with bf16(W)
"""
import copy
import math
import time

import pytest
import torch

from oracle import kdiff_oracle as O

DEV = "cuda"
U = 2.0 ** -8            # unit roundoff of bf16 (8-bit significand, round to nearest): |bf16(y) - y| <= U |y|

# ----------------------------------------------------------------------------------------------------------------------------
# Tolerance.  For a stage with input x_in, reference output y_want and update D_want = y_want - x_in (residual stages; the output
# itself for the others):
#
#     |y_got - y_want| <= U |y_want|  +  (2^-12 + 4 n U) rms(D_want)  +  n U |D_want|
#
# * U |y_want| is the stage's own output rounding (the reference's output is not rounded).
# * n = number of bf16 roundings strictly inside the stage (INNER below).  The reference rounds at the same points, so an inner
#   rounding differs from the kernel's only where fp32 accumulation-order noise carries a value across a rounding boundary (one ulp,
#   2U, at isolated elements), or where only the kernel rounds (the softmax numerators P of the attention kernels, U relative
#   everywhere).  A relative perturbation of size U in every element of one intermediate moves each output element by at most
#   U |D| where it acts coherently (a per-row scale: xn, the folded weight) -- the n U |D| term -- and by about U rms(D) as a
#   random-sign sum through the next linear map; 4 of those is the tail over the ~10^6 outputs of a stage -- the 4 n U rms(D) term.
# * 2^-12 rms(D) covers fp32 accumulation over K <= 3072 products and the MUFU tanh / exp2 / rsqrt approximations (relative
#   errors <= 2^-11 on a GELU that is then rounded to bf16 anyway).
#
# The constants depend on the stage kind only (no per-config tuning).  Every near miss below moves some outputs by several percent of
# rms(D), which is far outside this band; the CPU test at the bottom proves both directions before any GPU runs.
# ----------------------------------------------------------------------------------------------------------------------------
INNER = {
    "patch_in": 1,       # bf16(c_in * x)
    "attn": 4,           # xn (or the folded qkv weight), q/k/v, P, attention output
    "ff": 2,             # xn (or the folded up weight), GEGLU hidden
    "merge": 0,
    "split": 0,
    "qkv": 1,            # xn (or the folded weight)
    "ao": 1,             # P
    "geglu": 1,          # xn (or the folded weight)
    "out": 1,            # the out_norm-folded patch_out weight
}


def bf(t):
    return t.to(torch.bfloat16).to(t.dtype)


def gelu_tanh(x):
    """the tanh form of GELU that the tensor-core GEGLU epilogues evaluate (tc_common.cuh geglu2)"""
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608 * (x + 0.044715 * x ** 3)))


def tolerance(kind, d_want, round_of):
    n = INNER[kind]
    rms = float(d_want.double().pow(2).mean().sqrt())
    return U * round_of.abs() + (2.0 ** -12 + 4 * n * U) * rms + n * U * d_want.abs()


def ratio(kind, got, want, base=None, round_of=None):
    """max over elements of |got - want| / tol, and the number of elements out of tolerance"""
    got, want = got.double().cpu(), want.double().cpu()
    d_want = want if base is None else want - base.double().cpu()
    tol = tolerance(kind, d_want, want if round_of is None else round_of.double().cpu())
    r = (got - want).abs() / tol
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return float(r.max()), int((r > 1).sum())


# ----------------------------------------------------------------------------------------------------------------------------
# the model as a list of stages (execution order, names of engine.cu's taps)
# ----------------------------------------------------------------------------------------------------------------------------
class Layer:
    def __init__(self, k, prefix, level, index, C, F, attn):
        self.k, self.prefix, self.level, self.C, self.F = k, prefix, level, C, F
        self.kind = attn["type"]
        self.e = attn.get("d_head", 64)
        self.nh = C // self.e
        self.ws = attn.get("window_size", 0)
        self.ks = attn.get("kernel_size", 7)
        self.shift = self.ws // 2 if self.kind == "shifted-window" and index % 2 == 1 else 0     # image_transformer_v2.py:523
        self.ada_attn = self.ada_ff = None


class Plan:
    def __init__(self, mcfg, sd, H, W):
        self.sd, self.mcfg = sd, mcfg
        self.widths, depths, attns, dffs = mcfg["widths"], mcfg["depths"], mcfg["self_attns"], mcfg["d_ffs"]
        n = len(self.widths)
        self.n = n
        self.sigma_data = mcfg["sigma_data"]
        self.down, self.up, self.mid = [[] for _ in range(n - 1)], [[] for _ in range(n - 1)], []
        k = 0
        for l in range(n - 1):
            for i in range(depths[l]):
                self.down[l].append(Layer(k, f"down_levels.{l}.{i}.", l, i, self.widths[l], dffs[l], attns[l]))
                k += 1
        for i in range(depths[-1]):
            self.mid.append(Layer(k, f"mid_level.{i}.", n - 1, i, self.widths[-1], dffs[-1], attns[-1]))
            k += 1
        for l in reversed(range(n - 1)):
            for i in range(depths[l]):            # up-level layer index continues after the down level (image_transformer_v2.py:697)
                self.up[l].append(Layer(k, f"up_levels.{l}.{i}.", l, i + depths[l], self.widths[l], dffs[l], attns[l]))
                k += 1
        self.layers = [L for lv in self.down for L in lv] + self.mid + [L for l in reversed(range(n - 1)) for L in self.up[l]]
        off = 0
        for L in self.layers:                     # conditioning row: AdaRMSNorm scales in execution order, attention then ff
            if L.kind != "none":
                L.ada_attn, off = off, off + L.C
            L.ada_ff, off = off, off + L.C
        self.ada_total = off
        pos = O.make_axial_pos(H // mcfg["patch_size"][0], W // mcfg["patch_size"][1])
        self.pos = [pos]
        for _ in range(n - 1):
            self.pos.append(O.downscale_pos(self.pos[-1]))

    def gains_from_table(self, table):
        """{(k, 'attn'|'ff'): g [rows, C]} read from the engine's conditioning table (g = 1 + cond @ norm.linear.weight^T)"""
        g = {}
        for L in self.layers:
            if L.ada_attn is not None:
                g[L.k, "attn"] = table[:, L.ada_attn:L.ada_attn + L.C].float().cpu()
            g[L.k, "ff"] = table[:, L.ada_ff:L.ada_ff + L.C].float().cpu()
        return g

    def gains_from_cond(self, cond):
        """the same from the mapping network's output cond [rows, mw] (image_transformer_v2.py:166)"""
        g = {}
        for L in self.layers:
            if L.kind != "none":
                g[L.k, "attn"] = 1 + cond @ self.sd[L.prefix + "self_attn.norm.linear.weight"].T
            g[L.k, "ff"] = 1 + cond @ self.sd[L.prefix + "ff.norm.linear.weight"].T
        return g

    def cond_cpu(self, sigma):
        """mapping network on the CPU (oracle model_forward's conditioning, aug_cond = 0)"""
        sd = self.sd
        emb = O.fourier_features((torch.log(sigma) / 4)[:, None], sd["time_emb.weight"]) @ sd["time_in_proj.weight"].T
        emb = emb + O.fourier_features(sigma.new_zeros(sigma.shape[0], 9), sd["aug_emb.weight"]) @ sd["aug_in_proj.weight"].T
        return O.mapping_network(sd, emb)

    def neighbour_ff_gain(self, L, g):
        """the AdaRMSNorm scale of the nearest other layer of the same width (or, if there is none, this layer's attention scale)"""
        same = [M for M in self.layers if M.C == L.C and M.k != L.k]
        if not same:
            return g[L.k, "attn"]
        return g[min(same, key=lambda M: abs(M.k - L.k)).k, "ff"]


# ----------------------------------------------------------------------------------------------------------------------------
# stage references.  x: [B, h, w, C] holding the bf16 values the engine tapped.  emu=True evaluates the same stage in float64 with
# the kernels' extra roundings (P, the stored output): the CPU leg's stand-in for the GPU.  nm names a near miss.
# ----------------------------------------------------------------------------------------------------------------------------
def _dt(emu):
    return torch.float64 if emu else torch.float32


def _rstd(x, nm):
    xs = x[..., :128] if nm == "rms128" else x         # a statistics slot that covers only the first 128 channels
    return torch.rsqrt(xs.pow(2).mean(-1, keepdim=True) + O.EPS)


def _sdpa(q, k, v, allow, emu):
    s = q @ k.transpose(-1, -2)
    if allow is not None:
        s = s.masked_fill(~allow, float("-inf"))
    p = torch.exp(s - s.amax(-1, keepdim=True))
    if emu:
        p = bf(p)                                       # the attention kernels round P for the P V MMA and sum what it sees
    return (p @ v) / p.sum(-1, keepdim=True)


NA_DENSE_MAX_T = 1024    # larger neighbourhood grids take the gathered [T, 49] reference: a dense [T, T] mask of 128 x 128 tokens is 1 GiB


def _attend(q, k, v, L, shift, nm, emu, gathered=None):
    """q, k, v [B, h, w, nh, e] -> [B, h, w, nh, e] (oracle global / shifted-window / neighbourhood attention, scale 1).
    Neighbourhood attention over more than NA_DENSE_MAX_T tokens (or with gathered=True) gathers each query's 49 keys instead of
    masking a dense [T, T] score matrix (test_gpu_attn_na.na_attention)."""
    B, h, w, nh, e = q.shape
    if L.kind == "shifted-window":
        ws = L.ws

        def win(t):
            t = torch.roll(t, shifts=(shift, shift), dims=(1, 2))
            return t.reshape(B, h // ws, ws, w // ws, ws, nh, e).permute(0, 5, 1, 3, 2, 4, 6).reshape(B, nh, h // ws, w // ws, ws * ws, e)
        o = _sdpa(win(q), win(k), win(v), O.shifted_window_allow(h // ws, w // ws, ws, shift), emu)
        o = o.reshape(B, nh, h // ws, w // ws, ws, ws, e).permute(0, 2, 4, 3, 5, 1, 6).reshape(B, h, w, nh, e)
        return torch.roll(o, shifts=(-shift, -shift), dims=(1, 2))
    if L.kind == "neighborhood" and (gathered if gathered is not None else h * w > NA_DENSE_MAX_T):
        from test_gpu_attn_na import na_attention
        return na_attention(q, k, v, p_bf16=emu, nm="noclamp" if nm == "na_noclamp" else None)
    f = lambda t: t.reshape(B, h * w, nh, e).transpose(1, 2)
    allow = None
    if L.kind == "neighborhood":
        if nm == "na_noclamp":                          # window centred on the query and cut at the border instead of shifted inside
            i, j = torch.arange(h), torch.arange(w)
            rows = (i[None, :] - i[:, None]).abs() <= L.ks // 2
            cols = (j[None, :] - j[:, None]).abs() <= L.ks // 2
            allow = (rows[:, None, :, None] & cols[None, :, None, :]).reshape(h * w, h * w)
        else:
            allow = O.neighborhood_allow(h, w, L.ks)
    return _sdpa(f(q), f(k), f(v), allow, emu).transpose(1, 2).reshape(B, h, w, nh, e)


def _qkv(P, L, x, g, fold, nm, dt):
    """q, k, v after cosine-sim scaling and RoPE (fp32, not yet rounded)"""
    sd = P.sd
    p = L.prefix + "self_attn."
    B, h, w, C = x.shape
    rstd = _rstd(x, nm)
    Wq = bf(sd[p + "qkv_proj.weight"].to(dt))
    if fold:          # shared route: x @ bf16(bf16(W) g)^T; q and k are scale invariant, only v takes the row's 1 / rms
        hq = (x @ bf(Wq * g[0].to(dt)).T).view(B, h, w, 3, L.nh, L.e)
        q, k, v = hq[..., 0, :, :], hq[..., 1, :, :], hq[..., 2, :, :] * rstd[..., None]
    else:             # per-sample route: bf16(x g rstd) @ bf16(W)^T
        xn = bf(x * (g.to(dt).view(-1, 1, 1, C) * rstd))
        q, k, v = (xn @ Wq.T).view(B, h, w, 3, L.nh, L.e).unbind(3)
    scale = sd[p + "scale"].to(dt)
    if nm == "scale_swap":
        scale = scale[torch.arange(L.nh) ^ 1]                      # heads 0 <-> 1, 2 <-> 3, ...
    q, k = O.cosine_sim_scale(q, k, scale)
    pos = P.pos[L.level].to(dt)
    if nm == "rope_yx":
        pos = pos.flip(-1)
    theta = O.rope_theta(pos, sd[p + "pos_emb.freqs"].to(dt))
    return O.apply_rope(q, theta), O.apply_rope(k, theta), v


def ref_attn(P, L, x, g, fold, nm=None, emu=False):
    dt = _dt(emu)
    x = x.to(dt)
    B, h, w, C = x.shape
    q, k, v = _qkv(P, L, x, g, fold, nm, dt)
    shift = (L.ws // 2 - L.shift) if nm == "shift" else L.shift
    o = bf(_attend(bf(q), bf(k), bf(v), L, shift, nm, emu))
    y = o.reshape(B, h, w, C) @ bf(P.sd[L.prefix + "self_attn.out_proj.weight"].to(dt)).T + x
    return bf(y) if emu else y


def ref_qkv(P, L, x, g, fold, emu=False):
    dt = _dt(emu)
    q, k, v = _qkv(P, L, x.to(dt), g, fold, None, dt)
    B, h, w = x.shape[:3]
    y = torch.stack((q, k, v), 3).reshape(B, h, w, 3 * L.C)
    return bf(y) if emu else y


def ref_ao(P, L, qkv, emu=False):
    dt = _dt(emu)
    B, h, w, _ = qkv.shape
    q, k, v = qkv.to(dt).view(B, h, w, 3, L.nh, L.e).unbind(3)
    o = _attend(q, k, v, L, L.shift, None, emu).reshape(B, h, w, L.C)
    return bf(o) if emu else o


def _hidden(P, L, x, g, fold, nm, dt):
    sd = P.sd
    C = x.shape[-1]
    rstd = _rstd(x, nm)
    Wu = bf(sd[L.prefix + "ff.up_proj.weight"].to(dt))
    if fold:
        hh = (x @ bf(Wu * g[0].to(dt)).T) * rstd
    else:
        hh = bf(x * (g.to(dt).view(-1, 1, 1, C) * rstd)) @ Wu.T
    a, gate = hh.chunk(2, dim=-1)
    return a * gelu_tanh(gate)


def ref_ff(P, L, x, g, fold, nm=None, emu=False):
    dt = _dt(emu)
    x = x.to(dt)
    hid = bf(_hidden(P, L, x, g, fold, nm, dt))
    y = hid @ bf(P.sd[L.prefix + "ff.down_proj.weight"].to(dt)).T + x
    return bf(y) if emu else y


def ref_geglu(P, L, x, g, fold, emu=False):
    y = _hidden(P, L, x.to(_dt(emu)), g, fold, None, _dt(emu))
    return bf(y) if emu else y


def _gather(x, ph, pw, transposed):
    """TokenMerge's '(h nh) (w nw) e -> h w (nh nw e)'; transposed: (nw nh e)"""
    B, H, W, C = x.shape
    t = x.reshape(B, H // ph, ph, W // pw, pw, C)
    t = t.permute(0, 1, 3, 4, 2, 5) if transposed else t.permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B, H // ph, W // pw, ph * pw * C)


def _scatter(y, ph, pw, transposed):
    """TokenSplit's 'h w (nh nw e) -> (h nh) (w nw) e'; transposed: (nw nh e)"""
    B, h, w, N = y.shape
    t = y.reshape(B, h, w, ph, pw, N // (ph * pw))
    t = t.permute(0, 1, 4, 2, 3, 5) if transposed else t.permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B, h * ph, w * pw, N // (ph * pw))


def ref_merge(P, l, x, nm=None, emu=False):
    dt = _dt(emu)
    y = _gather(x.to(dt), 2, 2, nm == "quad_T") @ bf(P.sd[f"merges.{l}.proj.weight"].to(dt)).T
    return bf(y) if emu else y


def ref_split(P, l, x, skip, nm=None, emu=False):
    dt = _dt(emu)
    up = _scatter(x.to(dt) @ bf(P.sd[f"splits.{l}.proj.weight"].to(dt)).T, 2, 2, nm == "quad_T")
    fac = float(P.sd[f"splits.{l}.fac"])
    if nm == "fac_swap":
        fac = 1.0 - fac
    skip = skip.to(dt)
    if emu:           # the EPI_SPLIT_LERP epilogue's two-branch lerp
        d = up - skip
        return bf(skip + fac * d if fac < 0.5 else up - d * (1.0 - fac))
    return torch.lerp(skip, up, fac)


def ref_patch_in(P, img, sigma, nm=None, emu=False):
    dt = _dt(emu)
    c_in = 1.0 if nm == "no_cin" else O.karras_scalings(sigma.to(dt), P.sigma_data)[2].view(-1, 1, 1, 1)
    ph, pw = P.mcfg["patch_size"]
    y = _gather(bf(img.to(dt) * c_in).movedim(1, -1), ph, pw, nm == "pi_T") @ bf(P.sd["patch_in.proj.weight"].to(dt)).T
    return bf(y) if emu else y


def ref_out(P, x, img, sigma, nm=None, emu=False):
    """-> (denoised, c_skip x): fused out_norm + patch_out projection (F rounded to bf16) + un-patch + Karras combine"""
    dt = _dt(emu)
    sd = P.sd
    x = x.to(dt)
    W = bf(sd["patch_out.proj.weight"].to(dt))
    if nm != "no_out_norm":
        W = bf(W * sd["out_norm.scale"].to(dt))
    F = bf((x @ W.T) * _rstd(x, nm))
    ph, pw = P.mcfg["patch_size"]
    F = _scatter(F, ph, pw, False).movedim(-1, 1)
    s = sigma.to(dt).flip(0) if nm == "sigma_swap" else sigma.to(dt)
    c_skip, c_out, _ = O.karras_scalings(s, P.sigma_data)
    base = img.to(dt) * c_skip.view(-1, 1, 1, 1)
    return F * c_out.view(-1, 1, 1, 1) + base, base


# ----------------------------------------------------------------------------------------------------------------------------
# the stage walk, shared by the GPU tests (taps) and the CPU leg (emulation)
# ----------------------------------------------------------------------------------------------------------------------------
def near_misses(P, kind, L=None, B=1):
    """the wrong answers a stage of this kind must reject"""
    if kind == "patch_in":
        return ["pi_T", "no_cin"]
    if kind == "merge":
        return ["quad_T"]
    if kind == "split":
        return ["quad_T", "fac_swap"]
    # With a 128-wide row there is a single statistics slot: "the first 128 channels" is the whole row, and a wrong slot is a
    # NaN-poisoned one (the workspace is filled with NaN before every forward), so that near miss only exists from 256 channels.
    wide = ["rms128"] if (L.C if L is not None else P.widths[0]) >= 256 else []
    if kind == "attn":
        nm = ["scale_swap"]
        if L.kind == "shifted-window":
            nm += ["shift", "rope_yx"]
        if L.kind == "neighborhood":
            nm += ["na_noclamp"]
        return nm + wide
    if kind == "ff":
        return ["g_neighbour"] + wide
    if kind == "out":
        # the other image's sigma only differs when there is another image
        return ["no_out_norm"] + (["sigma_swap"] if B > 1 else []) + wide
    return []


class Walk:
    """Checks one stage at a time and records err/tol ratios; near misses are checked on the first stage of each (kind, level,
    shift) so that every branch is covered without repeating identical work."""

    def __init__(self, P, tag, fold, g):
        self.P, self.tag, self.fold, self.g = P, tag, fold, g
        self.worst = {}
        self.failures = []
        self.missed = []
        self.seen = set()

    def _record(self, kind, name, r, nbad):
        print(f"{self.tag} {name:>14s} [{kind}]: max err/tol {r:.3f}")
        self.worst[kind] = max(self.worst.get(kind, 0.0), r)
        if nbad:
            self.failures.append(f"{name}: {nbad} elements out of tolerance, max err/tol {r:.2f}")

    def stage(self, kind, name, got, want_fn, base=None, key=None, L=None, B=1):
        want = want_fn(None)
        if kind == "out":
            want, b = want
            r, nbad = ratio(kind, got, want, base=b, round_of=want - b)
        else:
            r, nbad = ratio(kind, got, want, base=base)
        self._record(kind, name, r, nbad)
        if key is not None and key not in self.seen:
            self.seen.add(key)
            for nm in near_misses(self.P, kind, L, B):
                w = want_fn(nm)
                if kind == "out":
                    w, b = w
                    rr, bad = ratio(kind, got, w, base=b, round_of=w - b)
                else:
                    rr, bad = ratio(kind, got, w, base=base)
                print(f"{self.tag} {name:>14s} near miss {nm:>12s}: max err/tol {rr:.1f} ({bad} out)")
                if bad == 0:
                    self.missed.append(f"{name}: near miss {nm} passes (max err/tol {rr:.3f})")

    def ff_gain(self, L, nm):
        return self.P.neighbour_ff_gain(L, self.g) if nm == "g_neighbour" else self.g[L.k, "ff"]


def walk(P, W, tap, img, sigma, inside=()):
    """Runs every stage in execution order.  tap(name, shape) -> the stage's output as the kernels left it (GPU: a debug tap;
    CPU: the emulation).  inside: layer indices whose .qkv / .ao / .geglu are checked as well."""
    B = img.shape[0]
    x = tap("patch_in", None)
    W.stage("patch_in", "patch_in", x, lambda nm: ref_patch_in(P, img, sigma, nm), key="patch_in", B=B)

    def layer(L, x):
        key = (L.level, L.shift)
        if L.kind != "none":
            a = tap(f"layer{L.k}.attn", x.shape)
            W.stage("attn", f"layer{L.k}.attn", a, lambda nm: ref_attn(P, L, x, W.g[L.k, "attn"], W.fold, nm), base=x, key=("attn",) + key, L=L)
            if L.k in inside:
                qkv = tap(f"layer{L.k}.qkv", x.shape[:3] + (3 * L.C,))
                W.stage("qkv", f"layer{L.k}.qkv", qkv, lambda nm: ref_qkv(P, L, x, W.g[L.k, "attn"], W.fold))
                ao = tap(f"layer{L.k}.ao", x.shape)
                W.stage("ao", f"layer{L.k}.ao", ao, lambda nm: ref_ao(P, L, qkv))
        else:
            a = x
        f = tap(f"layer{L.k}.ff", x.shape)
        W.stage("ff", f"layer{L.k}.ff", f, lambda nm: ref_ff(P, L, a, W.ff_gain(L, nm), W.fold, nm), base=a, key=("ff",) + key, L=L)
        if L.k in inside:
            gg = tap(f"layer{L.k}.geglu", x.shape[:3] + (L.F,))
            W.stage("geglu", f"layer{L.k}.geglu", gg, lambda nm: ref_geglu(P, L, a, W.g[L.k, "ff"], W.fold))
        return f

    skips = []
    for l in range(P.n - 1):
        for L in P.down[l]:
            x = layer(L, x)
        skip = tap(f"L{l}.down", x.shape)
        assert torch.equal(skip, x), f"L{l}.down differs from the last layer's output of the level"
        skips.append(skip)
        B_, h, w, C = x.shape
        m = tap(f"L{l}.merge", (B_, h // 2, w // 2, P.widths[l + 1]))
        W.stage("merge", f"L{l}.merge", m, lambda nm: ref_merge(P, l, x, nm), key=("merge", l))
        x = m
    for L in P.mid:
        x = layer(L, x)
    for l in reversed(range(P.n - 1)):
        B_, h, w, C = x.shape
        s = tap(f"L{l}.split", (B_, 2 * h, 2 * w, P.widths[l]))
        W.stage("split", f"L{l}.split", s, lambda nm: ref_split(P, l, x, skips[l], nm), base=skips[l], key=("split", l))
        x = s
        for L in P.up[l]:
            x = layer(L, x)
    out = tap("out", None)
    W.stage("out", "out", out, lambda nm: ref_out(P, x, img, sigma, nm), key="out", B=B)


# ----------------------------------------------------------------------------------------------------------------------------
# configurations
# ----------------------------------------------------------------------------------------------------------------------------
def _fixture_cfg(stem):
    import json
    from conftest import GOLDEN
    return json.loads((GOLDEN / f"{stem}_shapes.json").read_text())["config"]


def make(raw, H, W, seed=1):
    """(inner model, Plan) with synthetic weights; split 0 lerps with fac 0.3 and split 1 with fac 0.7 (both lerp branches)"""
    import k_diffusion as K
    from conftest import synth_sd
    cfg = K.config.load_config(raw)
    inner = K.config.make_model(cfg)
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, seed)
    for l, fac in enumerate((0.3, 0.7)):
        if f"splits.{l}.fac" in sd:
            sd[f"splits.{l}.fac"] = torch.tensor([fac])
    inner.load_state_dict(sd)
    return inner, Plan(cfg["model"], sd, H, W)


def cfg2_raw(H, W):
    raw = _fixture_cfg("cfg2_sw256")
    raw["model"] = dict(raw["model"], input_size=[H, W])
    return raw


def wide_raw():
    return {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [64, 64], "patch_size": [4, 4],
                      "depths": [1, 1], "widths": [384, 768], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160,
                      "self_attns": [{"type": "shifted-window", "d_head": 64, "window_size": 8}, {"type": "global", "d_head": 64}]}}


def na_raw():
    return {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [128, 128], "patch_size": [4, 4],
                      "depths": [2, 2, 2], "widths": [128, 256, 512], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160}}


def bench_raw(name):
    """bench.py's model config of a workload (cfg3 and cfg4: _NA_RAW at 256x256; cfg5: widths 256/512/1024 at 512x512)"""
    import bench
    return copy.deepcopy(bench.CONFIGS[name]["raw"])


def latent(seed, B, H, W, sigma):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, H, W, generator=g) * (sigma * sigma + 0.25).sqrt().view(-1, 1, 1, 1)


# name: (raw config, H, W, sigmas, layers whose .qkv / .ao / .geglu are checked)
CONFIGS = {
    # the benchmarked shape: attn_block + ffn_fused at level 0, merges with mwc 32 / 16 (box_h > 1), 2- and 4-slot statistics
    "cfg2_256_b2": (lambda: cfg2_raw(256, 256), 256, 256, [2.5, 40.0], (1, 2)),
    # M tails: level 1 has M = 192, the middle level M = 48; one-window attention; merges with mwc 8 / 4
    "cfg2_64_b3": (lambda: cfg2_raw(64, 64), 64, 64, [0.3, 2.5, 40.0], (1, 2)),
    # merge with mwc = 128 (box_h == 1); aspect ratio 16 RoPE positions; level-1 grid 8 x 128
    "cfg2_64x1024_b1": (lambda: cfg2_raw(64, 1024), 64, 1024, [2.5], (1, 2)),
    # 3 and 6 statistics slots; attn_block refused (C != 128); merge with K = 1536
    "w384_64_b2": (wide_raw, 64, 64, [2.5, 40.0], (0, 1)),
    # the tensor-core neighbourhood kernel (32 x 32 tokens at level 0), the generic one at level 1
    "na_128_b2": (na_raw, 128, 128, [2.5, 40.0], (1, 2)),
    # cfg3 / cfg4's model: the tensor-core neighbourhood kernel at 64 x 64 tokens with 2 heads and 32 x 32 with 4, the global kernel
    # over 256 tokens with 8 heads; layers 1, 3 and 4 are one layer of each level
    "cfg3_256_b2": (lambda: bench_raw("cfg3"), 256, 256, [2.5, 40.0], (1, 3, 4)),
    # cfg5's model: a 256-wide level 0 (no fused 128-wide kernels), all 8 row-statistics slots at width 1024, neighbourhood attention
    # at 128 x 128 tokens, global attention over 1024 tokens with 16 heads, merges with K = 1024 and 2048, a split with N = 2048 and a
    # down projection with K = 3072
    "cfg5_512_b2": (lambda: bench_raw("cfg5"), 512, 512, [2.5, 40.0], (1, 3, 4)),
}
ROUTES = [("cfg2_256_b2", "shared"), ("cfg2_256_b2", "per_sample"), ("cfg2_64_b3", "shared"), ("cfg2_64x1024_b1", "shared"),
          ("w384_64_b2", "shared"), ("na_128_b2", "shared"), ("cfg3_256_b2", "shared"), ("cfg3_256_b2", "per_sample"),
          ("cfg5_512_b2", "shared")]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,route", ROUTES)
def test_bf16_stages_vs_fp32_reference(config, route):
    from k_diffusion import _native as N_
    raw_fn, H, Wd, sigmas, inside = CONFIGS[config]
    t0 = time.time()
    inner, P = make(raw_fn(), H, Wd)
    inner = inner.to(DEV).eval().set_precision("bf16")
    eng = inner.engine()
    B = len(sigmas)
    sigma = torch.tensor(sigmas)
    img = latent(7, B, H, Wd, sigma)
    x_d, s_d = img.to(DEV), sigma.to(DEV)
    shared = route == "shared"
    table = eng.conditioning(s_d[:1] if shared else s_d)
    stride = 0 if shared else eng.cond_stride
    g = P.gains_from_table(table)
    # the table's AdaRMSNorm scales are 1 + cond @ W^T of the mapping network's output (stored after them): the offsets above are right
    cmap = table[:, P.ada_total:P.ada_total + P.mcfg["mapping_width"]].float().cpu()
    for key, want in P.gains_from_cond(cmap).items():
        assert torch.allclose(g[key], want, rtol=1e-4, atol=1e-4), f"conditioning table entry {key}"
    sd_ = P.sigma_data

    def forward(name, n):
        ws = eng._workspace(N_.PREC_BF16, B, H, Wd, x_d.device)
        ws.view(torch.float32).fill_(float("nan"))          # a statistics slot that was never written cannot pass on a stale value
        buf = None
        if name is not None:
            buf = eng.arm_tap(name, n, DEV)
            buf.fill_(float("nan"))
        out = eng.forward(x_d, s_d, table, stride, sd_, N_.PREC_BF16)
        torch.cuda.synchronize()
        if name is not None:
            assert eng.tap_count() == n, f"tap {name}: {eng.tap_count()} elements, expected {n}"
        return buf, out

    def tap(name, shape):
        if name == "out":
            return forward(None, 0)[1].cpu()
        if shape is None:                                    # patch_in
            ph, pw = P.mcfg["patch_size"]
            shape = (B, H // ph, Wd // pw, P.widths[0])
        n = math.prod(shape)
        buf, _ = forward(name, n)
        return buf.cpu().view(shape)

    # deterministic: the same stage tapped twice is bit-identical
    mid_shape = (B, H // 4 >> (P.n - 1), Wd // 4 >> (P.n - 1), P.widths[-1])
    assert torch.equal(tap("mid", mid_shape), tap("mid", mid_shape))

    W = Walk(P, f"{config}/{route}", shared, g)
    walk(P, W, tap, img, sigma, inside)
    print(f"{config}/{route}: worst err/tol per stage kind " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(W.worst.items())) +
          f"; {time.time() - t0:.1f} s")
    assert not W.failures, "\n".join(W.failures)
    assert not W.missed, "\n".join(W.missed)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,B", [("cfg3_256_b2", 64), ("cfg5_512_b2", 16)])
def test_benchmark_batch_images_equal_single_image_runs(config, B):
    """At the benchmark's batch (cfg3: 64, cfg5: 16) on the sampler's shared route (one conditioning row, stride 0), images 0, B/2
    and B - 1 of the batch are bit for bit the same images run alone.  Every kernel on this route computes an image's rows from that
    image only, in an order fixed by the shapes of one image (test_gpu_gemm_schedule.py and test_gpu_attn_persistent.py assert it
    kernel by kernel); here it holds for the whole forward, where a tile schedule, statistics slot or workspace offset that
    depended on the batch would show."""
    from k_diffusion import _native as N_
    raw_fn, H, Wd, _, _ = CONFIGS[config]
    inner, P = make(raw_fn(), H, Wd)
    inner = inner.to(DEV).eval().set_precision("bf16")
    eng = inner.engine()
    t0 = time.time()
    sigma = torch.full([B], 2.5)
    img, s_d = latent(13, B, H, Wd, sigma).to(DEV), sigma.to(DEV)
    table = eng.conditioning(s_d[:1])
    full = eng.forward(img, s_d, table, 0, P.sigma_data, N_.PREC_BF16).clone()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(full).all())
    for b in (0, B // 2, B - 1):
        one = eng.forward(img[b:b + 1].contiguous(), s_d[b:b + 1], table, 0, P.sigma_data, N_.PREC_BF16)
        torch.cuda.synchronize()
        d = (full[b:b + 1] - one).abs()
        assert torch.equal(full[b:b + 1].view(torch.int32), one.view(torch.int32)), \
            f"image {b} of {B} differs from the same image alone: {int((d > 0).sum())} elements, max |diff| {float(d.max()):.3g}"
    print(f"{config} B={B}: {time.time() - t0:.1f} s")


@pytest.mark.gpu
def test_patch_out_with_unaligned_x_and_out():
    """A contiguous fp32 x or out= buffer that starts 4 bytes into its storage takes the scalar patch_out kernels (the tensor-core
    epilogue reads x and writes out as float4) and gives the aligned result up to the weight rounding that route differs in."""
    inner, _ = make(cfg2_raw(64, 64), 64, 64)
    inner = inner.to(DEV).eval().set_precision("bf16")
    sigma = torch.tensor([2.5, 40.0], device=DEV)
    img = latent(3, 2, 64, 64, sigma.cpu()).to(DEV)
    want = inner.denoise(img, sigma, 0.5)
    n = img.numel()
    x_off = torch.empty(n + 1, device=DEV)[1:].view_as(img)
    x_off.copy_(img)
    assert x_off.is_contiguous() and x_off.data_ptr() % 16 == 4
    out_off = torch.full((n + 1,), float("nan"), device=DEV)[1:].view_as(img)
    c_skip = O.karras_scalings(sigma.cpu(), 0.5)[0].view(-1, 1, 1, 1)
    f_want = want.cpu() - img.cpu() * c_skip                      # c_out F
    for x_, o_ in ((img, out_off), (x_off, None), (x_off, out_off)):
        got = inner.denoise(x_, sigma, 0.5, out=o_)
        torch.cuda.synchronize()
        if o_ is not None:
            assert got.data_ptr() == o_.data_ptr()
        assert bool(torch.isfinite(got).all())                   # every element of the NaN-filled out= buffer was written
        f_got = got.cpu() - img.cpu() * c_skip
        if x_ is img:
            # only patch_out differs (fp32 weight, normalised tokens rounded to bf16, instead of the folded bf16 weight): two
            # roundings of F apart, 2U |F|, plus U rms(F) per rounded operand as random-sign sums
            err = (f_got - f_want).abs()
            tol = 2.0 ** -7 * f_want.abs() + 2.0 ** -6 * float(f_want.pow(2).mean().sqrt())
            assert bool((err <= tol).all()), f"max err/tol {float((err / tol).max()):.3f}"
        else:
            # an unaligned x also moves patch_in to its scalar kernel: the whole token stream rounds differently
            assert float((f_got - f_want).norm() / f_want.norm()) < 2e-2


# ----------------------------------------------------------------------------------------------------------------------------
# CPU leg: the tolerance accepts an emulation of the kernels' arithmetic and rejects every near miss
# ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["shared", "per_sample"])
def test_stage_tolerance_accepts_emulation_and_rejects_near_misses(route):
    """sw64 architecture (cfg2 at 64x64), B = 1, on the CPU.  The 'kernel' is the stage references evaluated in float64 with the
    kernels' rounding points (inner intermediates, P, the stored output); the reference is fp32 without those.  Every stage must
    pass and every near miss must put at least one element out of tolerance."""
    _, P = make(cfg2_raw(64, 64), 64, 64)
    sigma = torch.tensor([2.5])
    img = latent(11, 1, 64, 64, sigma)
    fold = route == "shared"
    g = P.gains_from_cond(P.cond_cpu(sigma))
    W = Walk(P, f"cpu-emulation/{route}", fold, g)
    layers = {L.k: L for L in P.layers}
    state = {}

    def tap(name, shape):
        # the emulated kernel output of this stage, fed (like the GPU taps) with the previous emulated stage.  state["x"] is the
        # stream, state["in"] a layer's input, state["a"] its attention output.
        if name == "patch_in":
            y = ref_patch_in(P, img, sigma, emu=True)
        elif name.startswith("layer"):
            k, part = name[5:].split(".")
            L = layers[int(k)]
            if part == "attn":
                state["in"] = state["x"]
                y = state["a"] = ref_attn(P, L, state["in"], g[L.k, "attn"], fold, emu=True).float()
            elif part == "qkv":
                return ref_qkv(P, L, state["in"], g[L.k, "attn"], fold, emu=True).float()
            elif part == "ao":
                return ref_ao(P, L, ref_qkv(P, L, state["in"], g[L.k, "attn"], fold, emu=True), emu=True).float()
            elif part == "geglu":
                return ref_geglu(P, L, state["a"], g[L.k, "ff"], fold, emu=True).float()
            else:
                y = ref_ff(P, L, state["x"], g[L.k, "ff"], fold, emu=True)
        elif name.endswith(".down"):
            return state["x"]
        elif name.endswith(".merge"):
            l = int(name[1:].split(".")[0])
            state[f"skip{l}"] = state["x"]
            y = ref_merge(P, l, state["x"], emu=True)
        elif name.endswith(".split"):
            l = int(name[1:].split(".")[0])
            y = ref_split(P, l, state["x"], state[f"skip{l}"], emu=True)
        elif name == "out":
            return ref_out(P, state["x"], img, sigma, emu=True)[0].float()
        else:
            raise KeyError(name)
        state["x"] = y.float()
        return state["x"]

    walk(P, W, tap, img, sigma, inside=(1, 2))
    print(f"cpu-emulation/{route}: worst err/tol " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(W.worst.items())))
    assert not W.failures, "\n".join(W.failures)
    assert not W.missed, "\n".join(W.missed)
    # every near-miss kind was exercised at least once
    assert {"attn", "ff", "merge", "split", "patch_in", "out", "qkv", "ao", "geglu"} <= set(W.worst)


@pytest.mark.parametrize("emu", [False, True], ids=["fp32", "emulation"])
@pytest.mark.parametrize("nm", [None, "na_noclamp"])
def test_gathered_and_dense_neighbourhood_references_agree(nm, emu):
    """na_128_b2's neighbourhood levels (32 x 32 tokens with 2 heads, 16 x 16 with 4) on the CPU: the gathered reference that the
    larger grids of cfg3 and cfg5 take gives what the dense mask gives, for the stage reference, its emulation and its near miss."""
    _, P = make(na_raw(), 128, 128)
    dt = _dt(emu)
    for L in (P.down[0][0], P.down[1][0]):
        assert L.kind == "neighborhood"
        h = 32 >> L.level
        g = torch.Generator().manual_seed(L.k)
        q, k, v = (torch.randn(2, h, h, L.nh, L.e, generator=g, dtype=dt) for _ in range(3))
        q, k = (t / t.norm(dim=-1, keepdim=True) * 10 ** 0.5 for t in (q, k))     # the cosine-sim scale of a layer: |q . k| <= 10
        dense = _attend(q, k, v, L, 0, nm, emu, gathered=False)
        gathered = _attend(q, k, v, L, 0, nm, emu, gathered=True)
        assert float((dense - gathered).abs().max()) < (1e-12 if emu else 1e-5), f"level {L.level}"
    # the near miss is a different answer at this size
    if nm is not None:
        assert float((_attend(q, k, v, L, 0, None, emu) - dense).abs().max()) > 0.1
