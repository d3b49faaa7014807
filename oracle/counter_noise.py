"""Host restatement of the counter-based noise kernels of csrc/solver.cu, in numpy (no torch).

- `philox4x32_10`: the Philox4x32-10 block function of Salmon et al., "Parallel random numbers: as easy as 1, 2, 3" (SC'11), on uint32
  words.  tests/test_noise_host.py pins it with the Random123 known-answer vectors.
- `u01`: the kernels' uint32 -> (0, 1] map, emulated in float32 so its rounding is the kernel's: (x >> 8) 2^-24 + 2^-25 rounds to even,
  so x >> 8 = 2^24 - 1 gives exactly 1.0f and x >> 8 = 2^24 - 2 gives 1 - 2^-23.
- `box_muller`: both Box-Muller forms in float64 from those float32 uniforms, with a per-element error bound of the kernel's float32
  evaluation (derivation above `_radius_err`).
- `noise_normal` / `brownian`: `noise_normal_kernel` and `noise_brownian_kernel`, with the counter layouts the kernels build, evaluated in
  float64 for any subset of (sample, group) pairs, each with a per-element bound.

Element i of sample b belongs to group g = i // 4, lane i % 4; a group is one Philox call.  The key is the sample's 64-bit seed (low word,
high word).  Counters:
- normal:   (g_lo, g_hi, stream_lo, stream_hi ^ "norm"); no state carries between samples, so every sample numbers its groups from 0.
- Brownian: (g_lo, g_hi, word, "brow"), word = 1 for the root draw W(t_max) = sqrt(t_max - t_min) z, and node + 2^31 for the bridge draw
  at the midpoint of node's interval.  The root interval is node 1, the children of node n are 2n (left) and 2n + 1 (right), and a walk
  toward t goes left when t < mid.  W(t_min) = 0; `depth` levels of midpoints are drawn on the way to t, then W is linear inside the last
  interval (the leaf).
"""
import math

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57          # Philox multipliers
W0, W1 = 0x9E3779B9, 0xBB67AE85          # Weyl key increments
TAG_NORMAL = 0x6E6F726D                  # "norm"
TAG_BROWNIAN = 0x62726F77                # "brow"
MID_OFFSET = 0x80000000                  # counter word of a bridge draw = node + 2^31
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key, rounds=10):
    """counter uint32 [..., 4], key uint32 [..., 2] (broadcast against each other) -> uint32 [..., 4].
    `rounds` exists for mutation tests only; Philox4x32-10 is rounds = 10."""
    counter, key = np.asarray(counter, dtype=np.uint32), np.asarray(key, dtype=np.uint32)
    c = [counter[..., i].astype(np.uint64) for i in range(4)]
    k0, k1 = key[..., 0].astype(np.uint64), key[..., 1].astype(np.uint64)
    for _ in range(rounds):
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + np.uint64(W0)) & _M32, (k1 + np.uint64(W1)) & _M32
    return np.stack(np.broadcast_arrays(*c), axis=-1).astype(np.uint32)


def u01(x):
    """(float)(x >> 8) * 2^-24 + 2^-25 in float32: the product is exact, so the kernel's fma contraction gives the same value."""
    x = np.asarray(x, dtype=np.uint32)
    return (x >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24) + np.float32(2.0 ** -25)


def seed_words(seeds):
    """int64 seeds (negative ones included) -> uint32 [B, 2] keys (low word, high word)"""
    s = np.array([int(v) & (2 ** 64 - 1) for v in np.ravel(seeds)], dtype=np.uint64)
    return np.stack([s & _M32, s >> np.uint64(32)], axis=-1).astype(np.uint32)


# ------------------------------------------------------------------------------------------------
# Error bounds of the kernels' float32 Box-Muller.
#
# The kernels compute z = r * cos(a), r * sin(a) with r = sqrt(-2 ln u) from one uniform and the angle a from another.  Let e_r bound
# |r~ - r| and e_t bound the error of the computed cosine or sine.  Then |z~ - z| <= |trig| e_r + r e_t + e_r e_t + 2^-24 |z|, the last
# term being the rounding of the product.
#
# Radius.  With m = -2 ln u = r^2 and |m~ - m| <= e_m, the square root gives |sqrt(m~) - sqrt(m)| <= min(sqrt(e_m), e_m / r) (exact, not
# linearised: near u -> 1, m is of the order of e_m itself), and the correctly rounded float32 square root adds 2^-24 r.
# - normal4 (library built without fast-math, see csrc/Makefile): logf has a maximum error of 1 ulp (CUDA C Programming Guide, "Standard
#   Functions"), the multiply by -2 is exact, sqrtf is correctly rounded.  e_m = 2 ulp(ln u).
# - normal4_fast: __log2f has a maximum absolute error of 2^-22 for u in [0.5, 2] and 2 ulp elsewhere (guide, "Intrinsic Functions"; some
#   editions print 2^-22.6, the looser figure is used).  It is multiplied by the float32 constant -2 ln 2 (relative error <= 2^-24) with
#   one rounding, and __fsqrt_rn is correctly rounded.  e_m = 2 ln 2 e_log2 + 2^-23 m.
#   At u = 1 - 2^-23, m = 2.4e-7 while 2 ln 2 2^-22 = 3.3e-7, so r = 4.9e-4 may be off by up to sqrt(e_m) = 5.8e-4: the guide does not
#   promise better than that.  At u = 1.0f both forms take the log of 1, and the tests require exactly 0 there.
#
# Angle.
# - normal4: sincospif(2u); 2u is exact and sinpif / cospif have a maximum error of 1 ulp: e_t = 2^-23 |trig| (+ the smallest subnormal).
# - normal4_fast: a = fl(2pi_f32 (u - 0.5)), u - 0.5 exact, so |a~ - a| <= |u - 0.5| |2pi_f32 - 2pi| + 2^-24 |a|; __cosf and __sinf have
#   maximum absolute errors of 2^-21.19 and 2^-21.41 on [-pi, pi] (a reaches pi_f32, 8.7e-8 past pi, at u = 1).
#   e_t = |a~ - a| + that.
#
# The bound is these first-order terms evaluated at the float64 values, times SAFETY for the second-order terms that are left out and for
# evaluating ulp() at the exact rather than the computed value.
# ------------------------------------------------------------------------------------------------
SAFETY = 2.0
_TWO_PI_F32 = float(np.float32(2 * math.pi))
_NEG_2LN2_F32 = float(np.float32(-2 * math.log(2)))


def _ulp32(v):
    """ulp of float32 values near |v| (float64 array in, float64 array out)"""
    v = np.abs(v)
    e = np.floor(np.log2(np.where(v > 0, v, 1.0)))
    return np.where(v > 0, np.exp2(np.maximum(e, -126) - 23), 2.0 ** -149)


def _radius_err(u, fast):
    """(r, bound on |r~ - r|) for float32 uniforms u"""
    u = u.astype(np.float64)
    lg = np.log(u)
    m = -2.0 * lg
    r = np.sqrt(m)
    if fast:
        l2 = np.log2(u)
        e_log2 = np.where(u >= 0.5, 2.0 ** -22, 2 * _ulp32(l2))
        e_m = 2 * math.log(2) * e_log2 + 2.0 ** -23 * m
    else:
        e_m = 2 * _ulp32(lg)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_r = np.minimum(np.sqrt(e_m), np.where(r > 0, e_m / r, np.inf))
    return r, e_r + 2.0 ** -24 * r


def box_muller(bits, fast):
    """Philox output uint32 [..., 4] -> (z float64 [..., 4], bound float64 [..., 4]).
    fast = False: normal4 (angle 2 pi u), fast = True: normal4_fast (angle 2 pi (u - 0.5))."""
    u = u01(bits)
    z = np.empty(u.shape, dtype=np.float64)
    err = np.empty(u.shape, dtype=np.float64)
    for rl, al in ((0, 1), (2, 3)):
        r, e_r = _radius_err(u[..., rl], fast)
        ua = u[..., al].astype(np.float64)
        a = 2 * math.pi * (ua - 0.5) if fast else 2 * math.pi * ua
        c, s = np.cos(a), np.sin(a)
        if fast:
            e_a = np.abs(ua - 0.5) * abs(_TWO_PI_F32 - 2 * math.pi) + 2.0 ** -24 * np.abs(a)
            e_c, e_s = e_a + 2.0 ** -21.19, e_a + 2.0 ** -21.41
        else:
            e_c, e_s = 2.0 ** -23 * np.abs(c) + 2.0 ** -149, 2.0 ** -23 * np.abs(s) + 2.0 ** -149
        for lane, t, e_t in ((rl, c, e_c), (rl + 1, s, e_s)):
            z[..., lane] = r * t
            err[..., lane] = SAFETY * (np.abs(t) * e_r + r * e_t + e_r * e_t + 2.0 ** -24 * np.abs(r * t))
    return z, err


def _pairs(batch, per_sample, groups):
    """(sample index, group index) int64 arrays [batch, G]: all groups of every sample, or `groups` ([G] for every sample, or [batch, G])"""
    if groups is None:
        groups = np.arange(-(-per_sample // 4), dtype=np.int64)
    groups = np.broadcast_to(np.asarray(groups, dtype=np.int64), (batch, np.shape(groups)[-1]))
    return np.broadcast_to(np.arange(batch, dtype=np.int64)[:, None], groups.shape), groups


def _flat(v, groups, per_sample):
    """[B, G, 4] -> [B, per_sample] when every group was evaluated"""
    return v.reshape(v.shape[0], -1)[:, :per_sample] if groups is None else v


def noise_normal(seeds, stream_id, per_sample, groups=None, rounds=10):
    """noise_normal_kernel: (z, bound), float64 [B, per_sample], or [B, G, 4] for the given groups"""
    keys = seed_words(seeds)
    b, g = _pairs(len(keys), per_sample, groups)
    s = int(stream_id) & (2 ** 64 - 1)
    ctr = np.stack([g & 0xFFFFFFFF, g >> 32, np.full_like(g, s & 0xFFFFFFFF), np.full_like(g, (s >> 32) ^ TAG_NORMAL)], -1)
    z, err = box_muller(philox4x32_10(ctr.astype(np.uint32), keys[b], rounds), fast=False)
    return _flat(z, groups, per_sample), _flat(err, groups, per_sample)


# ------------------------------------------------------------------------------------------------
# Brownian tree
# ------------------------------------------------------------------------------------------------
class Lin:
    """A linear form sum_w c_w z_w over independent unit normals z_w, one per counter word (the same form holds in every lane).
    The walk below runs on these, so one walk gives every output's coefficients, its variance and its covariances exactly."""

    def __init__(self, terms=None):
        self.terms = dict(terms or {})

    def __add__(self, o):
        t = dict(self.terms)
        for w, c in o.terms.items():
            t[w] = t.get(w, 0.0) + c
        return Lin(t)

    def __sub__(self, o):
        return self + o * -1.0

    def __mul__(self, s):
        return Lin({w: c * s for w, c in self.terms.items()})

    __rmul__ = __mul__

    def dot(self, o):
        """E[self * other]"""
        return sum(c * o.terms.get(w, 0.0) for w, c in self.terms.items())

    def eval(self, z):
        """z: {word: array} -> sum_w c_w z[w]"""
        return sum(c * z[w] for w, c in self.terms.items())


def clamp(t, t_min, t_max):
    return min(max(t, t_min), t_max)


def walk(t, t_min, t_max, depth):
    """W(t) as a Lin, and every W value the walk forms on the way (root, midpoints), in the kernel's order.  t is taken as given (the
    kernel clamps first).  The kernel shares the walks to t0 and t1 above the level where they part; a shared node has the same counter
    in both walks, hence the same draw, so two independent walks give the same numbers."""
    a, b = t_min, t_max
    wa, wb = Lin(), math.sqrt(t_max - t_min) * Lin({1: 1.0})
    node, seen = 1, [wb]
    for _ in range(depth):
        mid = 0.5 * (a + b)
        wm = 0.5 * (wa + wb) + 0.5 * math.sqrt(b - a) * Lin({node + MID_OFFSET: 1.0})
        seen.append(wm)
        if t < mid:
            b, wb, node = mid, wm, 2 * node
        else:
            a, wa, node = mid, wm, 2 * node + 1
    f = (t - a) / (b - a) if b > a else 0.0
    return wa + f * (wb - wa), seen


def increment(t_min, t_max, t0, t1, depth):
    """The kernel's output as a Lin: (W(clamp t1) - W(clamp t0)) / sqrt(|t1 - t0|), the norm taken from the UNCLAMPED times as
    kdb_noise_brownian does, so outside [t_min, t_max] the variance drops below 1.  Also returns every W formed by both walks."""
    w0, s0 = walk(clamp(t0, t_min, t_max), t_min, t_max, depth)
    w1, s1 = walk(clamp(t1, t_min, t_max), t_min, t_max, depth)
    return (w1 - w0) * (1.0 / math.sqrt(abs(t1 - t0))), s0 + s1 + [w0, w1]


def brownian(seeds, per_sample, t_min, t_max, t0, t1, depth, groups=None):
    """noise_brownian_kernel: (out, bound), float64 [B, per_sample], or [B, G, 4] for the given groups.

    bound = SAFETY * (sum over draws of |coefficient| * Box-Muller bound of that draw
                      + 2 (2 depth + 3) 2^-24 max|W| / sqrt|t1 - t0| + 3 2^-24 |out|)
    The second term is the float32 rounding of the walks: per level one rounding of the midpoint mean and one of the fma, per walk the
    root product and the leaf fma with its rounded fraction; each is at most 2^-24 of a W the walk forms, and an error in W is carried
    on with weights that sum to at most 1.  The third is the final difference, the product by the norm and the norm's own rounding."""
    d, seen = increment(t_min, t_max, t0, t1, depth)
    keys = seed_words(seeds)
    b, g = _pairs(len(keys), per_sample, groups)
    words = sorted({w for form in seen for w in form.terms})
    z, ez = {}, {}
    for w in words:
        ctr = np.stack([g & 0xFFFFFFFF, g >> 32, np.full_like(g, w), np.full_like(g, TAG_BROWNIAN)], -1).astype(np.uint32)
        z[w], ez[w] = box_muller(philox4x32_10(ctr, keys[b]), fast=True)
    out = d.eval(z)
    intrinsic = Lin({w: abs(c) for w, c in d.terms.items()}).eval(ez)
    max_w = np.max(np.stack([np.abs(f.eval(z)) if f.terms else np.zeros_like(out) for f in seen]), axis=0)
    bound = SAFETY * (intrinsic + 2 * (2 * depth + 3) * 2.0 ** -24 * max_w / math.sqrt(abs(t1 - t0)) + 3 * 2.0 ** -24 * np.abs(out))
    return _flat(out, groups, per_sample), _flat(bound, groups, per_sample)


def search_seeds(counter, lane, targets, n_seeds=1 << 25, chunk=1 << 22):
    """Seeds s in [0, n_seeds) whose Philox output at `counter` (key = (s, 0)) has (r[lane] >> 8) in `targets`: {target: [seeds]}"""
    hits = {t: [] for t in targets}
    ctr = np.asarray(counter, dtype=np.uint32)
    for lo in range(0, n_seeds, chunk):
        s = np.arange(lo, min(lo + chunk, n_seeds), dtype=np.uint64)
        keys = np.stack([s & _M32, s >> np.uint64(32)], -1).astype(np.uint32)
        top = philox4x32_10(ctr, keys)[..., lane] >> np.uint32(8)
        for t in targets:
            hits[t].extend(int(v) for v in s[top == t])
    return hits
