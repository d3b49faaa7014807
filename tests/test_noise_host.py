"""The host restatement of the noise kernels (oracle/counter_noise.py), on the CPU.

- Philox4x32-10 against the Random123 known-answer vectors, and the float32 edges of u01.
- The law of the Brownian tree, exactly rather than by sampling: W(t) is linear in the standard normals the tree draws, so the walk run
  on linear forms gives every W(t)'s coefficient vector, and covariances are dot products of those.
- BatchedBrownianTree's sign convention against the reference's rule (sampling.py:82-88 of k-diffusion), with the kernel replaced by the
  restatement.
- The per-element bound is a near miss: a float32 emulation of the kernels' arithmetic passes it, and each wrong kernel below fails it.
  Built for the GPU, all of them but t1_walk_wrong_node pass the moment tests of tests/test_gpu_parity.py, and every one fails
  tests/test_gpu_noise.py.
"""
import math

import numpy as np
import pytest
import torch

import k_diffusion as K
from oracle import counter_noise as N

S = K.sampling

KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


@pytest.mark.parametrize("counter,key,want", KAT)
def test_philox_known_answers(counter, key, want):
    got = N.philox4x32_10(np.array(counter, np.uint32), np.array(key, np.uint32))
    assert [int(v) for v in got] == list(want)
    batched = N.philox4x32_10(np.tile(np.array(counter, np.uint32), (3, 1)), np.tile(np.array(key, np.uint32), (3, 1)))
    assert (batched == got).all()


def test_u01_edges():
    top = lambda v: np.array([v << 8], np.uint32)                                    # noqa: E731
    assert N.u01(top(2 ** 24 - 1))[0] == np.float32(1.0)                             # + 2^-25 ties to even, up to 1
    assert N.u01(top(2 ** 24 - 2))[0] == np.float32(1 - 2.0 ** -23)
    assert N.u01(top(0))[0] == np.float32(2.0 ** -25)
    assert N.u01(top(0) | 0xFF)[0] == np.float32(2.0 ** -25)                         # the low 8 bits are dropped
    z, err = N.box_muller(np.array([(2 ** 24 - 1) << 8, 0, (2 ** 24 - 1) << 8, 1 << 30], np.uint32), fast=True)
    assert (z == 0).all() and np.isfinite(err).all()


def test_seed_words():
    assert N.seed_words([-1, 2 ** 32 + 5, 7]).tolist() == [[0xFFFFFFFF, 0xFFFFFFFF], [5, 1], [7, 0]]


# ------------------------------------------------------------------------------------------------
# the law of the tree
# ------------------------------------------------------------------------------------------------
T_MIN, T_MAX = 0.5, 4.5


def cov_matrix(ts, depth, t_min=T_MIN, t_max=T_MAX):
    forms = [N.walk(t, t_min, t_max, depth)[0] for t in ts]
    return np.array([[a.dot(b) for b in forms] for a in forms])


def test_covariance_exact_on_dyadic_grid():
    depth = 6
    ts = T_MIN + (T_MAX - T_MIN) * np.arange(2 ** depth + 1) / 2 ** depth
    got = cov_matrix(ts, depth)
    want = np.minimum.outer(ts, ts) - T_MIN
    assert np.abs(got - want).max() <= 1e-13 * (T_MAX - T_MIN)


@pytest.mark.parametrize("depth", [24, 30])
def test_covariance_exact_at_deep_dyadic_points(depth):
    rng = np.random.default_rng(depth)
    k = np.concatenate([rng.integers(0, 2 ** depth + 1, 30), [0, 1, 2 ** depth - 1, 2 ** depth]])
    ts = T_MIN + (T_MAX - T_MIN) * k / 2 ** depth                                      # exact in float64
    got = cov_matrix(ts, depth)
    want = np.minimum.outer(ts, ts) - T_MIN
    assert np.abs(got - want).max() <= 1e-13 * (T_MAX - T_MIN)


@pytest.mark.parametrize("depth", [1, 2, 5, 24])
def test_covariance_between_dyadic_points(depth):
    """Inside a leaf W is the linear interpolation of its ends: Cov(W(s), W(t)) = min(s, t) - t_min - leaf f_s (1 - f_t) for s <= t in
    one leaf (at most leaf / 4), and exactly min(s, t) - t_min across leaves."""
    leaf = (T_MAX - T_MIN) / 2 ** depth
    rng = np.random.default_rng(depth)
    ts = np.concatenate([rng.uniform(T_MIN, T_MAX, 40), T_MIN + leaf * (rng.integers(0, 2 ** min(depth, 20), 10) + rng.uniform(0, 1, 10))])
    if depth <= 5:                                                                   # several points in one leaf
        ts = np.concatenate([ts, T_MIN + leaf * (3 % 2 ** depth + np.array([0.1, 0.45, 0.5, 0.9]))])
    dev = np.minimum.outer(ts, ts) - T_MIN - cov_matrix(ts, depth)
    idx = np.floor((ts - T_MIN) / leaf)
    f = (ts - T_MIN) / leaf - idx
    same = idx[:, None] == idx[None, :]
    lo, hi = np.minimum.outer(f, f), np.maximum.outer(f, f)
    want = np.where(same, leaf * lo * (1 - hi), 0.0)
    assert np.abs(dev - want).max() <= 1e-12 * (T_MAX - T_MIN)
    assert dev.max() <= leaf / 4 * (1 + 1e-12) and dev.min() >= -1e-12


@pytest.mark.parametrize("depth", [2, 5, 24])
def test_disjoint_increments_uncorrelated(depth):
    leaf = (T_MAX - T_MIN) / 2 ** depth
    rng = np.random.default_rng(100 + depth)
    for _ in range(60):
        a, b, c, d = np.sort(rng.uniform(T_MIN, T_MAX, 4))
        if rng.random() < 0.5:                                                       # b and c in one leaf
            c = min(b + rng.uniform(0, leaf), d)
        wa, wb, wc, wd = (N.walk(t, T_MIN, T_MAX, depth)[0] for t in (a, b, c, d))
        assert abs((wb - wa).dot(wd - wc)) <= leaf / 4 * (1 + 1e-9)
        # increments between grid points are exactly uncorrelated
        ga, gb, gc, gd = (T_MIN + leaf * np.floor((t - T_MIN) / leaf) for t in (a, b, c, d))
        if gb <= gc:
            wa, wb, wc, wd = (N.walk(t, T_MIN, T_MAX, depth)[0] for t in (ga, gb, gc, gd))
            assert abs((wb - wa).dot(wd - wc)) <= 1e-13


def test_normalised_increment_variance_and_out_of_range():
    """In range and on the grid the normalised increment has variance exactly 1.  Outside [t_min, t_max] the kernel clamps t0 and t1 but
    normalises by the unclamped |t1 - t0|, so the variance is |clamped span| / |t1 - t0| < 1; pinned here as the current behaviour."""
    depth = 8
    d, _ = N.increment(T_MIN, T_MAX, 1.5, 3.75, depth)
    assert d.dot(d) == pytest.approx(1.0, abs=1e-13)
    d, _ = N.increment(T_MIN, T_MAX, 0.0, 5.5, depth)
    assert d.dot(d) == pytest.approx((T_MAX - T_MIN) / 5.5, abs=1e-13)
    d, _ = N.increment(T_MIN, T_MAX, 4.0, 6.0, depth)
    assert d.dot(d) == pytest.approx(0.5 / 2.0, abs=1e-13)
    d_rev, _ = N.increment(T_MIN, T_MAX, 3.75, 1.5, depth)
    d_fwd, _ = N.increment(T_MIN, T_MAX, 1.5, 3.75, depth)
    assert (d_rev + d_fwd).dot(d_rev + d_fwd) <= 1e-26


def test_batched_tree_sign_convention(monkeypatch):
    """BatchedBrownianTree(x, a, b)(s, t) = sign(b - a) sign(t - s) (W(max(s, t)) - W(min(s, t))) on the sorted interval, as the reference
    does, with the kernel replaced by the restatement."""
    from k_diffusion import _native
    monkeypatch.setattr(_native, "require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "noise_brownian", lambda like, seeds, t_min, t_max, t0, t1, depth: torch.from_numpy(
        N.brownian(seeds.tolist(), like[0].numel(), t_min, t_max, t0, t1, depth)[0]).reshape(like.shape))
    monkeypatch.setattr(_native, "lincomb", lambda ts, cs: sum(float(c) * t for t, c in zip(ts, cs)))
    x = torch.zeros(2, 3, 5)
    seeds = [5, -6]
    lo, hi, s, t = 2.0 ** -6, 160.0, 2.0, 40.0                                        # exact in float32, as the sampler converts
    base = N.brownian(seeds, 15, lo, hi, s, t, 24)[0].reshape(2, 3, 5) * math.sqrt(t - s)   # W(t) - W(s)
    for a, b in ((lo, hi), (hi, lo)):
        tree = S.BatchedBrownianTree(x, a, b, seed=seeds)
        for p, q in ((s, t), (t, s)):
            want = base * np.sign(b - a) * np.sign(q - p)
            np.testing.assert_allclose(tree(p, q).numpy(), want, rtol=1e-12, atol=1e-12)
    ns = S.BrownianTreeNoiseSampler(x, lo, hi, seed=seeds)
    np.testing.assert_allclose(ns(torch.tensor(t), torch.tensor(s)).numpy(), -base / math.sqrt(t - s), rtol=1e-12, atol=1e-12)
    single = S.BatchedBrownianTree(x, lo, hi, seed=9)
    want = N.brownian([9], 30, lo, hi, s, t, 24)[0].reshape(2, 3, 5)
    assert not single.batched and single.normalized(s, t).shape == x.shape
    np.testing.assert_allclose(single.normalized(s, t).numpy(), want, rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------
# near misses: a float32 emulation of the kernels passes the bound, wrong kernels fail it
# ------------------------------------------------------------------------------------------------
f32 = np.float32
NORMAL_MUTANTS = ["key_lo32", "stream_hi_dropped", "lanes_xy_swapped", "rounds9"]
BROWNIAN_MUTANTS = ["key_lo32", "lanes_xy_swapped", "rounds9", "leaf_snaps_to_endpoint", "t1_walk_wrong_node", "depth_clamped_24"]


def _keys(seeds, mutant):
    k = N.seed_words(seeds)
    if mutant == "key_lo32":
        k[:, 1] = 0
    return k


def emu_box_muller(bits, fast, mutant=None):
    """normal4 / normal4_fast in float32, each transcendental correctly rounded (within the bounds the guide gives)"""
    if mutant == "lanes_xy_swapped":
        bits = bits[..., [1, 0, 2, 3]]
    u = N.u01(bits).astype(np.float64)
    out = []
    for rl, al in ((0, 1), (2, 3)):
        if fast:
            m = f32(np.float64(f32(-2 * math.log(2))) * f32(np.log2(u[..., rl])))
            r = f32(np.sqrt(m.astype(np.float64)))
            a = f32(np.float64(f32(2 * math.pi)) * (u[..., al] - 0.5)).astype(np.float64)       # u - 0.5 is exact
        else:
            r = f32(np.sqrt(-2.0 * f32(np.log(u[..., rl])).astype(np.float64)))
            a = 2 * math.pi * u[..., al]                                                      # sincospif(2u)
        c, s = f32(np.cos(a)), f32(np.sin(a))
        out += [r * c, r * s]
    return np.stack(out, -1)


def emu_normal(seeds, stream_id, per_sample, mutant=None):
    keys = _keys(seeds, mutant)
    g = np.arange(-(-per_sample // 4), dtype=np.int64)[None, :].repeat(len(keys), 0)
    s = stream_id & (2 ** 64 - 1)
    hi = 0 if mutant == "stream_hi_dropped" else s >> 32
    ctr = np.stack([g & 0xFFFFFFFF, g >> 32, np.full_like(g, s & 0xFFFFFFFF), np.full_like(g, hi ^ N.TAG_NORMAL)], -1).astype(np.uint32)
    bits = N.philox4x32_10(ctr, keys[:, None, :], 9 if mutant == "rounds9" else 10)
    return emu_box_muller(bits, False, mutant).reshape(len(keys), -1)[:, :per_sample]


def fma32(a, b, c):
    return f32(np.float64(a) * np.float64(b) + np.float64(c))


def emu_brownian(seeds, per_sample, t_min, t_max, t0, t1, depth, mutant=None):
    """noise_brownian_kernel step by step in float32: the shared walk down to the split, one draw at the split, two walks below it"""
    keys = _keys(seeds, mutant)[:, None, :]
    g = np.arange(-(-per_sample // 4), dtype=np.int64)[None, :]
    rounds = 9 if mutant == "rounds9" else 10
    if mutant == "depth_clamped_24":
        depth = min(depth, 24)
    inv_norm = f32(1.0 / math.sqrt(abs(t1 - t0)))
    t0, t1 = N.clamp(t0, t_min, t_max), N.clamp(t1, t_min, t_max)
    split, a, b = depth, t_min, t_max
    for lv in range(depth):
        mid = 0.5 * (a + b)
        if (t0 < mid) != (t1 < mid):
            split = lv
            break
        a, b = (a, mid) if t0 < mid else (mid, b)

    def draw(word):
        ctr = np.stack(np.broadcast_arrays(g & 0xFFFFFFFF, g >> 32, word, N.TAG_BROWNIAN), -1).astype(np.uint32)
        return emu_box_muller(N.philox4x32_10(ctr, keys, rounds), True, mutant)

    def mid_draw(w):
        sd = f32(0.5 * math.sqrt(w["b"] - w["a"]))
        return fma32(sd, draw(w["node"] + N.MID_OFFSET), f32(0.5) * f32(w["wa"] + w["wb"]))

    def step(w, t, wm):
        mid = 0.5 * (w["a"] + w["b"])
        if t < mid:
            w.update(b=mid, wb=wm, node=2 * w["node"])
        else:
            w.update(a=mid, wa=wm, node=2 * w["node"] + 1)

    def finish(w, t):
        fr = f32((t - w["a"]) / (w["b"] - w["a"]))
        if mutant == "leaf_snaps_to_endpoint":
            fr = f32(round(float(fr)))
        return fma32(fr, f32(w["wb"] - w["wa"]), w["wa"])

    w0 = dict(a=t_min, b=t_max, wa=np.zeros((1, 1, 4), f32), wb=f32(f32(math.sqrt(t_max - t_min)) * draw(1)), node=1)
    for _ in range(split):
        step(w0, t0, mid_draw(w0))
    w1 = dict(w0)
    if split < depth:
        wm = mid_draw(w0)
        step(w0, t0, wm)
        step(w1, t1, wm)
        if mutant == "t1_walk_wrong_node":
            w1["node"] = w0["node"]
        for _ in range(split + 1, depth):
            step(w0, t0, mid_draw(w0))
            step(w1, t1, mid_draw(w1))
    out = f32(finish(w1, t1) - finish(w0, t0)) * inv_norm
    return out.reshape(len(seeds), -1)[:, :per_sample]


SEEDS = K.parallel.sample_seeds(3, 0, 3) + [-123456789, 2 ** 32 + 17]
NORMAL_CASES = [(1, 5), (2 ** 32 + 1, 75), (0x494E4954, 13), (2 ** 64 - 1, 8)]
# (t_min, t_max, t0, t1, depth): dyadic midpoints, one leaf, straddling the root midpoint, the interval ends, reversed, outside the range
BROWNIAN_CASES = [(0.25, 8.25, 2.25, 5.25, 5), (0.25, 8.25, 3.3, 3.4, 5), (0.25, 8.25, 4.2, 4.3, 24), (0.25, 8.25, 0.25, 8.25, 1),
                  (0.01, 160.0, 40.0, 2.0, 24), (0.25, 8.25, -1.0, 9.0, 2), (0.25, 8.25, 3.0 + 2.0 ** -22, 3.0 + 5 * 2.0 ** -25, 30),
                  (0.25, 8.25, 5.0, 7.5, 30)]


def _violations(got, want, bound):
    return int((np.abs(got.astype(np.float64) - want) > bound).sum())


def test_emulated_kernels_within_bound():
    for stream_id, per_sample in NORMAL_CASES:
        want, bound = N.noise_normal(SEEDS, stream_id, per_sample)
        assert _violations(emu_normal(SEEDS, stream_id, per_sample), want, bound) == 0
    for case in BROWNIAN_CASES:
        want, bound = N.brownian(SEEDS, 10, *case)
        assert _violations(emu_brownian(SEEDS, 10, *case), want, bound) == 0, case


@pytest.mark.parametrize("mutant", NORMAL_MUTANTS)
def test_normal_mutants_fail_the_bound(mutant):
    bad = sum(_violations(emu_normal(SEEDS, s, n, mutant), *N.noise_normal(SEEDS, s, n)) for s, n in NORMAL_CASES)
    assert bad > 0


@pytest.mark.parametrize("mutant", BROWNIAN_MUTANTS)
def test_brownian_mutants_fail_the_bound(mutant):
    bad = sum(_violations(emu_brownian(SEEDS, 10, *c, mutant=mutant), *N.brownian(SEEDS, 10, *c)) for c in BROWNIAN_CASES)
    assert bad > 0
