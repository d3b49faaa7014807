"""noise_normal_kernel and noise_brownian_kernel (csrc/solver.cu) value by value against the float64 restatement of their counter streams,
oracle/counter_noise.py, within its per-element bound.

- Every output is a view into a NaN-filled buffer with a NaN guard after it (and, for the offset cases, before it): every element must be
  written and nothing outside the view touched.  An offset of one float puts each sample's start off the 16-byte grid, so the kernels take
  their scalar store path.
- Seeds that differ only in the high word, negative seeds and parallel.sample_seeds values; stream ids whose high word is nonzero.
- init_noise and PhiloxNoiseSampler are pinned to the stream each uses.
- The Brownian tree at depths 1 to 30, at times on dyadic midpoints, inside one leaf, straddling the root midpoint, at the interval ends,
  reversed and outside the interval; the single-seed tree; the cfg4 shape (32 x 3x256x256) on a sample of groups.
- Extreme uniforms, hit on purpose with seeds found by counter_noise.search_seeds and re-verified here: u = 1.0f (r = 0, output exactly 0),
  u = 1 - 2^-23 (r = 4.9e-4, where the fast log's absolute error matters most) and u = 2^-25 (r = 5.89, the largest radius).
"""
import math

import numpy as np
import pytest
import torch

import k_diffusion as K
from k_diffusion import _native
from oracle import counter_noise as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
S = K.sampling
INIT = K.parallel._INIT_STREAM
GUARD = 37
WORST = {}          # kernel -> largest |error| / bound seen, printed at the end of the module (pytest -s)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nlargest |kernel - restatement| / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def nan_view(batch, per_sample, offset=0):
    buf = torch.full((offset + batch * per_sample + GUARD,), float("nan"), device=DEV)
    return buf, buf[offset:offset + batch * per_sample].view(batch, per_sample)


def check(kernel, buf, out, offset, want, bound, what):
    """every element of out written, nothing around it, and |out - want| <= bound element by element"""
    torch.cuda.synchronize()
    n = out.numel()
    assert torch.isnan(buf[:offset]).all() and torch.isnan(buf[offset + n:]).all(), f"{what}: wrote outside its output"
    got = out.double().cpu().numpy()
    assert np.isfinite(got).all(), f"{what}: {int((~np.isfinite(got)).sum())} elements not written"
    ratio = np.abs(got - want) / bound
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio.max() <= 1, f"{what}: {int((ratio > 1).sum())} elements out of bound, worst at {worst}: {got[worst]!r} vs {want[worst]!r} +- {bound[worst]:.3g}"
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(ratio.max()))
    return got


def seed_tensor(seeds):
    return torch.tensor(seeds, dtype=torch.int64, device=DEV)


def run_normal(seeds, stream_id, per_sample, offset=0):
    buf, out = nan_view(len(seeds), per_sample, offset)
    _native.noise_normal(out, seed_tensor(seeds), stream_id, out=out)
    want, bound = N.noise_normal(seeds, stream_id, per_sample)
    return check("noise_normal", buf, out, offset, want, bound, f"noise_normal(stream {stream_id}, per_sample {per_sample}, offset {offset})")


def run_brownian(seeds, per_sample, t_min, t_max, t0, t1, depth, offset=0):
    buf, out = nan_view(len(seeds), per_sample, offset)
    _native.noise_brownian(out, seed_tensor(seeds), t_min, t_max, t0, t1, depth, out=out)
    want, bound = N.brownian(seeds, per_sample, t_min, t_max, t0, t1, depth)
    return check("noise_brownian", buf, out, offset, want, bound, f"noise_brownian({t_min}, {t_max}, {t0!r}, {t1!r}, depth {depth}, offset {offset})")


BASE = 0x1234ABCD
SEED_POOL = [BASE, BASE + 2 ** 32, BASE + 2 ** 33 + 2 ** 62, -1, -BASE] + K.parallel.sample_seeds(11, 0, 5)
STREAMS = [1, 2 ** 32 + 1, INIT, 2 ** 64 - 1]


# ------------------------------------------------------------------------------------------------
# Philox normals
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("per_sample", [1, 3, 4, 5, 75, 4099, 3 * 256 * 256])
def test_noise_normal_shapes(per_sample, offset):
    batch = 1 + (per_sample + offset) % 5
    i = per_sample % len(SEED_POOL)
    seeds = (SEED_POOL * 2)[i:i + batch]
    run_normal(seeds, STREAMS[(per_sample + offset) % len(STREAMS)], per_sample, offset)


@pytest.mark.parametrize("stream_id", STREAMS)
def test_noise_normal_seeds_and_streams(stream_id):
    got = run_normal(SEED_POOL, stream_id, 75)
    assert not np.array_equal(got[0], got[1]) and not np.array_equal(got[0], got[2])      # the high word of the seed counts


def test_init_noise_and_sampler_streams():
    seeds = K.parallel.sample_seeds(5, 0, 3)
    shape, per_sample = (3, 8, 9), 216
    x = K.parallel.init_noise(seeds, shape, 80.0, DEV).double().cpu().numpy().reshape(3, -1)
    want, bound = N.noise_normal(seeds, INIT, per_sample)
    assert (np.abs(x - 80 * want) <= 80 * bound + 2.0 ** -23 * np.abs(80 * want)).all()
    like = torch.empty(3, *shape, device=DEV)
    for base in (1, 7):
        smp = S.PhiloxNoiseSampler(like, seeds, stream_base=base)
        for call in (1, 2):
            got = smp(1.0, 0.5).double().cpu().numpy().reshape(3, -1)
            want, bound = N.noise_normal(seeds, base + call, per_sample)
            assert (np.abs(got - want) <= bound).all(), f"PhiloxNoiseSampler(stream_base={base}) call {call}"


# ------------------------------------------------------------------------------------------------
# Brownian tree
# ------------------------------------------------------------------------------------------------
T_MIN, T_MAX = 0.25, 8.25


def placements(depth):
    span, leaf = T_MAX - T_MIN, (T_MAX - T_MIN) / 2 ** depth
    mid, k = 0.5 * (T_MIN + T_MAX), 2 ** depth // 3
    return {
        "dyadic": (T_MIN + leaf * k, T_MIN + leaf * (2 ** depth - 1)),
        "one_leaf": (T_MIN + leaf * (k + 0.2), T_MIN + leaf * (k + 0.7)),
        "straddle_root": (mid - 0.3 * leaf, mid + 0.4 * leaf),
        "ends": (T_MIN, T_MAX),
        "reversed": (T_MIN + 0.7 * span, T_MIN + 0.2 * span),
        "outside": (T_MIN - 1.0, T_MAX + 2.0),
    }


@pytest.mark.parametrize("where", ["dyadic", "one_leaf", "straddle_root", "ends", "reversed", "outside"])
@pytest.mark.parametrize("depth", [1, 2, 5, 24, 30])
def test_noise_brownian(depth, where):
    t0, t1 = placements(depth)[where]
    run_brownian(SEED_POOL[:3] + SEED_POOL[5:7], 75, T_MIN, T_MAX, t0, t1, depth)


@pytest.mark.parametrize("per_sample,offset", [(1, 1), (5, 0), (4099, 1)])
def test_noise_brownian_unaligned(per_sample, offset):
    run_brownian(SEED_POOL[3:7], per_sample, 0.01, 160.0, 2.0, 40.0, 24, offset)


def test_single_seed_tree_and_sampler():
    like = torch.empty(2, 3, 5, 7, device=DEV)
    tree = S.BatchedBrownianTree(like, 0.01, 160.0, seed=3)
    assert not tree.batched
    got = tree.normalized(2.0, 40.0).double().cpu().numpy().reshape(1, -1)
    want, bound = N.brownian([3], 210, 0.01, 160.0, 2.0, 40.0, 24)
    assert (np.abs(got - want) <= bound).all()
    scaled = tree(2.0, 40.0).double().cpu().numpy().reshape(1, -1)
    assert (np.abs(scaled - got * math.sqrt(38.0)) <= 2.0 ** -22 * np.abs(scaled)).all()
    seeds = K.parallel.sample_seeds(9, 0, 2)
    ns = S.BrownianTreeNoiseSampler(like, 0.01, 160.0, seed=seeds)
    lo, hi = float(torch.tensor(0.01)), float(torch.tensor(160.0))                          # the sampler's float32 times
    got = ns(torch.tensor(40.0), torch.tensor(2.0)).double().cpu().numpy().reshape(2, -1)
    want, bound = N.brownian(seeds, 105, lo, hi, 40.0, 2.0, 24)
    assert (np.abs(got - want) <= bound).all()


def test_cfg4_shape():
    """B = 32 at 3x256x256, one Karras step of the cfg4 schedule: the first and last group of every sample and 64 random ones"""
    seeds = K.parallel.sample_seeds(123, 0, 32)
    like = torch.empty(32, 3, 256, 256, device=DEV)
    ns = S.BrownianTreeNoiseSampler(like, 1e-2, 160.0, seed=seeds)
    sig = [float(v) for v in S.get_sigmas_karras(50, 1e-2, 160.0).tolist()]
    lo, hi = float(torch.tensor(1e-2)), float(torch.tensor(160.0))
    per_sample, gps = 3 * 256 * 256, 3 * 256 * 256 // 4
    rng = np.random.default_rng(4)
    groups = np.concatenate([np.tile([0, gps - 1], (32, 1)), rng.integers(0, gps, (32, 64))], axis=1)
    for i in (0, 25, 48):
        got = ns(torch.tensor(sig[i]), torch.tensor(sig[i + 1])).view(32, gps, 4)
        assert torch.isfinite(got).all()
        got = got.double().cpu().numpy()[np.arange(32)[:, None], groups]
        want, bound = N.brownian(seeds, per_sample, lo, hi, sig[i], sig[i + 1], 24, groups)
        ratio = np.abs(got - want) / bound
        assert ratio.max() <= 1, f"step {i}: {int((ratio > 1).sum())} elements out of bound"
        WORST["noise_brownian"] = max(WORST.get("noise_brownian", 0.0), float(ratio.max()))


# ------------------------------------------------------------------------------------------------
# extreme uniforms
# ------------------------------------------------------------------------------------------------
U_ONE, U_1M, U_MIN = 2 ** 24 - 1, 2 ** 24 - 2, 0          # x >> 8 for u = 1.0f, 1 - 2^-23, 2^-25
NORMAL_CTR = [0, 0, INIT & 0xFFFFFFFF, (INIT >> 32) ^ N.TAG_NORMAL]                    # group 0 of the init_noise stream
ROOT_CTR = [0, 0, 1, N.TAG_BROWNIAN]                                                    # group 0 of the Brownian root draw
# {(lane, x >> 8): seeds}, from counter_noise.search_seeds over seeds [0, 2^27)
NORMAL_HITS = {(0, U_ONE): [13732560, 23775063, 28494847], (0, U_1M): [37715234, 71440062, 84534969], (0, U_MIN): [1624595, 5204274],
               (2, U_ONE): [12630174, 13312293], (2, U_1M): [9525132, 19615828, 22510305], (2, U_MIN): [2883588, 14770117]}
ROOT_HITS = {(0, U_ONE): [5444583, 9942305, 19242427], (0, U_1M): [8732255], (0, U_MIN): [3755712],
             (2, U_ONE): [34997463, 50666019], (2, U_1M): [15505204, 27090550], (2, U_MIN): [35945920, 42811735]}


def extreme(hits, counter, got, want):
    """re-verify the recorded seeds, then: u = 1 gives exactly 0, and the largest |error| at u = 1 - 2^-23 and at u = 2^-25"""
    seeds = [s for v in hits.values() for s in v]
    bits = N.philox4x32_10(np.array(counter, np.uint32), N.seed_words(seeds))
    errs = {U_1M: 0.0, U_MIN: 0.0}
    row = 0
    for (lane, top), ss in hits.items():
        for _ in ss:
            assert bits[row, lane] >> 8 == top, f"seed {seeds[row]} no longer gives x >> 8 = {top} in lane {lane}"
            pair = [lane, lane + 1]
            if top == U_ONE:
                assert (got[row, pair] == 0).all(), f"u = 1.0f must give exactly 0, got {got[row, pair]}"
            else:
                errs[top] = max(errs[top], float(np.abs(got[row, pair] - want[row, pair]).max()))
            row += 1
    return seeds, errs


def test_extreme_uniforms_normal():
    seeds = [s for v in NORMAL_HITS.values() for s in v]
    got = run_normal(seeds, INIT, 4)
    want, _ = N.noise_normal(seeds, INIT, 4)
    _, errs = extreme(NORMAL_HITS, NORMAL_CTR, got, want)
    print(f"\nnormal4: largest |error| at u = 1 - 2^-23: {errs[U_1M]:.3g}, at u = 2^-25: {errs[U_MIN]:.3g}")


def test_extreme_uniforms_brownian_root():
    """depth 1, t0 = t_min, t1 = t_max: the output is the root draw itself (through sqrt(T) and back)"""
    seeds = [s for v in ROOT_HITS.values() for s in v]
    got = run_brownian(seeds, 4, T_MIN, T_MAX, T_MIN, T_MAX, 1)
    want, _ = N.brownian(seeds, 4, T_MIN, T_MAX, T_MIN, T_MAX, 1)
    root, _ = N.box_muller(N.philox4x32_10(np.array(ROOT_CTR, np.uint32), N.seed_words(seeds)), fast=True)
    assert np.allclose(want, root, rtol=1e-14, atol=1e-15)
    _, errs = extreme(ROOT_HITS, ROOT_CTR, got, want)
    print(f"\nnormal4_fast: largest |error| at u = 1 - 2^-23: {errs[U_1M]:.3g}, at u = 2^-25: {errs[U_MIN]:.3g}")
