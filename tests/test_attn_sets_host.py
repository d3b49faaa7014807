"""The SIMT attention kernels' key sets (KeySet) and their inverse (QuerySet) against the oracle's attention masks, exactly, on the host.

tests/attn_sets_host.cpp compiles k-diffusion_b200/csrc/attn_sets.cuh as plain C++ and enumerates both sets at every geometry below.
KeySet(q) must be row q of the oracle's allow matrix and QuerySet(k) column k, with no duplicates and -1 exactly where the seam mask hides
a window entry.  QuerySet::max_count sizes each warp's shared-memory slot of the VJP's per-key pass (attn_vjp_kv_kernel), so every key's
count must fit it; for neighbourhood attention it must also be reached, so the slot is not oversized.

Neighbourhood grid sides cover k, k + 1, 3 (k/2) + 1, 3 (k/2) + 2, the middle of 3 (k/2) + 2 .. 2k - 1, 2k - 1, 2k and 2k + 3 in every
pair: below 2k the windows clamped at the two borders overlap and a middle key is seen by every query of the axis (k = 7 on 12x12: 144
queries for one key).
"""
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import kdiff_oracle as O

GLOBAL, NEIGHBORHOOD, SHIFTED_WINDOW = 1, 2, 3      # KDB_ATTN_* of include/kdiffusion_b200.h


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = tmp_path_factory.mktemp("attn_sets") / "attn_sets_host"
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT / "include"),
                    "-I", str(ROOT / "k-diffusion_b200" / "csrc"), str(ROOT / "tests" / "attn_sets_host.cpp"), "-o", str(exe)], check=True)

    def run(geoms):
        """geoms: [(type, h, w, param, shift)] -> [(max_count, keys [T, nk], query counts [T], queries [T, T])]"""
        text = "".join(f"{t} {h} {w} {p} {s}\n" for t, h, w, p, s in geoms)
        raw = np.frombuffer(subprocess.run([str(exe)], input=text.encode(), check=True, capture_output=True).stdout, dtype=np.int32)
        out, at = [], 0
        for _ in geoms:
            T, nk, maxq = (int(v) for v in raw[at:at + 3])
            at += 3
            keys = raw[at:at + T * nk].reshape(T, nk)
            at += T * nk
            qs = raw[at:at + T * (T + 1)].reshape(T, T + 1)
            at += T * (T + 1)
            out.append((maxq, keys, qs[:, 0], qs[:, 1:]))
        assert at == raw.size
        return out
    return run


def shifted_window_token_allow(h, w, ws, shift):
    """O.shifted_window_allow (per window, in the rolled frame) as a token-by-token [h*w, h*w] matrix of the unrolled image"""
    win = O.shifted_window_allow(h // ws, w // ws, ws, shift).numpy()
    ri, rj = np.divmod(np.arange(h * w), w)
    ri, rj = (ri + shift) % h, (rj + shift) % w                  # where each token lands in the rolled image
    wi, wj, li, lj = ri // ws, rj // ws, ri % ws, rj % ws
    same = (wi[:, None] == wi[None, :]) & (wj[:, None] == wj[None, :])
    local = li * ws + lj
    return same & win[wi[:, None], wj[:, None], local[:, None], local[None, :]]


def allow_of(type_, h, w, param, shift):
    if type_ == NEIGHBORHOOD:
        return O.neighborhood_allow(h, w, param).numpy()
    if type_ == SHIFTED_WINDOW:
        return shifted_window_token_allow(h, w, param, shift)
    return np.ones((h * w, h * w), dtype=bool)


def _dense(tokens, valid, T):
    """set membership [rows, T] of the valid entries of tokens [rows, n], and how many valid entries each row has"""
    m = np.zeros((tokens.shape[0], T), dtype=bool)
    rows = np.broadcast_to(np.arange(tokens.shape[0])[:, None], tokens.shape)
    m[rows[valid], tokens[valid]] = True
    return m, valid.sum(axis=1)


def check_geometry(geom, result):
    """-> list of failure descriptions for one geometry"""
    type_, h, w, param, shift = geom
    maxq, keys, qcount, queries = result
    T = h * w
    name = f"{['', 'global', 'neighborhood', 'shifted-window'][type_]} param={param} shift={shift} {h}x{w}"
    allow = allow_of(type_, h, w, param, shift)
    bad = []

    if not ((keys == -1) | ((keys >= 0) & (keys < T))).all():
        return [f"{name}: KeySet token out of range"]
    kset, kn = _dense(keys, keys >= 0, T)
    if (kn != kset.sum(axis=1)).any():
        bad.append(f"{name}: KeySet of query {int(np.argmax(kn != kset.sum(axis=1)))} repeats a key")
    if not np.array_equal(kset, allow):
        q = int(np.argmax((kset != allow).any(axis=1)))
        bad.append(f"{name}: KeySet of query {q} is {sorted(np.flatnonzero(kset[q]))}, the mask allows {sorted(np.flatnonzero(allow[q]))}")
    masked = (keys == -1).sum(axis=1)
    if type_ != SHIFTED_WINDOW and masked.any():
        bad.append(f"{name}: KeySet masks {int(masked.max())} keys of a kind without a mask")

    over = np.flatnonzero(qcount > maxq)
    if over.size:
        k = int(over[np.argmax(qcount[over])])
        bad.append(f"{name}: key {k} is seen by {int(qcount[k])} queries > QuerySet::max_count {maxq}")
    if (qcount < 0).any() or (qcount > T).any():
        return bad + [f"{name}: QuerySet count out of [0, {T}]"]
    cols = np.arange(T)[None, :]
    in_set = cols < qcount[:, None]
    if (queries[~in_set] != -2).any() or not ((queries[in_set] == -1) | ((queries[in_set] >= 0) & (queries[in_set] < T))).all():
        return bad + [f"{name}: QuerySet token out of range"]
    qset, qn = _dense(queries, in_set & (queries >= 0), T)
    if (qn != qset.sum(axis=1)).any():
        bad.append(f"{name}: QuerySet of key {int(np.argmax(qn != qset.sum(axis=1)))} repeats a query")
    if not np.array_equal(qset, allow.T):
        k = int(np.argmax((qset != allow.T).any(axis=1)))
        bad.append(f"{name}: QuerySet of key {k} is {sorted(np.flatnonzero(qset[k]))}, the mask gives {sorted(np.flatnonzero(allow[:, k]))}")
    if type_ == NEIGHBORHOOD and int(qcount.max()) != maxq:
        bad.append(f"{name}: QuerySet::max_count {maxq} but at most {int(qcount.max())} queries see one key (slot oversized)")
    return bad


def neighborhood_sides(k):
    """k, k + 1, 2k, 2k + 3, and both ends and the middle of the band 3 (k/2) + 2 .. 2k - 1, where a key can be seen by more than
    3 (k/2) + 1 queries of an axis, with the side just below it"""
    lo, hi = 3 * (k // 2) + 2, 2 * k - 1
    return sorted({k, k + 1, lo - 1, lo, (lo + hi) // 2, hi, 2 * k, 2 * k + 3})


def run_and_check(harness, geoms):
    bad = []
    for geom, result in zip(geoms, harness(geoms)):
        bad += check_geometry(geom, result)
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:100])


@pytest.mark.parametrize("k", [1, 3, 5, 7, 9, 11, 13])
def test_neighborhood_sets_match_the_mask(harness, k):
    sides = neighborhood_sides(k)
    run_and_check(harness, [(NEIGHBORHOOD, h, w, k, 0) for h in sides for w in sides])


@pytest.mark.parametrize("ws", [1, 2, 3, 4, 8])
def test_shifted_window_sets_match_the_mask(harness, ws):
    run_and_check(harness, [(SHIFTED_WINDOW, nh * ws, nw * ws, ws, s) for s in range(ws) for nh in (1, 2, 3) for nw in (1, 2, 3)])


def test_global_sets_match_the_mask(harness):
    run_and_check(harness, [(GLOBAL, h, w, 0, 0) for h, w in ((1, 1), (1, 7), (5, 3))])


def test_the_oracle_masks_are_what_the_sets_are_checked_against():
    """The token-level shifted-window mask built here is the one O.shifted_window_attention applies: attention with that mask over the
    unrolled tokens gives the oracle's output."""
    g = torch.Generator().manual_seed(0)
    h, w, ws, shift = 8, 12, 4, 2
    q, k, v = (torch.randn(1, h, w, 1, 8, generator=g, dtype=torch.float64) for _ in range(3))
    allow = torch.from_numpy(shifted_window_token_allow(h, w, ws, shift))
    flat = lambda t: t.reshape(1, h * w, 8)
    logits = (flat(q) @ flat(k).transpose(-1, -2)).masked_fill(~allow, float("-inf"))
    want = O.shifted_window_attention(q, k, v, ws, shift).reshape(1, h * w, 8)
    assert torch.allclose(torch.softmax(logits, -1) @ flat(v), want, rtol=1e-12, atol=1e-12)
