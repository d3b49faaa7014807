"""The fp32 attention derivatives kernel by kernel: attn_jvp_kernel (kdb_attention_jvp) and the two passes of the VJP, attn_vjp_q_kernel and
attn_vjp_kv_kernel over QuerySet (kdb_attention_vjp), against float64 torch.func.jvp / torch.func.vjp of the oracle's global,
shifted-window and neighbourhood attention, at the key-set geometries tests/test_attn_sets_host.py checks on the host.

- Gate: check_tangent of tests/test_jvp_bound.py on the forward output, the JVP output and each third of dqkv (dq, dk, dv) separately.
- Support, with no tolerance: one image per query, nearly uniform softmax, an output gradient (or a v tangent) that is one-hot in the
  token.  The keys whose dk / dv come out nonzero must be exactly the keys the query sees, and the queries whose JVP output comes out
  nonzero exactly the queries that see the key.  A dropped or extra query of the per-key pass contributes P_ij times something, which the
  gate cannot see when the cosine-sim logits make P_ij ~ e^-20; here it shows as an exact zero or nonzero.
- Every output element written: outputs and scratch are NaN-filled before each call.
- Adjoint identity <dO, J v> = <J^T dO, v> from the two kernels alone.
- The shared-memory budget of the per-key pass (and of the JVP): global attention at 64x66 tokens, the largest it accepts at d_head 64,
  runs and matches; at 65x65 both entries return KDB_ERR_UNSUPPORTED before any launch.
"""
import pytest
import torch

from k_diffusion import _native
from oracle import kdiff_oracle as O
from test_attn_sets_host import shifted_window_token_allow
from test_jvp_bound import check_tangent

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"

# |<dO, J v> - <J^T dO, v>| / (|dO| |J v|) from the fp32 kernels, accumulated in float64: at most 3.8e-8 over the cases below, measured
# on an H100 80GB HBM3 (700 W power limit); the kernels are deterministic, so the bound leaves a margin of 5 for other GPUs and toolchains
ADJOINT_BOUND = 2e-7


def oracle_fn(kind, h, w, nh, e, param, shift):
    """qkv [B, h*w, 3*nh*e] -> attention output [B, h*w, nh*e] of the oracle, differentiable"""
    def f(qkv):
        B = qkv.shape[0]
        q, k, v = qkv.reshape(B, h, w, 3, nh, e).unbind(3)
        if kind == "global":
            o = O.global_attention(q, k, v)
        elif kind == "shifted-window":
            o = O.shifted_window_attention(q, k, v, param, shift)
        else:
            o = O.neighborhood_attention(q, k, v, param)
        return o.reshape(B, h * w, nh * e)
    return f


def allow_of(kind, h, w, param, shift):
    if kind == "global":
        return torch.ones(h * w, h * w, dtype=torch.bool)
    if kind == "shifted-window":
        return torch.from_numpy(shifted_window_token_allow(h, w, param, shift))
    return O.neighborhood_allow(h, w, param)


def make_qkv(B, T, nh, e, s, seed, q_norm=None):
    """qkv [B, T, 3*nh*e] fp32: q and k cosine-normalised to norm sqrt(s) as the layer leaves them (|q.k| <= s), v standard normal;
    q_norm overrides the norm of q"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(B, T, 3, nh, e, generator=g, dtype=torch.float64)
    t[:, :, :2] = t[:, :, :2] / t[:, :, :2].norm(dim=-1, keepdim=True) * s ** 0.5
    if q_norm is not None:
        t[:, :, 0] = t[:, :, 0] / t[:, :, 0].norm(dim=-1, keepdim=True) * q_norm
    return t.float().reshape(B, T, 3 * nh * e)


def nan_like(shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def native(qkv, dqkv, dout, h, w, nh, e, kind, param, shift):
    """-> (forward output, JVP output, dqkv of the VJP), each written into NaN-filled memory and checked finite"""
    B, T = qkv.shape[:2]
    qkv, dqkv, dout = qkv.to(DEV), dqkv.to(DEV), dout.to(DEV)
    o = _native.attention(qkv, h, w, nh, e, kind, param, shift)
    jv = _native.attention_jvp(qkv, dqkv, h, w, nh, e, kind, param, shift, out=nan_like((B, T, nh * e)))
    stats = nan_like((B, nh, T, 3))
    g = _native.attention_vjp(qkv, o, dout, h, w, nh, e, kind, param, shift, dqkv=nan_like(qkv.shape), stats=stats)
    torch.cuda.synchronize()
    for name, t in (("forward", o), ("JVP output", jv), ("dqkv", g), ("stats", stats)):
        assert bool(torch.isfinite(t).all()), f"{name}: {int((~torch.isfinite(t)).sum())} elements not written (or not finite)"
    return o.cpu(), jv.cpu(), g.cpu()


def thirds(t, nh, e):
    B, T = t.shape[:2]
    return t.reshape(B, T, 3, nh * e).unbind(2)


# (kind, h, w, param, shift).  Neighbourhood: square and non-square grids at k, k + 1, inside the band 3 (k/2) + 2 .. 2k - 1 where a key is
# seen by more than 3 (k/2) + 1 queries of an axis (k = 7 on 12x12: 144), at its edges and beyond 2k.  Shifted window: every window size
# of the host test with seam shifts, 1 to 3 windows per axis.
GEOMETRIES = [
    ("neighborhood", 2, 5, 1, 0), ("neighborhood", 3, 3, 3, 0), ("neighborhood", 5, 5, 3, 0), ("neighborhood", 4, 9, 3, 0),
    ("neighborhood", 5, 6, 5, 0), ("neighborhood", 8, 9, 5, 0), ("neighborhood", 13, 7, 5, 0),
    ("neighborhood", 7, 8, 7, 0), ("neighborhood", 12, 12, 7, 0), ("neighborhood", 11, 13, 7, 0), ("neighborhood", 10, 16, 7, 0),
    ("neighborhood", 14, 17, 7, 0), ("neighborhood", 15, 15, 9, 0), ("neighborhood", 9, 20, 9, 0), ("neighborhood", 19, 21, 11, 0),
    ("neighborhood", 11, 25, 11, 0), ("neighborhood", 22, 22, 13, 0), ("neighborhood", 29, 13, 13, 0),
    ("shifted-window", 1, 2, 1, 0), ("shifted-window", 4, 6, 2, 1), ("shifted-window", 9, 9, 3, 1), ("shifted-window", 3, 6, 3, 2),
    ("shifted-window", 8, 8, 4, 2), ("shifted-window", 12, 4, 4, 3), ("shifted-window", 4, 12, 4, 0), ("shifted-window", 16, 24, 8, 4),
    ("shifted-window", 8, 8, 8, 0), ("shifted-window", 24, 16, 8, 7),
    ("global", 1, 1, 0, 0), ("global", 1, 7, 0, 0), ("global", 5, 3, 0, 0), ("global", 16, 16, 0, 0),
]
# d_head, heads, images and logit scale cycle through the geometries so that every geometry kind meets each of them
CASES = [g + (e, nh, B, s) for i, g in enumerate(GEOMETRIES)
         for e, nh, B, s in [((8, 32, 64, 128)[i % 4], (1, 3)[i // 4 % 2], (1, 3)[i // 2 % 2], (10.0, 50.0)[i % 2])]]


def _id(c):
    return f"{c[0]}-{c[1]}x{c[2]}-p{c[3]}-s{c[4]}-e{c[5]}-nh{c[6]}-B{c[7]}-scale{int(c[8])}"


def check_near_zero(got, want_scale, what):
    """a derivative that is exactly zero in exact arithmetic (a query with one key: dS = P (dO.v - dO.O) = 0) is only rounding noise"""
    assert float(got.abs().max()) <= 1e-5 * want_scale, f"{what}: {float(got.abs().max()):.3e} where the exact value is 0"


@pytest.mark.parametrize("kind,h,w,param,shift,e,nh,B,s", CASES, ids=[_id(c) for c in CASES])
def test_derivatives_vs_float64_oracle(kind, h, w, param, shift, e, nh, B, s):
    T = h * w
    seed = h * 1000 + w * 10 + param + shift + e
    qkv = make_qkv(B, T, nh, e, s, seed)
    g = torch.Generator().manual_seed(seed + 1)
    dqkv = torch.randn(qkv.shape, generator=g)
    dout = torch.randn(B, T, nh * e, generator=g)
    o, jv, gq = native(qkv, dqkv, dout, h, w, nh, e, kind, param, shift)

    f = oracle_fn(kind, h, w, nh, e, param, shift)
    want_o, want_jv = torch.func.jvp(f, (qkv.double(),), (dqkv.double(),))
    _, pull = torch.func.vjp(f, qkv.double())
    (want_g,) = pull(dout.double())
    check_tangent(o, want_o, "forward")
    check_tangent(jv, want_jv, "JVP output")
    dv_scale = float(thirds(want_g, nh, e)[2].abs().max())
    for name, got, want in zip(("dq", "dk", "dv"), thirds(gq, nh, e), thirds(want_g, nh, e)):
        if float(want.norm()) == 0:
            check_near_zero(got, dv_scale * (s * e) ** 0.5, name)
        else:
            check_tangent(got, want, name)

    lhs = float((dout.double() * jv.double()).sum())
    rhs = float((gq.double() * dqkv.double()).sum())
    rel = abs(lhs - rhs) / float(dout.double().norm() * jv.double().norm())
    print(f"{_id((kind, h, w, param, shift, e, nh, B, s))}: adjoint identity {rel:.3e}")
    assert rel <= ADJOINT_BOUND, f"|<dO, J v> - <J^T dO, v>| / (|dO| |J v|) = {rel:.3e}"


# grids up to 13x13 from the geometries above and the host test (B = T images: one per query)
SUPPORT = [
    ("neighborhood", 12, 12, 7, 0), ("neighborhood", 11, 13, 7, 0), ("neighborhood", 8, 13, 7, 0), ("neighborhood", 7, 7, 7, 0),
    ("neighborhood", 13, 13, 13, 0), ("neighborhood", 9, 13, 9, 0), ("neighborhood", 11, 12, 11, 0), ("neighborhood", 8, 9, 5, 0),
    ("neighborhood", 12, 10, 5, 0), ("neighborhood", 5, 5, 3, 0), ("neighborhood", 4, 9, 3, 0), ("neighborhood", 2, 5, 1, 0),
    ("shifted-window", 12, 8, 4, 2), ("shifted-window", 12, 12, 4, 3), ("shifted-window", 9, 9, 3, 1), ("shifted-window", 6, 4, 2, 1),
    ("shifted-window", 8, 8, 8, 4), ("shifted-window", 3, 2, 1, 0),
    ("global", 5, 3, 0, 0), ("global", 1, 7, 0, 0), ("global", 1, 1, 0, 0), ("global", 13, 13, 0, 0),
]


@pytest.mark.parametrize("kind,h,w,param,shift", SUPPORT, ids=[f"{c[0]}-{c[1]}x{c[2]}-p{c[3]}-s{c[4]}" for c in SUPPORT])
def test_support_is_exactly_the_mask(kind, h, w, param, shift):
    """Image b: q of norm 1e-3 (P nearly uniform, nothing underflows), dO one-hot at query b -> dv_j, dk_j != 0 exactly for the keys j of
    query b, and dq nonzero at query b only; v tangent one-hot at key b -> JVP output nonzero exactly at the queries that see key b."""
    T = h * w
    B, nh, e = T, 1, 32
    allow = allow_of(kind, h, w, param, shift)
    qkv = make_qkv(B, T, nh, e, 10.0, T + param + shift, q_norm=1e-3)
    g = torch.Generator().manual_seed(T + 7)
    onehot = torch.zeros(B, T, 1)
    onehot[torch.arange(B), torch.arange(B)] = 1
    dout = onehot * torch.randn(B, 1, nh * e, generator=g)
    dqkv = torch.zeros(qkv.shape)
    dqkv[:, :, 2 * nh * e:] = onehot * torch.randn(B, 1, nh * e, generator=g)
    _, jv, gq = native(qkv, dqkv, dout, h, w, nh, e, kind, param, shift)
    dq, dk, dv = (t.ne(0).any(dim=-1) for t in thirds(gq, nh, e))
    jvz = jv.ne(0).any(dim=-1)

    one_key = allow.sum(dim=1) == 1        # dS = P (dO.v - dO.O) vanishes in exact arithmetic: its sign in fp32 is rounding
    for b in range(B):
        assert torch.equal(dv[b], allow[b]), (f"image {b}: dv nonzero at keys {dv[b].nonzero().flatten().tolist()}, "
                                              f"query {b} sees {allow[b].nonzero().flatten().tolist()}")
        if not one_key[b]:
            assert torch.equal(dk[b], allow[b]), (f"image {b}: dk nonzero at keys {dk[b].nonzero().flatten().tolist()}, "
                                                  f"query {b} sees {allow[b].nonzero().flatten().tolist()}")
            assert dq[b].nonzero().flatten().tolist() == [b], f"image {b}: dq nonzero at {dq[b].nonzero().flatten().tolist()}"
        assert torch.equal(jvz[b], allow[:, b]), (f"image {b}: JVP output nonzero at queries {jvz[b].nonzero().flatten().tolist()}, "
                                                  f"key {b} is seen by {allow[:, b].nonzero().flatten().tolist()}")


def test_shared_memory_budget_edge():
    """64x66 = 4224 tokens at d_head 64: 4 warps x (2 e + 3 T) floats = 200 KiB, the per-key pass's and the JVP's whole budget.  It runs and
    matches; at 65x65 both entry points refuse with KDB_ERR_UNSUPPORTED and launch nothing."""
    h, w, nh, e, s = 64, 66, 1, 64, 10.0
    T = h * w
    qkv = make_qkv(1, T, nh, e, s, 5)
    g = torch.Generator().manual_seed(6)
    dqkv = torch.randn(qkv.shape, generator=g)
    dout = torch.randn(1, T, nh * e, generator=g)
    o, jv, gq = native(qkv, dqkv, dout, h, w, nh, e, "global", 0, 0)
    f = oracle_fn("global", h, w, nh, e, 0, 0)
    want_o, want_jv = torch.func.jvp(f, (qkv.double(),), (dqkv.double(),))
    _, pull = torch.func.vjp(f, qkv.double())
    (want_g,) = pull(dout.double())
    check_tangent(o, want_o, "forward")
    check_tangent(jv, want_jv, "JVP output")
    for name, got, want in zip(("dq", "dk", "dv"), thirds(gq, nh, e), thirds(want_g, nh, e)):
        check_tangent(got, want, name)

    h = w = 65
    T = h * w
    qkv = torch.zeros(1, T, 3 * nh * e, device=DEV)
    out, stats = torch.zeros(1, T, nh * e, device=DEV), torch.zeros(1, nh, T, 3, device=DEV)
    L, p = _native.lib(), _native.ptr
    torch.cuda.synchronize()
    n0 = _native.launch_count()
    rc = L.kdb_attention_jvp(p(qkv), p(qkv), p(out), 1, h, w, nh, e, _native.ATTN_GLOBAL, 0, 0, _native.stream())
    assert rc == -2 and b"shared-memory" in L.kdb_last_error(), (rc, L.kdb_last_error())
    rc = L.kdb_attention_vjp(p(qkv), p(out), p(out), p(qkv), p(stats), 1, h, w, nh, e, _native.ATTN_GLOBAL, 0, 0, _native.stream())
    assert rc == -2 and b"shared-memory" in L.kdb_last_error(), (rc, L.kdb_last_error())
    assert _native.launch_count() == n0
    with pytest.raises(RuntimeError, match="shared-memory"):
        _native.attention_jvp(qkv, qkv, h, w, nh, e, "global")
