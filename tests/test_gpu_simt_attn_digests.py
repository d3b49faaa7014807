"""The warp-per-query SIMT attention kernels bit for bit: SHA-256 digests of their outputs against tests/golden/simt_attn_digests.json.
These kernels carry every exact-path attention result: attn_generic_kernel<float> (the fp32 forward and the U-Net's self-attention),
attn_generic_kernel<bf16> (kdb_attention with fast = 0, the fallback of shapes the tensor-core kernels reject), attn_jvp_kernel and the
two VJP passes, attn_vjp_q_kernel and attn_vjp_kv_kernel.  They share one key walk, one softmax pass, one weighted sum and one launcher;
a change to any of them must leave every result bit where it was.

The geometries cover global attention over a token count that is not a multiple of 32 and at 64x66 tokens (the largest grid the
shared-memory budget accepts at d_head 64), shifted windows of 8 with shift 0 and 4 and of 4 with shift 2, and neighbourhood 7 on two long
axes and on a short one (9 < 2k, where one key is seen by every query of the axis), each at d_head 64 and 40.  Every output buffer, the VJP's
stats scratch included, starts as NaN, so an element left unwritten changes the digest and fails the finiteness check.

Record the golden (on the build whose results are the reference):  python tests/test_gpu_simt_attn_digests.py --record OUT.json
"""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
from test_gpu_attn_derivatives import make_qkv  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "simt_attn_digests.json"
DEV = "cuda"
SCALE = 10.0            # |q . k| bound of the inputs, the cosine-sim scale of a layer

# (kind, h, w, param, shift)
GEOMETRIES = [
    ("global", 5, 7, 0, 0),                  # 35 keys: one full and one partial lane-strided pass
    ("shifted-window", 16, 24, 8, 0),
    ("shifted-window", 16, 24, 8, 4),        # both seams masked
    ("shifted-window", 8, 12, 4, 2),
    ("neighborhood", 16, 18, 7, 0),          # both axes n >= 2k
    ("neighborhood", 9, 20, 7, 0),           # a short axis: the per-key query count reaches n
]
# (kind, h, w, param, shift, d_head, n_heads, batch)
CASES = [g + (e, 2, 2) for g in GEOMETRIES for e in (64, 40)] + [("global", 64, 66, 0, 0, 64, 1, 1)]


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def run(kind, h, w, param, shift, e, nh, B):
    """-> {output: digest} of the fp32 and bf16 forwards, the JVP and the VJP's dqkv and stats of one seeded case"""
    from k_diffusion import _native as N_
    T = h * w
    seed = h * 1000 + w * 10 + param + shift + e
    qkv = make_qkv(B, T, nh, e, SCALE, seed).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    dqkv = torch.randn(qkv.shape, generator=g).to(DEV)
    dout = torch.randn(B, T, nh * e, generator=g).to(DEV)
    code = N_._ATTN_CODE[kind]
    outs = {}
    for name, x, dtype, prec in (("forward fp32", qkv, torch.float32, N_.PREC_FP32),
                                 ("forward bf16", qkv.to(torch.bfloat16), torch.bfloat16, N_.PREC_BF16)):
        outs[name] = _nan((B, T, nh * e), dtype)
        N_.check(N_.lib().kdb_attention(prec, 0, N_.ptr(x), N_.ptr(outs[name]), B, h, w, nh, e, code, param, shift, None, N_.stream()))
    o = outs["forward fp32"]
    outs["jvp"] = N_.attention_jvp(qkv, dqkv, h, w, nh, e, kind, param, shift, out=_nan((B, T, nh * e)))
    outs["vjp stats"] = _nan((B, nh, T, 3))
    outs["vjp dqkv"] = N_.attention_vjp(qkv, o, dout, h, w, nh, e, kind, param, shift, dqkv=_nan(qkv.shape), stats=outs["vjp stats"])
    torch.cuda.synchronize()
    for name, t in outs.items():
        assert bool(torch.isfinite(t.float()).all()), f"{name}: an output element was not written"
    return {name: _digest(t) for name, t in outs.items()}


def _key(case):
    return " ".join(str(c) for c in case)


def _id(c):
    return f"{c[0]}-{c[1]}x{c[2]}-p{c[3]}-s{c[4]}-e{c[5]}-nh{c[6]}-B{c[7]}"


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_simt_attention_digests(golden, case):
    assert run(*case) == golden[_key(case)]


if __name__ == "__main__":
    assert len(sys.argv) == 3 and sys.argv[1] == "--record", __doc__
    rec = {}
    for case in CASES:
        rec[_key(case)] = run(*case)
        assert run(*case) == rec[_key(case)], f"{_key(case)}: two runs differ"
    Path(sys.argv[2]).write_text(json.dumps(rec, indent=1) + "\n")
    print(f"recorded {len(rec)} cases -> {sys.argv[2]}")
