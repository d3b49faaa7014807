#!/usr/bin/env python
"""KID / FID fixtures from the REAL reference (checkout named by $K_DIFFUSION_REFERENCE), run on the CPU:

    python oracle/make_golden_metrics.py      # -> tests/golden/metrics.npz, tests/golden/metrics_meta.json

The reference's evaluation module imports cleanfid and clip at top level; both are stubbed in sys.modules first (make_golden.py).
Over seeded fp32 features at several shapes (d = 1, 7 and 2048; m != n; kid partitions whose bounds hit round() ties) it records the
inputs and the reference's own fp32 outputs of polynomial_kernel, squared_mmd, kid and fid, the float64 oracle's values
(oracle/metrics_oracle.py) and the reference's error against them -- the accuracy a native result has to match.  It also records the
row bounds of every partition the reference's kid hands to squared_mmd, and the signatures of the five public functions.
"""
import inspect
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np
import torch

import make_golden as G
import metrics_oracle as O

# name: (m, n, d, kid max_size, scale of the features)
CASES = {
    "d1": (40, 33, 1, 5000, 1.0),
    "d7": (96, 70, 7, 5000, 2.0),
    "d2048": (24, 17, 2048, 5000, 1.0),
    "ragged": (65, 129, 16, 5000, 1.0),
    "ties2": (45, 27, 8, 30, 1.0),        # 2 partitions: 22.5 -> 22 and 13.5 -> 14
    "ties6": (15, 33, 5, 6, 1.0),         # 6 partitions: 2.5 -> 2, 7.5 -> 8, 12.5 -> 12
}


def sig_of(fn):
    return [[name, p.kind.name, None if p.default is inspect._empty else repr(p.default)]
            for name, p in inspect.signature(fn).parameters.items()]


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    from k_diffusion import evaluation as E
    torch.set_num_threads(8)
    arrays, meta = {}, {"how": "reference evaluation.py on the CPU in fp32; oracle = oracle/metrics_oracle.py in float64; err = |ref - oracle|",
                        "signatures": {}, "cases": {}}
    for name in ("polynomial_kernel", "squared_mmd", "kid", "sqrtm_eig", "fid"):
        meta["signatures"][name] = sig_of(getattr(E, name))
    seen = []
    orig = E.squared_mmd

    def spy(x, y, *args, **kwargs):      # the partitions kid slices, as row bounds of its inputs
        seen.append((x, y))
        return orig(x, y, *args, **kwargs)

    for i, (name, (m, n, d, max_size, scale)) in enumerate(CASES.items()):
        g = torch.Generator().manual_seed(1000 + i)
        x = torch.randn(m, d, generator=g) * scale
        y = torch.randn(n, d, generator=g) * scale + 0.1
        x64, y64 = x.double().numpy(), y.double().numpy()
        rec = {}
        kxy = E.polynomial_kernel(x, y)
        arrays[f"{name}.x"], arrays[f"{name}.y"], arrays[f"{name}.kxy"] = x.numpy(), y.numpy(), kxy.numpy()
        ok = O.polynomial_kernel(x64, y64)
        rec["kernel_err"] = float(np.abs(kxy.double().numpy() - ok).max() / np.abs(ok).max())
        mmd = float(E.squared_mmd(x, y))
        terms = O.mmd_terms(x64, y64)
        rec["mmd"], rec["mmd_oracle"], rec["mmd_terms_oracle"] = mmd, float(terms[3]), [float(t) for t in terms[:3]]
        rec["mmd_err"] = abs(mmd - float(terms[3]))
        seen.clear()
        E.squared_mmd = spy
        try:
            kv = float(E.kid(x, y, max_size=max_size))
        finally:
            E.squared_mmd = orig
        base_x, base_y = x.data_ptr(), y.data_ptr()
        rec["kid_bounds_x"] = [(a.data_ptr() - base_x) // (4 * d) for a, _ in seen] + [m]
        rec["kid_bounds_y"] = [(b.data_ptr() - base_y) // (4 * d) for _, b in seen] + [n]
        assert [a.shape[0] for a, _ in seen] == list(np.diff(rec["kid_bounds_x"]))
        rec["max_size"] = max_size
        kt = O.kid_terms(x64, y64, max_size)
        rec["kid"], rec["kid_oracle"] = kv, float(O.kid(x64, y64, max_size))
        rec["kid_terms_oracle"] = [[float(v) for v in t] for t in kt]
        rec["kid_err"] = abs(kv - rec["kid_oracle"])
        rec["fid_oracle"] = O.fid(x64, y64)
        mu, cov = O.mean_cov(x64)
        if d > 1:      # at d = 1 torch.cov returns a 0-d tensor and the reference's fid raises IndexError
            fv = float(E.fid(x, y))
            rec["fid"], rec["fid_err"] = fv, abs(fv - rec["fid_oracle"])
        rec["cov_err"] = float(np.abs(torch.cov(x.T).double().numpy().reshape(d, d) - cov).max() / np.abs(cov).max())
        rec["mean_err"] = float(np.abs(x.mean(0).double().numpy() - mu).max() / max(np.abs(mu).max(), 1e-30))
        meta["cases"][name] = rec
        print(name, {k: v for k, v in rec.items() if k.endswith("err") or k.startswith("kid_bounds")})
    np.savez_compressed(G.OUT / "metrics.npz", **arrays)
    (G.OUT / "metrics_meta.json").write_text(json.dumps(meta, indent=1))


if __name__ == "__main__":
    main()
