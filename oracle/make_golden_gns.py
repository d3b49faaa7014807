#!/usr/bin/env python
"""Record the reference's gradient noise scale (k_diffusion/gns.py) from the REAL reference (run by hand, with $K_DIFFUSION_REFERENCE naming
a checkout; the reference's package imports with make_golden.py's stubs):

    python oracle/make_golden_gns.py   # -> tests/golden/gns.json

All on the CPU: the signatures of DDPGradientStatsHook's and GradientNoiseScale's public methods, and for seeded sequences of update()
arguments, each update's return value, get_gns, get_stats, and state_dict after every step.  The sequences cover per-sample and
per-rank small batches, estimates that go negative (the eps floor of the ratio), a non-default beta and eps, and a load_state_dict
round trip in the middle of a sequence."""
import inspect
import json
import random
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as G

SIGNATURES = ["DDPGradientStatsHook.__init__", "DDPGradientStatsHook.get_stats", "GradientNoiseScale.__init__",
              "GradientNoiseScale.state_dict", "GradientNoiseScale.load_state_dict", "GradientNoiseScale.update",
              "GradientNoiseScale.get_gns", "GradientNoiseScale.get_stats"]

# name: (constructor kwargs, n_small, n_large, steps, seed, step after which the state goes through load_state_dict or None)
CASES = {
    "default_per_rank": ({}, 32, 64, 40, 0, None),
    "default_per_sample": ({}, 1, 256, 25, 1, 12),
    "beta_0.9_eps_1e-3": (dict(beta=0.9, eps=1e-3), 16, 128, 60, 2, 30),
    "noisy_negative": (dict(beta=0.5), 8, 32, 50, 3, None),
}


def sig_of(fn):
    return [[name, p.kind.name, None if p.default is inspect._empty else repr(p.default)]
            for name, p in inspect.signature(fn).parameters.items()]


def draws(seed, steps, noisy):
    """(sq_norm_small_batch, sq_norm_large_batch) per step: positive norms where the small batch's is the larger, as a gradient's is on
    average; `noisy` swaps them on some steps, so that both estimates go negative there"""
    rng = random.Random(seed)
    out = []
    for _ in range(steps):
        large = rng.uniform(0.01, 5.0)
        small = large * rng.uniform(1.0, 4.0)
        if noisy and rng.random() < 0.4:
            small, large = large, small
        out.append((small, large))
    return out


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K
    gns = K.gns
    obj = {}
    for name in SIGNATURES:
        cls, meth = name.split(".")
        obj[name] = sig_of(getattr(getattr(gns, cls), meth))
    cases = {}
    for name, (kwargs, n_small, n_large, steps, seed, reload_at) in CASES.items():
        g = gns.GradientNoiseScale(**kwargs)
        seq = draws(seed, steps, name.startswith("noisy"))
        rec = dict(kwargs=kwargs, n_small=n_small, n_large=n_large, inputs=seq, reload_at=reload_at, initial=g.state_dict(),
                   returned=[], gns=[], stats=[], states=[])
        for i, (small, large) in enumerate(seq):
            rec["returned"].append(g.update(small, large, n_small, n_large))
            rec["gns"].append(g.get_gns())
            rec["stats"].append(list(g.get_stats()))
            rec["states"].append(g.state_dict())
            if i == reload_at:
                fresh = gns.GradientNoiseScale()
                fresh.load_state_dict(g.state_dict())
                g = fresh
        cases[name] = rec
    out = G.OUT / "gns.json"
    out.write_text(json.dumps(dict(signatures=obj, cases=cases), indent=1))
    print("wrote", out, len(cases), "cases")


if __name__ == "__main__":
    main()
