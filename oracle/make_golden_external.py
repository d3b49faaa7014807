#!/usr/bin/env python
"""The reference's external model wrappers (k_diffusion/external.py) as data, recorded from the REAL reference (build container only):

    python oracle/make_golden_external.py      # -> tests/golden/external.npz, tests/golden/external_signatures.json

Records the signatures of the six wrappers' public methods; their noise tables and sigma_to_t on a Stable Diffusion schedule, quantized
and not, at table entries, midpoints, below the minimum, above the maximum and at 0; forward outputs around the toy models of
oracle/external_oracle.py (fp32 and fp16 eps, learned-variance eps, v); the gradient of a scalar loss with respect to x; and Euler, Heun,
DPM++(2M), LMS and Euler-ancestral (recorded noise) trajectories.  Everything runs on the CPU in fp32."""
import inspect
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np
import torch

import make_golden as G
from oracle import external_oracle as E

CLASSES = ("VDenoiser", "DiscreteEpsDDPMDenoiser", "OpenAIDenoiser", "CompVisDenoiser", "DiscreteVDDPMDenoiser", "CompVisVDenoiser")
METHODS = ("__init__", "get_scalings", "sigma_to_t", "t_to_sigma", "get_eps", "get_v", "loss", "forward")


def signatures(ext):
    out = {}
    for cls in CLASSES:
        obj = getattr(ext, cls)
        for m in METHODS:
            if hasattr(obj, m):
                out[f"external.{cls}.{m}"] = [[n, p.kind.name, None if p.default is inspect._empty else repr(p.default)]
                                              for n, p in inspect.signature(getattr(obj, m)).parameters.items()]
    return out


def queries(log_sigmas):
    """sigma_to_t probes: every 37th table entry, midpoints (in log space) between neighbours, below the minimum, above the maximum, 0"""
    ls = log_sigmas
    idx = torch.arange(0, len(ls), 37)
    mids = ((ls[idx[:-1]] + ls[idx[:-1] + 1]) / 2).exp()
    return torch.cat([ls[idx].exp(), mids, ls[0:1].exp() * 0.5, ls[-1:].exp() * 2, torch.tensor([1e-6, 0.0])])


def main():
    G._stub_missing()
    sys.path.insert(0, str(G.REF))
    import k_diffusion as K
    ext, S = K.external, K.sampling
    torch.set_num_threads(8)
    rec = {}

    # ------------------------------------------------------------------ schedules and sigma_to_t
    ac = E.sd_alphas_cumprod()
    toy_cv = E.ToyCompVis(4)
    for quantize in (False, True):
        w = ext.CompVisDenoiser(toy_cv, quantize=quantize)
        q = queries(w.log_sigmas)
        rec[f"cv_q{int(quantize)}_query"] = q
        rec[f"cv_q{int(quantize)}_t"] = w.sigma_to_t(q)
    rec["sigmas"], rec["log_sigmas"] = w.sigmas, w.log_sigmas
    rec["get_sigmas_12"] = w.get_sigmas(12)
    oa = ext.OpenAIDenoiser(E.ToyModel(3, learned_sigmas=True), E.ToyDiffusion())
    rec["openai_sigmas"] = oa.sigmas
    vq = torch.tensor([0.0, 1e-3, 0.5, 1.0, 3.0, 14.6, 80.0, 1e4])
    rec["vdenoiser_query"], rec["vdenoiser_t"] = vq, ext.VDenoiser(None).sigma_to_t(vq)
    rec["vdenoiser_t_to_sigma"] = ext.VDenoiser(None).t_to_sigma(torch.tensor([0.0, 0.1, 0.5, 0.9, 0.999]))

    # ------------------------------------------------------------------ forwards and gradients
    g = torch.Generator().manual_seed(3)
    x4 = torch.randn(3, 4, 8, 8, generator=g) * 3
    x3 = torch.randn(3, 3, 8, 8, generator=g) * 3
    cond = torch.randn(3, 4, 8, 8, generator=g)
    loss_w = torch.randn(3, 4, 8, 8, generator=g)
    sig = torch.tensor([14.6, 1.3, 0.05])
    rec.update(x4=x4, x3=x3, cond=cond, loss_w=loss_w, sigma=sig)
    wrappers = {
        "compvis_q0": (ext.CompVisDenoiser(E.ToyCompVis(4), quantize=False), x4, dict(cond=cond)),
        "compvis_q1": (ext.CompVisDenoiser(E.ToyCompVis(4), quantize=True), x4, dict(cond=cond)),
        "compvis_fp16": (ext.CompVisDenoiser(E.ToyCompVis(4, out_dtype=torch.float16)), x4, dict(cond=cond)),
        "compvis_v": (ext.CompVisVDenoiser(E.ToyCompVis(4)), x4, dict(cond=cond, ignored=1)),
        "eps_ddpm": (ext.DiscreteEpsDDPMDenoiser(E.ToyModel(4), ac, quantize=True), x4, {}),
        "v_ddpm": (ext.DiscreteVDDPMDenoiser(E.ToyModel(4), ac, quantize=False), x4, {}),
        "openai": (ext.OpenAIDenoiser(E.ToyModel(3, learned_sigmas=True), E.ToyDiffusion()), x3, {}),
        "openai_nols": (ext.OpenAIDenoiser(E.ToyModel(3), E.ToyDiffusion(), quantize=True, has_learned_sigmas=False), x3, {}),
        "vdenoiser": (ext.VDenoiser(E.ToyModel(4, t_scale=1.0)), x4, {}),
    }
    for name, (w, x, kw) in wrappers.items():
        rec[f"{name}_out"] = w(x, sig, **kw).detach()
        xg = x.clone().requires_grad_()
        rec[f"{name}_grad_x"] = torch.autograd.grad((w(xg, sig, **kw) * loss_w[:, :x.shape[1]]).sum(), xg)[0]

    # ------------------------------------------------------------------ sampler trajectories
    for name, w in (("eps", ext.CompVisDenoiser(E.ToyCompVis(4), quantize=False)), ("v", ext.CompVisVDenoiser(E.ToyCompVis(4)))):
        sigmas = w.get_sigmas(8)
        x = torch.randn(2, 4, 8, 8, generator=g) * sigmas[0]
        c = torch.randn(2, 4, 8, 8, generator=g)
        noise = torch.randn(8, 2, 4, 8, 8, generator=g)
        rec[f"{name}_traj_x"], rec[f"{name}_traj_cond"], rec[f"{name}_traj_noise"], rec[f"{name}_traj_sigmas"] = x, c, noise, sigmas
        ea = dict(cond=c)
        for s in ("euler", "heun", "dpmpp_2m", "lms"):
            rec[f"{name}_traj_{s}"] = getattr(S, f"sample_{s}")(w, x, sigmas, extra_args=ea, disable=True)
        it = iter(noise)
        rec[f"{name}_traj_euler_ancestral"] = S.sample_euler_ancestral(w, x, sigmas, extra_args=ea, disable=True,
                                                                       noise_sampler=lambda a, b: next(it))

    np.savez(G.OUT / "external.npz", **{k: v.detach().numpy() for k, v in rec.items()})
    (G.OUT / "external_signatures.json").write_text(json.dumps(signatures(ext), indent=1))
    print("wrote", G.OUT / "external.npz", len(rec), "arrays and", G.OUT / "external_signatures.json")


if __name__ == "__main__":
    main()
