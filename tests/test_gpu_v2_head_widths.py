"""image_transformer_v2 levels whose d_head is a multiple of 8 but not of 16 (AxialRoPE(d_head // 2) then rotates a width R = d_head / 2
that is not a multiple of 8): the fp32 forward, its JVP and its VJP against the oracle and torch.func of it, in float64."""
import pytest
import torch

import k_diffusion as K
from conftest import assert_close
from oracle import kdiff_oracle as O
from oracle.fixtures import synth_sd

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda"


def config(width, d_head):
    return K.config.load_config({
        "model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [16, 16], "patch_size": [2, 2], "widths": [width],
                  "depths": [2], "d_ffs": [2 * width], "self_attns": [{"type": "global", "d_head": d_head}], "mapping_width": 64,
                  "sigma_data": 1.0, "sigma_min": 1e-2, "sigma_max": 80.0},
        "dataset": {"num_classes": 0}})


@pytest.mark.parametrize("width, d_head", [(96, 24), (120, 40)])
def test_fp32_forward_jvp_vjp_match_the_oracle(width, d_head):
    cfg = config(width, d_head)
    model = K.config.make_model(cfg).eval().requires_grad_(False)
    sd = synth_sd({k: list(v.shape) for k, v in model.state_dict().items()}, 1)
    model.load_state_dict(sd)
    model = model.to(DEV).set_precision("fp32")
    mcfg = cfg["model"]
    sd64 = {k: v.double() for k, v in sd.items()}
    g = torch.Generator().manual_seed(d_head)
    x = torch.randn(2, 3, 16, 16, generator=g, dtype=torch.float64) * 2
    v = torch.randn(2, 3, 16, 16, generator=g, dtype=torch.float64)
    u = torch.randn(2, 3, 16, 16, generator=g, dtype=torch.float64)
    sig = torch.tensor([0.5, 4.0], dtype=torch.float64)
    f = lambda xi: O.model_forward(sd64, mcfg, xi, sig)
    want_f, want_t = torch.func.jvp(f, (x,), (v,))
    _, vjp_fn = torch.func.vjp(f, x)
    (want_g,) = vjp_fn(u)
    xd, sd_ = x.float().to(DEV), sig.float().to(DEV)
    assert_close(model(xd, sd_), want_f, what=f"d_head {d_head} forward")
    got_f, got_t = model.jvp(xd, sd_, v.float().to(DEV))
    assert_close(got_f, want_f, what=f"d_head {d_head} jvp primal")
    assert_close(got_t, want_t, what=f"d_head {d_head} jvp tangent")
    got_f2, got_g = model.vjp(xd, sd_, u.float().to(DEV))
    assert_close(got_f2, want_f, what=f"d_head {d_head} vjp primal")
    assert_close(got_g, want_g, what=f"d_head {d_head} vjp gradient")
