"""CPU oracle of the learned variance of an image_v1 U-Net with has_variance.  TEST INFRASTRUCTURE ONLY.

A functional restatement of

    k_diffusion/models/image_v1.py:150-156   (ImageDenoiserModelV1.forward with return_variance=True)
    k_diffusion/layers.py:93-101             (DenoiserWithVariance.loss)

on top of unet_oracle: its forward drops proj_out's variance channel, so logvar is formed here from the U-Net's output (proj_out's
input), which unet_oracle records as its last debug tap.  The taps are clones, so autograd reaches every parameter through them.
PINNED: tests/test_unet_variance_host.py checks it against the reference outputs that oracle/make_golden_unet_variance.py recorded.
"""
import torch.nn.functional as F

from . import unet_oracle as U
from .kdiff_oracle import karras_scalings


def _with_logvar(run, sd):
    taps = {}
    f = run(taps)
    y = list(taps.values())[-1]               # the last UBlock's output: proj_out's input
    logvar = F.conv2d(y, sd["proj_out.weight"][-1:], sd["proj_out.bias"][-1:]).flatten(1).mean(1)
    return f, logvar


def model_forward(sd, mcfg, x, sigma, mapping_cond=None):
    """image_v1.py:135-157 with return_variance=True: (output, logvar [B]), logvar the variance channel's mean over the token grid"""
    return _with_logvar(lambda taps: U.model_forward(sd, mcfg, x, sigma, mapping_cond, taps), sd)


def augment_forward(sd, mcfg, x, sigma, aug_cond=None, mapping_cond=None):
    """KarrasAugmentWrapper around model_forward (augmentation.py:97-104, return_variance passed through)"""
    return _with_logvar(lambda taps: U.augment_forward(sd, mcfg, x, sigma, aug_cond, mapping_cond, taps), sd)


def variance_loss(f, logvar, x, noise, sigma, sigma_data):
    """layers.py:93-101 (DenoiserWithVariance.loss) on the inner model's output f and logvar [B] for the noised input"""
    c_skip, c_out, _ = [c.view(-1, 1, 1, 1) for c in karras_scalings(sigma, sigma_data)]
    noised = x + noise * sigma.view(-1, 1, 1, 1)
    target = (x - c_skip * noised) / c_out
    lv = logvar.view(-1, 1, 1, 1)
    return (((f - target) ** 2 / lv.exp() + lv) / 2).flatten(1).mean(1)
