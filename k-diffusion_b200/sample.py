#!/usr/bin/env python3
"""Draw images from a k-diffusion checkpoint on the H100-native engine.

Command line of the reference's sample.py (same flags, same `<prefix>_<index>.png` files), plus three optional ones:

    python sample.py --checkpoint model.safetensors [--config config.json] [-n 64] [--batch-size 64] [--steps 50] [--prefix out]
                     [--seed S] [--precision fp32|bf16] [--sampler sample_lms]
    python -m torch.distributed.run --nproc-per-node 8 sample.py --checkpoint ...        # one process per GPU, batch shards

What is different from the reference script (sample.py:37-66): there is no `accelerate` -- `k_diffusion.parallel.ProcessGroup`
supplies the few members of its interface used here; denoiser and sampler run on libkdb200 kernels; with `--seed` image i is a
function of (seed, i) only, so the set does not depend on the number of processes; `--precision bf16` selects the tensor-core path
(the default, fp32, is the arithmetic the reference script runs in).
"""
import argparse
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))

import torch

import k_diffusion as K


def cli(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    # the reference's flags
    ap.add_argument('--checkpoint', type=Path, required=True, help='safetensors file (the model config may be embedded in its metadata)')
    ap.add_argument('--config', type=Path, default=None, help='model config JSON; default: read it from the checkpoint')
    ap.add_argument('-n', type=int, default=64, help='how many images')
    ap.add_argument('--batch-size', type=int, default=64, help='images per sampler call and process')
    ap.add_argument('--steps', type=int, default=50, help='Karras schedule length')
    ap.add_argument('--prefix', type=str, default='out', help='files are written as <prefix>_<index>.png')
    # additions
    ap.add_argument('--seed', type=int, default=None, help='make image i depend on (seed, i) only')
    ap.add_argument('--precision', choices=['fp32', 'bf16'], default='fp32', help='arithmetic of the token stream')
    ap.add_argument('--sampler', default='sample_lms', help='name of a k_diffusion.sampling entry point')
    return ap.parse_args(argv)


def image_shape(model_cfg):
    h, w = model_cfg['input_size']
    if h != w:
        raise SystemExit(f'square inputs only (like the reference script), got {h}x{w}')
    return model_cfg['input_channels'], h, w


def load_denoiser(args, cfg, group):
    """checkpoint -> inner model on this process's GPU -> Karras preconditioner (sample.py:43-47)"""
    from safetensors.torch import load_file
    net = K.config.make_model(cfg).eval().requires_grad_(False)
    net.load_state_dict(load_file(str(args.checkpoint)))
    net = net.to(group.device).set_precision(args.precision)
    group.print('Parameters:', K.utils.n_params(net))
    return K.Denoiser(net, sigma_data=cfg['model']['sigma_data'])


def main(argv=None):
    args = cli(argv)
    cfg = K.config.load_config(args.config or args.checkpoint)
    mc = cfg['model']
    shape = image_shape(mc)
    sampler = getattr(K.sampling, args.sampler)

    group = K.parallel.ProcessGroup()
    print('Using device:', group.device, flush=True)
    denoiser = load_denoiser(args, cfg, group)
    sigmas = K.sampling.get_sigmas_karras(args.steps, mc['sigma_min'], mc['sigma_max'], rho=7., device=group.device)

    quiet = not group.is_local_main_process
    if not quiet:
        print('Sampling...', flush=True)
    try:
        with torch.no_grad(), K.utils.eval_mode(denoiser):
            images = K.evaluation.sample_images(group, denoiser, sigmas, args.n, args.batch_size, shape, mc['sigma_max'],
                                                sampler=sampler, seed=args.seed, disable=quiet)
    except KeyboardInterrupt:
        return
    if group.is_main_process:
        for index, image in enumerate(images):
            K.utils.to_pil_image(image).save(f'{args.prefix}_{index:05}.png')


if __name__ == '__main__':
    main()
