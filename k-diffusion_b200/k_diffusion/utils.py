"""Small helpers on the sampling path (reference: k_diffusion/utils.py:43-48,82-85,429-443)."""
from contextlib import contextmanager


def append_dims(x, target_dims):
    """Right-pad x's shape with singleton dims up to `target_dims` (utils.py:43-48)."""
    extra = target_dims - x.ndim
    if extra < 0:
        raise ValueError(f'input has {x.ndim} dims but target_dims is {target_dims}, which is less')
    return x.reshape(tuple(x.shape) + (1,) * extra)


def to_pil_image(x):
    """[-1, 1] tensor [C,H,W] / [1,C,H,W] -> PIL image (utils.py:27-34): clamp, map to [0, 255] as torchvision's to_pil_image does
    for float input (mul 255, truncate to uint8)."""
    import numpy as np
    from PIL import Image
    if x.ndim == 4:
        assert x.shape[0] == 1
        x = x[0]
    if x.shape[0] == 1:
        x = x[0]
    arr = ((x.detach().float().clamp(-1, 1) + 1) / 2).mul(255).byte().cpu().numpy()
    if arr.ndim == 3:
        arr = np.transpose(arr, (1, 2, 0))
    return Image.fromarray(arr)


def from_pil_image(x):
    """PIL image -> [-1, 1] tensor [C,H,W] (utils.py:19-24)."""
    import numpy as np
    import torch
    arr = np.asarray(x)
    t = torch.from_numpy(arr.copy())
    t = t[None] if t.ndim == 2 else t.permute(2, 0, 1)
    return t.float().div(255) * 2 - 1


def n_params(module):
    return sum(p.numel() for p in module.parameters())


@contextmanager
def _mode(model, training):
    was = [m.training for m in model.modules()]
    try:
        yield model.train(training)
    finally:
        for m, t in zip(model.modules(), was):
            m.training = t


def eval_mode(model):
    """Context manager: put `model` in eval mode, restore on exit (utils.py:82)."""
    return _mode(model, False)


def train_mode(model):
    return _mode(model, True)


@contextmanager
def tf32_mode(cudnn=None, matmul=None):
    """Context manager (and decorator) setting whether cuDNN convolutions and CUDA matmuls may use TF32 (utils.py:429-443).  A flag
    given as True or False is put back to its previous value on exit, also when the body raises; None leaves that flag alone."""
    import torch
    flags = [(torch.backends.cudnn, cudnn), (torch.backends.cuda.matmul, matmul)]
    saved = [owner.allow_tf32 for owner, _ in flags]
    try:
        for owner, value in flags:
            if value is not None:
                owner.allow_tf32 = value
        yield
    finally:
        for (owner, value), old in zip(flags, saved):
            if value is not None:
                owner.allow_tf32 = old
