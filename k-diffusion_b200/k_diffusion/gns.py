"""The gradient noise scale of train.py --gns (reference: k_diffusion/gns.py): a DistributedDataParallel comm hook that records the
squared norm of each rank's gradient and of the averaged one, and the exponential moving averages that turn them into B_simple, the
critical batch size of McCandlish et al., "An Empirical Model of Large-Batch Training" (arXiv:1812.06162).

The hook's reductions run once per gradient bucket per step, off the hot path, on torch's own kernels.  A native model's backward writes
every gradient in one engine call, then DDP's reducer hands the buckets to this hook as it does for a torch model."""
import torch
import torch.distributed as dist


def _record_stats(hook, bucket):
    """Comm hook: the squared norm of this rank's bucket, then of the bucket averaged over the ranks; returns the averaged bucket, which
    DDP copies into the parameters' gradients as its default hook would."""
    local = bucket.buffer()
    hook.bucket_sq_norms_small_batch.append(local.pow(2).sum(dtype=torch.float32))

    def averaged(fut):
        mean = fut.value()[0]
        hook.bucket_sq_norms_large_batch.append(mean.pow(2).sum(dtype=torch.float32))
        return mean
    return dist.all_reduce(local, op=dist.ReduceOp.AVG, async_op=True).get_future().then(averaged)


class DDPGradientStatsHook:
    """Registers itself as the comm hook of `ddp_module` (a torch DistributedDataParallel model) and collects, over the buckets of each
    backward, the squared 2-norm of the local gradient and of the all-reduced mean gradient.  A module that is not DDP-wrapped raises
    ValueError."""

    def __init__(self, ddp_module):
        register = getattr(ddp_module, 'register_comm_hook', None)
        if register is None:
            raise ValueError('DDPGradientStatsHook does not support non-DDP wrapped modules')
        register(self, _record_stats)
        self._clear_state()

    def _clear_state(self):
        self.bucket_sq_norms_small_batch = []
        self.bucket_sq_norms_large_batch = []

    def get_stats(self):
        """(squared norm of the per-rank gradient, squared norm of the mean gradient) since the last call, each averaged over the ranks
        (a collective: every rank calls it).  Clears the collected norms."""
        stats = torch.stack([sum(self.bucket_sq_norms_small_batch), sum(self.bucket_sq_norms_large_batch)])
        self._clear_state()
        dist.all_reduce(stats, op=dist.ReduceOp.AVG)
        return stats[0].item(), stats[1].item()


class GradientNoiseScale:
    """Exponential moving averages of the unbiased estimates of |G|^2 and tr(Sigma) from two batch sizes, and their ratio, the gradient
    noise scale B_simple = tr(Sigma) / |G|^2.

    Args:
        beta (float): The decay factor of the moving averages. Default: 0.9998
        eps (float): The floor of both averages in the ratio, for numerical stability. Default: 1e-8
    """

    def __init__(self, beta=0.9998, eps=1e-8):
        self.beta = beta
        self.eps = eps
        self.ema_sq_norm = 0.
        self.ema_var = 0.
        self.beta_cumprod = 1.
        self.gradient_noise_scale = float('nan')

    def state_dict(self):
        """The object's state as a dict (every attribute)."""
        return dict(self.__dict__)

    def load_state_dict(self, state_dict):
        """Restore a state returned by `state_dict`."""
        self.__dict__.update(state_dict)

    def update(self, sq_norm_small_batch, sq_norm_large_batch, n_small_batch, n_large_batch):
        """Fold in one step's statistics and return the current gradient noise scale.

        Args:
            sq_norm_small_batch (float): The mean squared 2-norm of the gradients of the small (per-rank or per-sample) batches.
            sq_norm_large_batch (float): The squared 2-norm of the mean gradient over the large batch.
            n_small_batch (int): The size of a small batch (1 if per sample).
            n_large_batch (int): The size of the large batch.
        """
        # E|G_B|^2 = |G|^2 + tr(Sigma) / B at both sizes, solved for |G|^2 and tr(Sigma)
        est_sq_norm = (n_large_batch * sq_norm_large_batch - n_small_batch * sq_norm_small_batch) / (n_large_batch - n_small_batch)
        est_var = (sq_norm_small_batch - sq_norm_large_batch) / (1 / n_small_batch - 1 / n_large_batch)
        self.ema_sq_norm = self.beta * self.ema_sq_norm + (1 - self.beta) * est_sq_norm
        self.ema_var = self.beta * self.ema_var + (1 - self.beta) * est_var
        self.beta_cumprod *= self.beta
        self.gradient_noise_scale = max(self.ema_var, self.eps) / max(self.ema_sq_norm, self.eps)
        return self.gradient_noise_scale

    def get_gns(self):
        """The current gradient noise scale."""
        return self.gradient_noise_scale

    def get_stats(self):
        """The debiased moving averages (|G|^2, tr(Sigma))."""
        debias = 1 - self.beta_cumprod
        return self.ema_sq_norm / debias, self.ema_var / debias
