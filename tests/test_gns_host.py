"""k_diffusion.gns on the CPU: GradientNoiseScale against values recorded from the reference (tests/golden/gns.json, written by
oracle/make_golden_gns.py), and DDPGradientStatsHook on a world-size-2 gloo group around a plain torch module."""
import inspect
import json
import math
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

import k_diffusion as K

RECORDED = json.loads((GOLDEN / "gns.json").read_text())


def same(got, want):
    return (math.isnan(got) and math.isnan(want)) if isinstance(want, float) and math.isnan(want) else got == want


def same_state(got, want):
    return got.keys() == want.keys() and all(same(got[k], want[k]) for k in want)


def test_signatures_equal_the_references():
    for name, want in RECORDED["signatures"].items():
        cls, meth = name.split(".")
        fn = getattr(getattr(K.gns, cls), meth)
        got = [[n, p.kind.name, None if p.default is inspect._empty else repr(p.default)] for n, p in inspect.signature(fn).parameters.items()]
        assert got == want, name


@pytest.mark.parametrize("case", sorted(RECORDED["cases"]))
def test_gradient_noise_scale_matches_the_reference_bit_for_bit(case):
    rec = RECORDED["cases"][case]
    g = K.gns.GradientNoiseScale(**rec["kwargs"])
    assert same_state(g.state_dict(), rec["initial"])
    assert math.isnan(g.get_gns())
    for i, (small, large) in enumerate(rec["inputs"]):
        assert g.update(small, large, rec["n_small"], rec["n_large"]) == rec["returned"][i], (case, i)
        assert g.get_gns() == rec["gns"][i]
        assert list(g.get_stats()) == rec["stats"][i]
        assert same_state(g.state_dict(), rec["states"][i])
        if i == rec["reload_at"]:
            fresh = K.gns.GradientNoiseScale()
            fresh.load_state_dict(g.state_dict())
            g = fresh


def test_state_dict_is_a_copy():
    g = K.gns.GradientNoiseScale()
    state = g.state_dict()
    g.update(2.0, 1.0, 1, 4)
    assert state["beta_cumprod"] == 1.0 and g.state_dict()["beta_cumprod"] == 0.9998


def test_hook_refuses_a_module_without_ddp():
    with pytest.raises(ValueError):
        K.gns.DDPGradientStatsHook(torch.nn.Linear(3, 2))


def _net():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(12, 40), torch.nn.GELU(), torch.nn.Linear(40, 40), torch.nn.GELU(), torch.nn.Linear(40, 3))


def _batch(rank, step):
    g = torch.Generator().manual_seed(100 * step + rank)
    return torch.randn(5, 12, generator=g), torch.randn(5, 3, generator=g)


def _loss(net, x, y):
    return (net(x) - y).pow(2).mean()


def _worker(rank, world, port, q):
    sys.path.insert(0, str(ROOT / "k-diffusion_b200"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import k_diffusion as K
    local = _net()
    # a bucket cap below the model's size: from the second step on, several buckets per backward, each with its own pair of norms
    ddp = torch.nn.parallel.DistributedDataParallel(_net(), bucket_cap_mb=0.004)
    hook = K.gns.DDPGradientStatsHook(ddp)
    out = []
    for step in range(2):
        grads = []
        for r in range(world):   # every rank's local gradient, without DDP, on the same weights
            local.zero_grad()
            _loss(local, *_batch(r, step)).backward()
            grads.append(torch.cat([p.grad.flatten() for p in local.parameters()]))
        ddp.zero_grad()
        _loss(ddp, *_batch(rank, step)).backward()
        n_buckets = len(hook.bucket_sq_norms_small_batch)
        stats = hook.get_stats()
        mean = torch.cat([p.grad.flatten() for p in ddp.parameters()])
        out.append(dict(stats=stats, n_buckets=n_buckets, cleared=len(hook.bucket_sq_norms_large_batch),
                        want_small=sum(float(g.double().pow(2).sum()) for g in grads) / world,
                        want_large=float((sum(g.double() for g in grads) / world).pow(2).sum()),
                        mean_err=float((mean.double() - sum(g.double() for g in grads) / world).abs().max())))
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_ddp_hook_collects_local_and_averaged_squared_norms():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 1000) % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=240) for _ in procs)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for step in range(2):
        a, b = res[0][step], res[1][step]
        assert a["stats"] == b["stats"]                       # get_stats averages over the ranks
        assert a["n_buckets"] >= (2 if step else 1) and a["cleared"] == 0   # DDP rebuilds its buckets at the cap after the first step
        small, large = a["stats"]
        assert small == pytest.approx(a["want_small"], rel=1e-5)
        assert large == pytest.approx(a["want_large"], rel=1e-5)
        assert small > large > 0
        assert a["mean_err"] < 1e-6 and b["mean_err"] < 1e-6   # the hook hands DDP the averaged gradient
