"""CPU: the N>1 host path (view-pair sharding, max-over-ranks timing) with world_size=2 over gloo."""
import os
import sys

import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, ws, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(ws), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    from gps_gaussian_b200 import shard
    r, w = shard.init(backend="gloo")
    assert (r, w) == (rank, ws)
    units = shard.shard_units(7, r, w)
    seeds = shard.unit_seeds(1314, 8, r)
    shard.barrier()
    thr, total, ms = shard.aggregate_throughput(len(units), 100.0 * (r + 1))     # rank 1 is the slow one
    out.put((r, units, seeds, thr, total, ms))
    shard.finalize()


def test_shard_and_reduce_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, 29611, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    (r0, u0, s0, thr0, tot0, ms0), (r1, u1, s1, thr1, tot1, ms1) = res
    assert sorted(u0 + u1) == list(range(7)) and abs(len(u0) - len(u1)) <= 1     # every unit exactly once, balanced
    assert s0 == list(range(1314, 1322)) and s1 == list(range(1322, 1330))       # disjoint weak-scaling seeds
    assert tot0 == tot1 == 7 and ms0 == ms1 == 200.0                             # MAX over ranks
    assert abs(thr0 - 35.0) < 1e-9 and thr0 == thr1


def test_shard_units_properties():
    sys.path.insert(0, ROOT)
    from gps_gaussian_b200 import shard
    for n in (0, 1, 7, 64, 65):
        for w in (1, 2, 3, 8):
            parts = [shard.shard_units(n, r, w) for r in range(w)]
            assert sum(parts, []) == list(range(n))
            assert max(map(len, parts)) - min(map(len, parts)) <= 1


def _make_model():
    import torch
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.GroupNorm(2, 8), torch.nn.ReLU(),
                            torch.nn.Conv2d(8, 4, 3, padding=1))
    unused = torch.nn.Linear(4, 4)                      # like the reference's never-called gru16/gru32: grad stays None
    return m, unused


def _batch():
    import torch
    g = torch.Generator().manual_seed(1)
    return torch.randn(2, 3, 16, 16, generator=g), torch.randn(2, 4, 16, 16, generator=g)


def _ddp_worker(rank, ws, port, out):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(ws), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    import torch
    from gps_gaussian_b200 import shard
    shard.init(backend="gloo")
    m, unused = _make_model()
    x, y = _batch()
    # each rank sees ONE sample of the batch of two; loss is a per-sample mean, as in train_stage2.py:70-72
    loss = (m(x[rank:rank + 1]) - y[rank:rank + 1]).abs().mean()
    (loss * 1024.0).backward()                           # GradScaler-style scaled loss: averaging commutes with the scale
    params = list(m.parameters()) + list(unused.parameters())
    bucket = shard.allreduce_grads(params)
    gn = torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 1e9)
    # numpy arrays travel by value: a torch tensor on the queue is shared through a file descriptor, which is gone once
    # this process has exited
    out.put((rank, [(p.grad / 1024.0).numpy() for p in m.parameters()], float(gn) / 1024.0, int(bucket.numel()),
             all(p.grad is None for p in unused.parameters())))
    shard.finalize()


def test_allreduce_grads_world2_equals_single_process_batch2():
    """C5 (reference train_stage2.py:83-85 under data parallelism): the averaged per-rank gradients of a batch split over
    two ranks equal the single-process batch-2 gradients; the global grad norm is identical on every rank."""
    import torch
    sys.path.insert(0, ROOT)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, 29633, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted((q.get(timeout=180) for _ in range(2)), key=lambda t: t[0])
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    m, _ = _make_model()
    x, y = _batch()
    # single process, batch of two: mean over the two per-sample losses == what the two ranks average
    loss = 0.5 * ((m(x[0:1]) - y[0:1]).abs().mean() + (m(x[1:2]) - y[1:2]).abs().mean())
    loss.backward()
    want = [p.grad for p in m.parameters()]
    n_params = sum(p.numel() for p in m.parameters())
    for rank, grads, gn, nb, unused_none in res:
        assert nb == n_params and unused_none            # one flat bucket over exactly the parameters that have gradients
        for a, b in zip(grads, want):
            assert torch.allclose(torch.from_numpy(a), b, rtol=1e-5, atol=1e-7)
    assert abs(res[0][2] - res[1][2]) < 1e-9             # same global norm on both ranks => same clipping decision
