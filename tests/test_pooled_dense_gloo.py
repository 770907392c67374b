"""dist.combine_welford_dense at world size 2 over gloo: each rank holds a block of chains (dist.chain_block), the two
all-reduces of the pooled dense window (chains and the sum of the means, then the n^2 sums around the pooled mean) run through
dist.allreduce_window_stats, and the result equals the single-process pooled estimate."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rainier_b200 import dist as rdist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHAINS, N, L = 301, 4, 9


def _stats():
    """small integer statistics with an integer pooled mean: every sum is exact in any order"""
    rng = np.random.default_rng(12)
    mean = rng.integers(-20, 20, size=(CHAINS, N)).astype(np.float64)
    mean[0] -= mean.sum(axis=0) - 3 * CHAINS
    cov = rng.integers(-100, 100, size=(CHAINS, N, N)).astype(np.float64)
    return mean, cov


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    import sys
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mean, cov = _stats()
    lo, hi = rdist.chain_block(CHAINS, rank, world)
    m, c = mean[lo:hi], cov[lo:hi]
    head = torch.tensor(np.concatenate([[hi - lo], m.sum(axis=0)]), dtype=torch.float64)
    rdist.allreduce_window_stats(head)
    g = head[1:].numpy() / head[0].item()
    d = m - g
    s = torch.tensor((c + L * d[:, :, None] * d[:, None, :]).sum(axis=0).reshape(-1), dtype=torch.float64)
    rdist.allreduce_window_stats(s)
    if rank == 0:
        np.save(os.path.join(out_dir, "pooled.npy"), s.numpy().reshape(N, N) / (head[0].item() * L))
    dist.destroy_process_group()


def test_combine_welford_dense_two_ranks_gloo(tmp_path):
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    got = np.load(os.path.join(str(tmp_path), "pooled.npy"))
    mean, cov = _stats()
    want = rdist.combine_welford_dense(L, mean, cov)
    assert np.array_equal(got, want)
