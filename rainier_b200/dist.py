"""
rainier_b200.dist -- multi-GPU plumbing: one process per GPU, chains sharded over ranks (SURVEY.md 8e).

Chains are the unit of parallelism (each Driver.sample call owns its sampler, tuners, LeapFrog and Stats:
rainier-sampler/.../sampler/Driver.scala:13-17), so the sampling path needs NO collective: rank r runs the contiguous
chain block `chain_block(total, r, world)` with the same per-chain seeds a single process would use, and results are
rank-local until gathered.  The only exchange step is optional and warmup-only: pooling mass-matrix window statistics
over all chains of all ranks (RN_ADAPT_POOLED) -- two sum all-reduces per window of the chains' Welford statistics: first
{chains, sum of the chains' window means} (n+1 doubles), then sum of M2_c + L (mean_c - pooled mean)^2 (n doubles).

torch.distributed is used purely as plumbing (NCCL on GPUs, gloo in the CPU tests).
"""
import numpy as np


def chain_block(total_chains, rank, world):
    """contiguous block [lo, hi) of chains owned by `rank`; blocks differ by at most one chain"""
    base, rem = divmod(int(total_chains), int(world))
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def seeds_for_rank(seeds, rank, world):
    """the slice of the job-wide seed vector this rank runs: chain c behaves like ScalaRNG(seeds[c]) on any layout"""
    seeds = np.asarray(seeds, dtype=np.int64)
    lo, hi = chain_block(len(seeds), rank, world)
    return seeds[lo:hi]


def pooled_variance(count, s1, s2):
    """variance per parameter from pooled sums: count draws, s1 = sum q, s2 = sum q^2 (population variance, like
    VarianceEstimator.variance = raw / samples, MassMatrixEstimator.scala:92-100).  Textbook form, kept for reference: the
    library itself combines Welford statistics (`combine_welford`), which does not cancel when |mean| >> sd."""
    mean = s1 / count
    return s2 / count - mean * mean


def combine_welford(n, mean, m2):
    """Host mirror of the library's pooled window reduction (rn_k_pool_reduce, two passes + two all-reduces): chains (or
    ranks) each hold n draws with mean `mean[k]` and M2 `m2[k]` (sum of squared deviations from their own mean); the pooled
    population variance is [sum_k m2[k] + n (mean[k] - mean)^2] / (K n) around the pooled mean (Chan et al.)."""
    mean, m2 = np.asarray(mean, dtype=np.float64), np.asarray(m2, dtype=np.float64)
    k = mean.shape[0]
    g = mean.sum(axis=0) / k
    return (m2 + n * (mean - g) ** 2).sum(axis=0) / (k * n)


def allreduce_window_stats(stats, group=None):
    """stats: this rank's pooled-window buffer [2n+1] = [chains, sum of the chains' means (0..n-1), sum of M2_c +
    L (mean_c - pooled mean)^2 (0..n-1)], or a slice of it -> summed over all ranks (in place)"""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(stats, op=dist.ReduceOp.SUM, group=group)
    return stats


def max_over_ranks(seconds, device=None, group=None):
    """multi-GPU timings are the MAX over ranks of device-side durations"""
    import torch
    import torch.distributed as dist
    t = torch.tensor([float(seconds)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


def gather_samples(local, total_chains, group=None):
    """all ranks' [chains_r][iters][n] blocks -> [total_chains][iters][n] on every rank (chain order preserved)"""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    pieces = [None] * world
    dist.all_gather_object(pieces, np.asarray(local), group=group)
    out = np.concatenate(pieces, axis=0)
    assert out.shape[0] == total_chains
    return out


def best_start(x, f, info=None, group=None):
    """multi-start MAP over ranks (rn_optimize, SURVEY.md 8f-4): every rank optimises its block of starts
    (`chain_block(total_starts, rank, world)`); the job's answer is the converged start with the smallest f = -density.
    x: [starts_r][n], f: [starts_r], info: [starts_r] exit codes (0 = converged) -> (x_best [n], f_best, owner_rank) on
    every rank.  One small all-gather of (f, x) per rank; ties and NaNs resolve to the lowest (rank, index), so the
    result does not depend on the rank layout."""
    import torch.distributed as dist
    x, f = np.asarray(x, dtype=np.float64), np.asarray(f, dtype=np.float64).copy()
    if info is not None:
        f[np.asarray(info) != 0] = np.inf
    f[np.isnan(f)] = np.inf
    k = int(np.argmin(f)) if len(f) else -1
    mine = (float(f[k]), x[k].copy()) if k >= 0 else (np.inf, None)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return mine[1], mine[0], 0
    world = dist.get_world_size(group)
    pieces = [None] * world
    dist.all_gather_object(pieces, mine, group=group)
    owner = min(range(world), key=lambda r: (pieces[r][0], r))
    return pieces[owner][1], pieces[owner][0], owner
