"""
rainier_b200.dist -- multi-GPU plumbing: one process per GPU, chains sharded over ranks (SURVEY.md 8e).

Chains are the unit of parallelism (each Driver.sample call owns its sampler, tuners, LeapFrog and Stats:
rainier-sampler/.../sampler/Driver.scala:13-17), so the sampling path needs NO collective: rank r runs the contiguous
chain block `chain_block(total, r, world)` with the same per-chain seeds a single process would use, and results are
rank-local until gathered.  The only exchange step is optional and warmup-only: pooling mass-matrix window statistics
over all chains of all ranks (RN_ADAPT_POOLED) -- two sum all-reduces per window of the chains' Welford statistics: first
{chains, sum of the chains' window means} (n+1 doubles), then sum of M2_c + L (mean_c - pooled mean)^2 (n doubles), or
with the dense tuner the n^2 sums of C2_c[j][k] + L d_c[j] d_c[k] (`combine_welford_dense`).  Tracked diagnostics
(rn_sampler_tracked_diagnostics) are the other collective, on demand: two all-reduces of the same shape
(`combine_diagnostics`).

torch.distributed is used purely as plumbing (NCCL on GPUs, gloo in the CPU tests).
"""
import os

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


def combine_welford_dense(n, mean, cov):
    """Host mirror of the pooled dense window reduction (rn_k_pool_reduce pass 0, rn_k_pool_reduce_dense): chains (or ranks)
    each hold n draws with mean `mean[k]` ([K][d]) and co-moment `cov[k]` ([K][d][d], the sum of products of deviations from
    their own mean); the pooled population covariance [d][d] is [sum_k cov[k] + n (mean[k] - g)(mean[k] - g)^T] / (K n)
    around the pooled mean g.  With a communicator the library all-reduces {K, sum of the means} (d + 1 doubles), then the
    d^2 sums, and factors the result once per window."""
    mean, cov = np.asarray(mean, dtype=np.float64), np.asarray(cov, dtype=np.float64)
    k = mean.shape[0]
    d = mean - mean.sum(axis=0) / k
    return (cov + n * d[:, :, None] * d[:, None, :]).sum(axis=0) / (k * n)


DIAG_LAGS = 99  # variogram lags the ESS loop of Trace.diagnostics can add (Trace.scala:106)


def diagnostics_pass0(kept, sums):
    """Host mirror of pass 0 of rn_sampler_tracked_diagnostics on one rank: kept draws T_r per chain and the chains' running
    sums [C_r][n] -> the vector that is all-reduced, [0 (not tracking), 0 (out of memory), C_r, T_r, T_r^2, sum_c mean_c]"""
    sums = np.asarray(sums, dtype=np.float64)
    return np.concatenate([[0.0, 0.0, sums.shape[0], kept, float(kept) * float(kept)], (sums / kept).sum(axis=0)])


def equal_kept_counts(world, pass0_total):
    """the all-reduced verdict that every rank kept the same number of draws: R * sum T_r^2 == (sum T_r)^2, exact in fp64"""
    return world * pass0_total[4] == pass0_total[3] * pass0_total[3]


def diagnostics_pass1(kept, sums, m2, vg, pass0_total):
    """pass 1 on one rank around the pooled mean of pass 0: [sum_c (mean_c - meanMean)^2, sum_c M2_c / (T - 1),
    sum_c vg_c(lag) / (T - lag) for lag = 1..L], L = min(99, T - 1); vg: [C_r][99][n] variogram sums"""
    sums, m2, vg = (np.asarray(a, dtype=np.float64) for a in (sums, m2, vg))
    L = min(DIAG_LAGS, kept - 1)
    mm = pass0_total[5:] / pass0_total[2]
    lags = np.arange(1, L + 1, dtype=np.float64)[None, :, None]
    return np.concatenate([((sums / kept - mm) ** 2).sum(axis=0), (m2 / (kept - 1)).sum(axis=0),
                           (vg[:, :L, :] / (kept - lags)).sum(axis=0).reshape(-1)])


def diagnostics_epilogue(chains, kept, dev2, var_sum, vg_sum):
    """Trace.scala:60,75-109 for one parameter (rn_runtime.cpp: diag_epilogue): vg_sum[lag - 1] for lag = 1..L"""
    m, nn, L = float(chains), float(kept), len(vg_sum)
    b = (nn / (m - 1)) * dev2
    w = var_sum / m
    v = (nn - 1) / nn * w + b / nn
    acc, lag = 0.0, 1
    while True:
        vt = vg_sum[lag - 1] / m if lag <= L else (np.nan if lag == kept else -0.0)
        pt = 1.0 - (vt / (2.0 * v))
        if not (pt > 0.0 and lag < 100):
            break
        acc, lag = acc + pt, lag + 1
    return np.sqrt(v / w), nn * m / (1 + (2 * acc))


def diagnostics_finish(kept, pass0_total, pass1_total):
    """[n][2] = (rHat, effectiveSampleSize) from the two all-reduced vectors"""
    n = len(pass0_total) - 5
    p1 = np.asarray(pass1_total).reshape(-1, n)
    return np.array([diagnostics_epilogue(pass0_total[2], kept, p1[0, i], p1[1, i], p1[2:, i]) for i in range(n)])


def combine_diagnostics(blocks):
    """Host mirror of rn_sampler_tracked_diagnostics over ranks: blocks[r] = (T_r, sums [C_r][n], M2 [C_r][n], variogram
    sums [C_r][99][n]) of rank r's chains; the two all-reduces are sums in rank order.  Raises ValueError where the library
    returns RN_E_INVALID."""
    p0 = sum(diagnostics_pass0(b[0], b[1]) for b in blocks)
    if p0[2] < 2:
        raise ValueError("requirement failed: diagnostics requires multiple chains (Trace.scala:12)")
    if not equal_kept_counts(len(blocks), p0):
        raise ValueError("the ranks kept different numbers of draws")
    kept = blocks[0][0]
    if kept < 2:
        raise ValueError("at least 2 kept draws")
    p1 = sum(diagnostics_pass1(b[0], b[1], b[2], b[3], p0) for b in blocks)
    return diagnostics_finish(kept, p0, p1)


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


def save_rank_checkpoint(sampler, directory, group=None):
    """rn_sampler_save on every rank: rank r writes its sampler's checkpoint to <directory>/rank<r>.ckpt (written to a temporary
    name, then renamed, so a lost process leaves the previous file whole) and the ranks meet at a barrier.  The files of all
    ranks, restored in rank order with CudaSampler.restore(model, config, [blobs]), are the job's chains in their global order;
    a resumed job may use fewer or more GPUs (checkpoint_slice re-cuts the chains) once warmup has finished, or at any phase
    with per-chain adaptation.  Returns the path."""
    import torch.distributed as dist
    rank = dist.get_rank(group) if dist.is_available() and dist.is_initialized() else 0
    path = os.path.join(directory, "rank%d.ckpt" % rank)
    with open(path + ".tmp", "wb") as f:
        f.write(sampler.save())
        f.flush()
        os.fsync(f.fileno())
    os.replace(path + ".tmp", path)
    if dist.is_available() and dist.is_initialized():
        dist.barrier(group)
    return path
