"""python scripts/bench_pooled_trajectory.py  |  torchrun --nproc-per-node N scripts/bench_pooled_trajectory.py

Pooled EHMC trajectory lengths (rn_config.trajectory_adaptation = RN_ADAPT_POOLED) against per-chain lengths, alternated in one
call.  The two modes are different samplers, so besides the sampling rate the line reports the minimum effective sample size
per second of sampling (tracked diagnostics over every chain of every rank).
  cfg 4: eight schools, DefaultConfig, 8192 chains sharded over the ranks, thread-per-chain shape, 500 warmup + 500 sampling
         iterations: warmup ms, sampling ms and rate, min ESS/s, and the COUNTED lockstep factor of the per-chain run,
         sum over warps and iterations of the warp's longest trajectory / sum of all trajectories (from the per-chain trace of
         rank 0; a pooled run's factor is 1 by construction).
  logreg: streamed logistic regression (--rows x --cols), 2048 chains, short warmup: per-chain EHMC on the per-warp path
         against pooled EHMC on the DMMA path.
Device-timed (CUDA events on the sampler's stream), max over ranks.  One JSON line, with the card, its power limit and clock."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from oracle.rainier_py import configs  # noqa: E402
from rainier_b200 import abi, api  # noqa: E402


def card(device):
    q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(device)


def lockstep_factor(steps, warp=32):
    """steps [chains][iterations]: sum over warps of 32 consecutive chains and iterations of the longest trajectory, over the
    sum of all trajectories (1.0: no lane idles)"""
    c = (steps.shape[0] // warp) * warp
    w = steps[:c].reshape(-1, warp, steps.shape[1])
    return float(w.max(axis=1).sum() * warp) / float(w.sum())


def timed(model, config, seeds, dev, comm, world):
    s = api.CudaSampler(model, config, seeds=seeds)
    if comm is not None:
        s.set_comm(comm)
    stream = torch.cuda.ExternalStream(s.stream, device=dev)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record(stream)
    s.warmup(-1)
    ev[1].record(stream)
    s.track_diagnostics(1)
    s.run(config.iterations)
    ev[2].record(stream)
    s.sync()
    torch.cuda.synchronize()
    st, _ = s.stats()
    diag = np.asarray(s.tracked_diagnostics())  # [n][2] rHat, ESS over all chains of all ranks
    s.close()
    t = torch.tensor([ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])], dtype=torch.float64, device=dev)
    n = torch.tensor([float(sum(x.leapfrogSteps for x in st))], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(n, op=dist.ReduceOp.SUM)
    ms = float(t[1])
    return {"warmup_ms": float(t[0]), "sampling_ms": ms, "sampling_steps_x_chains_per_s": float(n[0]) / (ms * 1e-3),
            "min_ess": float(diag[:, 1].min()), "min_ess_per_sampling_s": float(diag[:, 1].min()) / (ms * 1e-3),
            "max_rhat": float(diag[:, 0].max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--rows", type=int, default=20000)
    ap.add_argument("--cols", type=int, default=50)
    ap.add_argument("--skip-logreg", action="store_true")
    args = ap.parse_args()
    rank, local, world = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    comm = api.Comm.from_torch_distributed(local) if world > 1 else None
    out = {}

    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    model = api.CudaModel(rir, [], device=local)
    total = 8192
    per = total // world
    seeds = np.arange(total, dtype=np.int64)[rank * per:(rank + 1) * per] + 1
    modes = {"per_chain": abi.RN_ADAPT_PER_CHAIN, "pooled": abi.RN_ADAPT_POOLED}
    mk = lambda mode, it=500: api.SamplerConfig(iterations=it, warmupIterations=500, backend=abi.RN_BACKEND_THREAD,  # noqa: E731
                                                trajectoryAdaptation=modes[mode])
    for mode in modes:  # compile both modules outside the timed runs
        timed(model, mk(mode, 2), seeds, dev, comm, world)
    runs = {m: [] for m in modes}
    for rep in range(args.reps):  # alternated
        for mode in modes:
            runs[mode].append(timed(model, mk(mode), seeds, dev, comm, world))
    cfg4 = {m: {k: float(np.median([r[k] for r in rs])) for k in rs[0]} for m, rs in runs.items()}
    # the counted lockstep factor of per-chain lengths (rank 0's chains, warps of 32 consecutive chains)
    s = api.CudaSampler(model, mk("per_chain"), seeds=seeds, trace=True)
    s.warmup(-1)
    s.run(500)
    tr = s.read_trace()
    s.close()
    cfg4["per_chain"]["lockstep_factor_counted"] = lockstep_factor(tr[:, 500:, 3])
    cfg4["pooled"]["lockstep_factor_counted"] = 1.0
    out["cfg4"] = dict(cfg4, config="eight schools, DefaultConfig, 500 warmup + 500 sampling, thread per chain", chains_total=total,
                       reps=args.reps, statistic="median over reps")
    model.close()

    if not args.skip_logreg:
        prir, pcols = configs.logreg(args.rows, args.cols).compile(False)
        lm = api.CudaModel(prir, pcols, device=local)
        lchains = 2048 // world
        lseeds = np.arange(2048, dtype=np.int64)[rank * lchains:(rank + 1) * lchains] + 7
        lmk = lambda mode, it=100: api.SamplerConfig(iterations=it, warmupIterations=100, backend=abi.RN_BACKEND_WARP,  # noqa: E731
                                                     trajectoryAdaptation=modes[mode])
        for mode in modes:
            timed(lm, lmk(mode, 2), lseeds, dev, comm, world)
        lr = {m: [] for m in modes}
        for rep in range(args.reps):
            for mode in modes:
                lr[mode].append(timed(lm, lmk(mode), lseeds, dev, comm, world))
        out["logreg"] = {m: {k: float(np.median([r[k] for r in rs])) for k in rs[0]} for m, rs in lr.items()}
        out["logreg"]["config"] = "logistic regression %d x %d, DefaultConfig, 100 warmup + 100 sampling, warp per chain" % (args.rows,
                                                                                                                           args.cols)
        out["logreg"]["path"] = "per_chain: per-warp rows-across-lanes; pooled: chain-batched DMMA in sampling"
        lm.close()
    if comm is not None:
        comm.close()
    if rank == 0:
        print(json.dumps(dict(out, n_gpus=world, gpu=card(local))), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
