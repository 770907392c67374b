"""python scripts/bench_pooled_step.py  |  torchrun --nproc-per-node N scripts/bench_pooled_step.py

Cost of pooled step-size adaptation (rn_config.step_adaptation = RN_ADAPT_POOLED) on BASELINE.json's cfg 4: eight schools,
DefaultConfig (EHMC + DualAvg + diagonal mass windows), 8192 chains sharded over the ranks, 500 warmup + 500 sampling
iterations.  Three modes on the same chains: per_chain (reference semantics), pooled (mass windows pooled) and pooled_step
(one DualAvg step size over all chains, per-chain mass windows).  Device-timed (CUDA events on the sampler's stream), max over
ranks.  Prints one JSON line with warmup ms, the sampling rate, the all-reduce calls and their device time, and the card and
its power limit.  With one process no all-reduce runs; under torchrun the pooled modes all-reduce over NCCL (rn_comm)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from rainier_b200 import abi, api  # noqa: E402


def card(device):
    q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(device)


def main():
    rank, local, world = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    model = api.CudaModel(rir, [], device=local)
    total = 8192
    per = total // world
    seeds = np.arange(total, dtype=np.int64)[rank * per:(rank + 1) * per] + 1
    comm = api.Comm.from_torch_distributed(local) if world > 1 else None
    modes = {"per_chain": {}, "pooled": {"adaptation": abi.RN_ADAPT_POOLED}, "pooled_step": {"stepAdaptation": abi.RN_ADAPT_POOLED}}
    if comm is not None:  # NCCL sets its channels up inside the first collective: not a warmup's cost
        w = api.CudaSampler(model, api.SamplerConfig(iterations=1, warmupIterations=20, stepAdaptation=abi.RN_ADAPT_POOLED), seeds=seeds)
        w.set_comm(comm)
        w.warmup(-1)
        w.sync()
        w.close()
    res = {}
    for mode, ext in modes.items():
        for rep in range(2):  # the first run of a mode compiles its kernels (NVRTC) outside the timed window; time the second
            s = api.CudaSampler(model, api.SamplerConfig(iterations=500, warmupIterations=500, **ext), seeds=seeds)
            if mode != "per_chain" and comm is not None:
                s.set_comm(comm)
            stream = torch.cuda.ExternalStream(s.stream, device=dev)
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record(stream)
            s.warmup(-1)
            ev[1].record(stream)
            s.run(500)
            ev[2].record(stream)
            s.sync()
            torch.cuda.synchronize()
            st, mass = s.stats()
            calls, us = s.comm_stats()
            s.close()
        steps = float(sum(x.leapfrogSteps for x in st))
        t = torch.tensor([ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), us], dtype=torch.float64, device=dev)
        n = torch.tensor([steps], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            dist.all_reduce(n, op=dist.ReduceOp.SUM)
        res[mode] = {"warmup_ms": float(t[0]), "sampling_ms": float(t[1]),
                     "sampling_steps_x_chains_per_s": float(n[0]) / (float(t[1]) * 1e-3),
                     "allreduce_calls": int(calls), "allreduce_us_total": float(t[2]),
                     "step_size_chain0": st[0].stepSize, "step_size_identical_on_all_chains": all(x.stepSize == st[0].stepSize for x in st)}
    if comm is not None:
        comm.close()
    model.close()
    if rank == 0:
        print(json.dumps(dict(res, config="cfg 4: eight schools, DefaultConfig, 500 warmup + 500 sampling iterations",
                              chains_total=total, chains_per_gpu=per, n_gpus=world, gpu=card(local))), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
