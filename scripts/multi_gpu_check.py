"""torchrun --nproc-per-node N scripts/multi_gpu_check.py : chains sharded over ranks reproduce the single-GPU run bit
for bit (no collective on the sampling path), and RN_ADAPT_POOLED all-reduces window statistics over NCCL so that every
rank ends warmup with the same shared mass matrix; tracked diagnostics cover every chain of every rank, identically on all."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from rainier_b200 import abi, api
from rainier_b200 import dist as rdist

rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rir = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rainier_b200", "models", "eight_schools.rir"), "rb").read()
total = 1024
seeds = np.arange(total) + 7
model = api.CudaModel(rir, [], device=local)
cfg = api.SamplerConfig(iterations=50, warmupIterations=300)
mine = rdist.seeds_for_rank(seeds, rank, world)
tr = model.sample(cfg, seeds=mine)
full = rdist.gather_samples(tr.chains, total)
if rank == 0:
    ref = model.sample(cfg, seeds=seeds)
    assert np.array_equal(full, ref.chains), "sharded run differs from the single-GPU run"
    print("sharded == single-GPU: bit-identical samples for %d chains over %d ranks" % (total, world))
# pooled adaptation over NCCL
cfgp = api.SamplerConfig(iterations=20, warmupIterations=300, adaptation=abi.RN_ADAPT_POOLED)
comm = api.Comm.from_torch_distributed(local)
s = api.CudaSampler(model, cfgp, seeds=mine)
s.set_comm(comm)
s.warmup(-1)
s.run(20)
stats, mass = s.stats()
m = torch.tensor(mass[0], device="cuda")
gathered = [torch.empty_like(m) for _ in range(world)]
dist.all_gather(gathered, m)
assert all(torch.equal(g, gathered[0]) for g in gathered), "ranks disagree on the pooled mass matrix"
assert np.all(mass == mass[0])
if rank == 0:
    print("pooled adaptation: identical mass matrix on all %d ranks:" % world, np.round(mass[0], 4))
s.close()

# pooled step sizes over NCCL: exact int64 sums, so N ranks x C/N chains reproduce 1 rank x C chains bit for bit
cfgs = api.SamplerConfig(iterations=50, warmupIterations=300, stepAdaptation=abi.RN_ADAPT_POOLED)
s = api.CudaSampler(model, cfgs, seeds=mine)
s.set_comm(comm)
d = torch.empty((50, model.nVars, len(mine)), dtype=torch.float64, device="cuda")
s.warmup(-1)
s.run(50, d.data_ptr())
s.sync()
calls, _ = s.comm_stats()
full = rdist.gather_samples(d.permute(2, 0, 1).contiguous().cpu().numpy(), total)
s.close()
if rank == 0:
    assert world == 1 or calls == cfgs.warmupIterations + 1, calls
    ref = model.sample(cfgs, seeds=seeds)
    assert np.array_equal(full, ref.chains), "pooled steps: sharded run differs from the single-GPU run"
    print("pooled step sizes: %d ranks x %d chains == 1 rank x %d chains bit for bit; %d all-reduce calls"
          % (world, total // world, total, calls))

# tracked diagnostics over NCCL: Trace.diagnostics of every chain of every rank, the same numbers on every rank
from oracle.rainier_py.diagnostics import trace_diagnostics  # noqa: E402
cfgt = api.SamplerConfig(iterations=300, warmupIterations=300)
s = api.CudaSampler(model, cfgt, seeds=mine)
s.set_comm(comm)
d = torch.empty((300, model.nVars, len(mine)), dtype=torch.float64, device="cuda")
s.warmup(-1)
s.track_diagnostics(1)
s.run(120, d.data_ptr())
s.run(180, d[120:].data_ptr())
got = s.tracked_diagnostics()
s.close()
g = torch.tensor(got, device="cuda")
gathered = [torch.empty_like(g) for _ in range(world)]
dist.all_gather(gathered, g)
assert all(torch.equal(x, gathered[0]) for x in gathered), "ranks disagree on the tracked diagnostics"
full = rdist.gather_samples(d.permute(2, 0, 1).contiguous().cpu().numpy(), total)
if rank == 0:
    one = api.CudaSampler(model, cfgt, seeds=seeds)
    one.warmup(-1)
    one.track_diagnostics(1)
    one.run(300)
    single = one.tracked_diagnostics()
    one.close()
    rel = lambda a, b: float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-12)))
    assert rel(got, single) < 1e-12, (got, single)
    ref = np.array(trace_diagnostics(full))
    assert rel(got, ref) < 1e-9, (got, ref)
    print("tracked diagnostics: identical on all %d ranks; vs one process %.2g, vs the restatement %.2g"
          % (world, rel(got, single), rel(got, ref)))

# BASELINE.json configs[3]: eight schools, DefaultConfig (EHMC + DualAvg + diagonal mass), 8192 chains over the ranks,
# warmup with the pooled mass-matrix all-reduce (NCCL over NVLink); device-resident, timed on the device, max over ranks
import time
total = 8192
per = total // world
seeds_all = np.arange(total) + 1
cfgb = api.SamplerConfig(iterations=500, warmupIterations=500, adaptation=abi.RN_ADAPT_POOLED)
for mode, cfg_run in (("pooled", cfgb), ("per-chain", api.SamplerConfig(iterations=500, warmupIterations=500))):
    sb = api.CudaSampler(model, cfg_run, seeds=rdist.seeds_for_rank(seeds_all, rank, world))
    if mode == "pooled":
        sb.set_comm(comm)
    stream = torch.cuda.ExternalStream(sb.stream)
    d = torch.empty((500, model.nVars, per), dtype=torch.float64, device="cuda")
    dist.barrier()
    torch.cuda.synchronize()
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record(stream)
    sb.warmup(-1)
    e1.record(stream)
    sb.run(500, d.data_ptr())
    e2.record(stream)
    sb.sync()
    torch.cuda.synchronize()
    st, _ = sb.stats()
    steps = float(sum(x.leapfrogSteps for x in st))
    t = torch.tensor([e0.elapsed_time(e1), e1.elapsed_time(e2), steps], dtype=torch.float64, device="cuda")
    tmax = t.clone()
    dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    if rank == 0:
        print("cfg4 eight schools, %d chains over %d GPU(s), %s adaptation: warmup(500) %.1f ms, sampling(500) %.1f ms, "
              "sampling-phase leapfrog-steps*chains/s %.3e" % (total, world, mode, tmax[0].item(), tmax[1].item(),
                                                              t[2].item() / (tmax[1].item() * 1e-3)), flush=True)
    sb.close()
comm.close()
dist.destroy_process_group()
