"""Sampler checkpoints on the CPU.  rn_state.cuh's pack / unpack kernels run under RN_HOST_EMULATION against a numpy statement
of the SoA <-> chain-major transpose; rn_checkpoint_info, rn_checkpoint_slice and rn_sampler_restore's refusals run on
synthetic blobs built here from include/rainier_ckpt.h (the refusals that precede any device work need no GPU)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from oracle.rainier_py.cachedir import private_dir
from rainier_b200 import abi, api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIAG_FIELDS = 201  # rn_diag.cuh: RN_DIAG_FIELDS

_SHIM = r"""
// one launch, every CTA in turn (a call of the kernel runs a whole CTA under RN_HOST_EMULATION)
extern "C" void emu_state(int unpack, const RnStateArgs* a, unsigned gy) {
  rn_st_grid.x = (unsigned)((a->count + 31) / 32); rn_st_grid.y = gy; rn_st_grid.z = 1;
  for (unsigned bx = 0; bx < rn_st_grid.x; bx++)
    for (unsigned by = 0; by < gy; by++) {
      rn_st_block.x = bx; rn_st_block.y = by; rn_st_block.z = 0;
      if (unpack) rn_k_state_unpack(*a); else rn_k_state_pack(*a);
    }
}
"""


class StateField(C.Structure):
    _fields_ = [("ptr", C.c_uint64), ("elems", C.c_int64), ("words", C.c_int32), ("rec_word", C.c_int32)]


class StateArgs(C.Structure):
    _fields_ = [("f", StateField * 32), ("n_fields", C.c_int32), ("pad0", C.c_int32), ("rec_words", C.c_int64), ("C", C.c_int64),
                ("c0", C.c_int64), ("count", C.c_int64), ("staging", C.c_void_p)]


@pytest.fixture(scope="module")
def emu():
    src = open(os.path.join(ROOT, "rainier_b200", "csrc", "rn_state.cuh")).read() + _SHIM
    d = private_dir("rn_emul")
    so = os.path.join(d, "state_" + hashlib.sha1(src.encode()).hexdigest()[:16] + ".so")
    if not os.path.exists(so):
        cpp = so[:-3] + ".cpp"
        with open(cpp, "w") as f:
            f.write(src)
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-DRN_HOST_EMULATION", "-w", cpp, "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_state.argtypes = [C.c_int, C.c_void_p, C.c_uint]
    return L


def layout(n, W=5, buf=0, mass_max=1, track=False):
    """the record layout rn_runtime.cpp's ckpt_layout gives a sampler: [(field id, type, elements per chain)]"""
    F64, I64, I32 = abi.CKPT_F64, abi.CKPT_I64, abi.CKPT_I32
    dense, diag = mass_max == 2, mass_max >= 1
    L = [(abi.CKPT_PARAMS, F64, 2 * n + 1), (abi.CKPT_GRAD, F64, n), (abi.CKPT_RNG_SEED, I64, 1), (abi.CKPT_RNG_NNG, F64, 1),
         (abi.CKPT_DA, F64, 5), (abi.CKPT_MASS, F64, n * n if dense else (n if diag else 0)),
         (abi.CKPT_CHOL, F64, n * (n + 1) // 2 if dense else 0), (abi.CKPT_EST_MEAN, F64, n if diag else 0),
         (abi.CKPT_EST_RAW, F64, n if diag else 0), (abi.CKPT_EST_COV, F64, n * n if dense else 0), (abi.CKPT_RING, F64, buf),
         (abi.CKPT_ST_GRADS, I64, 1), (abi.CKPT_ST_STEPS, I64, 1), (abi.CKPT_ST_ENERGY, F64, 3), (abi.CKPT_ST_RINGS, F64, 3 * W),
         (abi.CKPT_TRACK, F64, DIAG_FIELDS * n if track else 0), (abi.CKPT_RNG_HAVE, I32, 1), (abi.CKPT_DA_ITER, I32, 1),
         (abi.CKPT_RING_I, I32, 1), (abi.CKPT_RING_FULL, I32, 1), (abi.CKPT_ST_ERR, I32, 1), (abi.CKPT_ST_ITERS, I32, 1),
         (abi.CKPT_ST_ACCEPTED, I32, 1), (abi.CKPT_ST_ENERGY_N, I32, 1), (abi.CKPT_ST_RING_I, I32, 3), (abi.CKPT_ST_RING_FULL, I32, 3)]
    return [f for f in L if f[2] > 0]


def record_bytes(L):
    b = sum(e * (4 if t == abi.CKPT_I32 else 8) for _, t, e in L)
    return (b + 7) // 8 * 8


def soa_state(L, chains, seed):
    """random bit patterns for every field, [elements][chains] (NaN payloads included: only bits are moved)"""
    rng = np.random.default_rng(seed)
    out = []
    for _, t, e in L:
        dt = np.uint32 if t == abi.CKPT_I32 else np.uint64
        out.append(rng.integers(0, np.iinfo(dt).max, size=(e, chains), dtype=dt, endpoint=True))
    return out


def records(L, soa, c0, count):
    """the chain-major records of chains [c0, c0 + count): [count][record_bytes] bytes"""
    parts = [np.ascontiguousarray(a[:, c0:c0 + count].T).view(np.uint8).reshape(count, -1) for a in soa]
    pad = record_bytes(L) - sum(p.shape[1] for p in parts)
    parts.append(np.zeros((count, pad), dtype=np.uint8))
    return np.concatenate(parts, axis=1)


def launch(emu, L, soa, chains, c0, count, staging, unpack, gy):
    a = StateArgs()
    off = 0
    for k, ((_, t, e), arr) in enumerate(zip(L, soa)):
        a.f[k] = StateField(arr.ctypes.data, e, 1 if t == abi.CKPT_I32 else 2, off // 4)
        off += e * arr.dtype.itemsize
    a.n_fields, a.rec_words, a.C, a.c0, a.count = len(L), record_bytes(L) // 4, chains, c0, count
    a.staging = staging.ctypes.data
    emu.emu_state(1 if unpack else 0, C.byref(a), gy)


CASES = {  # (n, stats window, EHMC ring, mass_max, tracked)
    "thread-identity-hmc": (10, 100, 0, 0, False),
    "thread-diagonal": (4, 5, 0, 1, False),
    "warp-diagonal": (7, 3, 0, 1, False),
    "dense": (5, 4, 0, 2, False),
    "ehmc": (3, 6, 10, 1, False),
    "tracked": (3, 2, 4, 1, True),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("chains", [1, 31, 33])
def test_pack_unpack_is_the_transpose(emu, case, chains):
    n, W, buf, mm, track = CASES[case]
    L = layout(n, W, buf, mm, track)
    soa = soa_state(L, chains, seed=chains)
    R = record_bytes(L)
    staging = np.zeros((chains, R), dtype=np.uint8)
    launch(emu, L, soa, chains, 0, chains, staging, False, 65535)
    assert np.array_equal(staging, records(L, soa, 0, chains))
    back = [np.zeros_like(a) for a in soa]
    launch(emu, L, back, chains, 0, chains, staging, True, 3)
    for a, b in zip(soa, back):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("case", ["thread-diagonal", "tracked"])
def test_chunks_that_cut_the_chain_range_mid_tile(emu, case):
    """save and restore in chunks whose boundaries fall inside 32-chain tiles, restored at a chain offset (concatenation)"""
    n, W, buf, mm, track = CASES[case]
    L = layout(n, W, buf, mm, track)
    chains = 16 * 1024 + 7 if case == "thread-diagonal" else 203
    soa = soa_state(L, chains, seed=5)
    R = record_bytes(L)
    blob = np.zeros((chains, R), dtype=np.uint8)
    c0 = 0
    for k, per in enumerate([45, 1, 1000, 33, 7000, 10**6]):
        cnt = min(per, chains - c0)
        if cnt <= 0:
            break
        stage = np.zeros((cnt, R), dtype=np.uint8)
        launch(emu, L, soa, chains, c0, cnt, stage, False, 1 + k % 3)
        blob[c0:c0 + cnt] = stage
        c0 += cnt
    assert c0 == chains
    assert np.array_equal(blob, records(L, soa, 0, chains))
    total = chains + 50  # restored at chain offset 17 of a larger sampler
    back = [np.zeros((a.shape[0], total), dtype=a.dtype) for a in soa]
    c0 = 0
    for per in [77, 5000, 10**6]:
        cnt = min(per, chains - c0)
        if cnt <= 0:
            break
        stage = np.ascontiguousarray(blob[c0:c0 + cnt])
        launch(emu, L, back, total, 17 + c0, cnt, stage, True, 2)
        c0 += cnt
    for a, b in zip(soa, back):
        assert np.array_equal(b[:, 17:17 + chains], a)
        assert not b[:, :17].any() and not b[:, 17 + chains:].any()


# ---- synthetic blobs ----------------------------------------------------------------------------------------------------
_M, _BASIS, _PRIME = (1 << 64) - 1, 1469598103934665603, 1099511628211


def hash_words(b):
    """rn_runtime.cpp: hash_words"""
    h = [_BASIS, _BASIS ^ 1, _BASIS ^ 2, _BASIS ^ 3]
    words = len(b) // 8
    for i, w in enumerate(np.frombuffer(b[:words * 8], dtype="<u8").tolist()):
        h[i & 3] = ((h[i & 3] ^ w) * _PRIME) & _M
    r = ((_BASIS ^ int.from_bytes(b[words * 8:], "little")) * _PRIME) & _M
    for x in h:
        r = ((r ^ x) * _PRIME) & _M
    return ((r ^ len(b)) * _PRIME) & _M


def blob_hash(b):
    seg = 16 << 20
    hs = [hash_words(b[k * seg:(k + 1) * seg]) for k in range(max(1, -(-len(b) // seg)))]
    return hash_words(np.array(hs, dtype="<u8").tobytes())


def seal(body):
    return bytes(body) + blob_hash(bytes(body)).to_bytes(8, "little")


def make_blob(chains=10, n=4, mass_max=1, seed=0, **hdr):
    """a checkpoint as rn_sampler_save lays it out: DefaultConfig fields, HMC on the thread shape, sampling phase"""
    cfg = abi.Config()
    api.lib().rn_config_default(C.byref(cfg))
    h = abi.CkptHeader()
    C.memmove(C.addressof(h), abi.CKPT_MAGIC, 8)  # (a c_char array would stop at the magic's NUL)
    h.version, h.header_bytes = abi.CKPT_VERSION, C.sizeof(abi.CkptHeader)
    for f, _ in abi.CkptHeader._fields_:
        if hasattr(cfg, f) and f != "backend":
            setattr(h, f, getattr(cfg, f))
    h.sampler, h.n_steps, h.mass_max, h.ehmc = abi.RN_SAMPLER_HMC, 5, mass_max, 0
    h.n, h.chains, h.initialized, h.warm_done, h.stats_reset_for_sampling = n, chains, 1, cfg.warmup_iterations, 1
    for k, v in hdr.items():
        setattr(h, k, v)
    L = layout(n, h.stats_window, 0, mass_max, bool(h.track))
    h.n_fields, h.record_bytes = len(L), record_bytes(L)
    h.step_bytes, h.pool_bytes = 8, (2 * n + 1) * 8
    rng = np.random.default_rng(seed)
    body = bytes(h) + b"".join(bytes(abi.CkptField(*f)) for f in L) + rng.bytes(h.step_bytes + h.pool_bytes)
    return seal(body + rng.bytes(chains * h.record_bytes)), h


def test_info_reports_the_header():
    blob, h = make_blob(chains=12, n=4, chain_offset=3, track=1, track_thin=3, track_seen=10, track_kept=4, win_size=75)
    i = api.checkpoint_info(blob)
    assert (i["version"], i["n"], i["chains"], i["chain_offset"], i["phase"]) == (1, 4, 12, 3, 3)
    assert (i["track"], i["track_thin"], i["track_seen"], i["track_kept"], i["win_size"]) == (1, 3, 10, 4, 75)
    assert i["header_bytes"] == 312 and i["table_bytes"] == 16 * h.n_fields and i["replicated_bytes"] == 8 + 72
    assert i["record_bytes"] == h.record_bytes and i["records_bytes"] == 12 * h.record_bytes and i["total_bytes"] == len(blob)
    assert api.checkpoint_info(make_blob(initialized=0, warm_done=0, stats_reset_for_sampling=0)[0])["phase"] == 0
    assert api.checkpoint_info(make_blob(warm_done=17, stats_reset_for_sampling=0)[0])["phase"] == 1
    assert api.checkpoint_info(make_blob(stats_reset_for_sampling=0)[0])["phase"] == 2


def test_slice_is_the_byte_range_of_its_chains():
    blob, h = make_blob(chains=10, chain_offset=100)
    R, off = h.record_bytes, len(blob) - 8 - 10 * h.record_bytes
    s = api.checkpoint_slice(blob, 3, 7)
    i = api.checkpoint_info(s)
    assert (i["chains"], i["chain_offset"]) == (4, 103)
    assert s[off:off + 4 * R] == blob[off + 3 * R:off + 7 * R]
    assert s[312:off] == blob[312:off]  # field table and replicated buffers
    ss = api.checkpoint_slice(s, 1, 2)  # a slice of a slice
    assert api.checkpoint_info(ss)["chain_offset"] == 104 and ss[off:off + R] == blob[off + 4 * R:off + 5 * R]
    assert bytes(api.checkpoint_slice(blob, 0, 10)) == blob
    for b, e in [(-1, 3), (3, 3), (5, 11)]:
        with pytest.raises(api.RainierCudaError) as err:
            api.checkpoint_slice(blob, b, e)
        assert err.value.code == abi.RN_E_INVALID


def refused(fn, *words):
    with pytest.raises(api.RainierCudaError) as err:
        fn()
    assert err.value.code == abi.RN_E_INVALID, str(err.value)
    for w in words:
        assert w in str(err.value), str(err.value)


def test_truncated_corrupted_and_foreign_blobs_are_refused():
    blob, h = make_blob()
    refused(lambda: api.checkpoint_info(blob[:-1]), "truncated")
    refused(lambda: api.checkpoint_info(blob[:200]), "truncated")
    refused(lambda: api.checkpoint_info(blob + b"\0"), "after the checksum")
    for at in (20, 400, len(blob) - 30, len(blob) - 1):  # header, table, a record, the checksum itself
        bad = bytearray(blob)
        bad[at] ^= 0x10
        refused(lambda: api.checkpoint_info(bad), "checksum")
        refused(lambda: api.checkpoint_slice(bad, 0, 1), "checksum")
    v2 = bytearray(blob[:-8])
    v2[8] = 2  # version 2, sealed with a valid checksum
    refused(lambda: api.checkpoint_info(seal(v2)), "version 2")
    refused(lambda: api.checkpoint_info(b"x" * len(blob)), "magic")


def test_pooled_warmup_cannot_be_cut():
    mid, _ = make_blob(chains=8, adaptation=abi.RN_ADAPT_POOLED, warm_done=300, stats_reset_for_sampling=0)
    refused(lambda: api.checkpoint_slice(mid, 0, 4), "pooled warmup")
    assert api.checkpoint_info(api.checkpoint_slice(mid, 0, 8))["chains"] == 8  # the whole blob is no cut
    steps, _ = make_blob(chains=8, step_adaptation=abi.RN_ADAPT_POOLED, initialized=0, warm_done=0, stats_reset_for_sampling=0)
    refused(lambda: api.checkpoint_slice(steps, 2, 8), "pooled warmup")
    done, _ = make_blob(chains=8, adaptation=abi.RN_ADAPT_POOLED)  # warmup finished: chains are independent again
    assert api.checkpoint_info(api.checkpoint_slice(done, 0, 4))["chains"] == 4
    per_chain, _ = make_blob(chains=8, warm_done=300, stats_reset_for_sampling=0)
    assert api.checkpoint_info(api.checkpoint_slice(per_chain, 5, 8))["chains"] == 3


def test_dmma_slices_keep_the_chain_groups():
    blob, _ = make_blob(chains=40, backend=1, mma=1, mma_chains=16)
    refused(lambda: api.checkpoint_slice(blob, 8, 24), "DMMA")
    refused(lambda: api.checkpoint_slice(blob, 0, 20), "DMMA")
    assert api.checkpoint_info(api.checkpoint_slice(blob, 16, 40))["chains"] == 24  # whole groups + the original tail
    assert api.checkpoint_info(api.checkpoint_slice(blob, 0, 32))["chains"] == 32


@pytest.fixture(scope="module")
def model4():
    """a 4-parameter model without a device: restore's checks that come before any device work"""
    rir = open(os.path.join(ROOT, "rainier_b200", "models", "eight_schools.rir"), "rb").read()
    m = api.CudaModel(rir, [], device=-1)
    yield m
    m.close()


def config_for(h):
    cfg = api.make_config(iterations=50, warmupIterations=h.warmup_iterations, sampler=api.HMCSampler(h.n_steps),
                          stepSizeTuner=api.DualAvgTuner(h.delta), massMatrixTuner=api.DiagonalMassMatrixTuner(
                              h.initial_window_size, h.window_expansion, h.skip_first, h.skip_last))
    return cfg


def test_restore_refusals_that_need_no_device(model4):
    n = model4.nVars
    blob, h = make_blob(n=n, warm_done=300, stats_reset_for_sampling=0)
    cfg = config_for(h)

    def restore(blobs, config=cfg):
        return api.CudaSampler.restore(model4, config, blobs)

    refused(lambda: api.CudaSampler.restore(model4, cfg, make_blob(n=n + 1)[0]), "n differs")
    refused(lambda: restore(blob, api.make_config(
        iterations=50, warmupIterations=h.warmup_iterations, sampler=api.HMCSampler(h.n_steps), stepSizeTuner=api.DualAvgTuner(0.7),
        massMatrixTuner=api.DiagonalMassMatrixTuner(h.initial_window_size, h.window_expansion, h.skip_first, h.skip_last))),
        "rn_config.delta")
    refused(lambda: restore(blob, api.make_config(
        iterations=50, warmupIterations=h.warmup_iterations, sampler=api.HMCSampler(h.n_steps), stepSizeTuner=api.DualAvgTuner(h.delta),
        massMatrixTuner=api.DenseMassMatrixTuner(h.initial_window_size, h.window_expansion, h.skip_first, h.skip_last))),
        "rn_config.mass_tuner")
    refused(lambda: restore(blob, api.make_config(
        iterations=50, warmupIterations=h.warmup_iterations + 1, sampler=api.HMCSampler(h.n_steps), stepSizeTuner=api.DualAvgTuner(h.delta),
        massMatrixTuner=api.DiagonalMassMatrixTuner(h.initial_window_size, h.window_expansion, h.skip_first, h.skip_last))),
        "rn_config.warmup_iterations")
    refused(lambda: restore(blob, api.make_config(
        iterations=50, warmupIterations=h.warmup_iterations, sampler=api.HMCSampler(h.n_steps), stepSizeTuner=api.DualAvgTuner(h.delta),
        massMatrixTuner=api.DiagonalMassMatrixTuner(h.initial_window_size, h.window_expansion, h.skip_first, h.skip_last), statsWindow=50)),
        "rn_config.stats_window")
    bad = bytearray(blob)
    bad[-1] ^= 1
    refused(lambda: restore(bad), "checkpoint 0", "checksum")
    refused(lambda: restore([blob, blob[:-3]]), "checkpoint 1", "truncated")
    refused(lambda: restore([blob, make_blob(n=n, warm_done=300, stats_reset_for_sampling=0, win_i=7)[0]]), "checkpoint 1", "win_i")
    pooled, hp = make_blob(n=n, adaptation=abi.RN_ADAPT_POOLED, warm_done=300, stats_reset_for_sampling=0)
    refused(lambda: restore([pooled, pooled]), "pooled warmup")

    # what may differ gets past every check: the call fails only for want of a device
    done, hd = make_blob(n=n)
    for blobs, config in [(blob, cfg), ([blob, blob], cfg), (done, api.make_config(
            iterations=5000, warmupIterations=10, sampler=api.HMCSampler(hd.n_steps), stepSizeTuner=api.DualAvgTuner(hd.delta),
            massMatrixTuner=api.DiagonalMassMatrixTuner(hd.initial_window_size, hd.window_expansion, hd.skip_first, hd.skip_last)))]:
        with pytest.raises(api.RainierCudaError) as err:
            restore(blobs, config)
        assert err.value.code == abi.RN_E_CUDA, str(err.value)


def test_python_hash_mirror_matches_the_library():
    """the synthetic blobs above are sealed by the Python statement of the checksum; a slice made by the library verifies"""
    blob, _ = make_blob(chains=3)
    s = api.checkpoint_slice(blob, 1, 3)
    assert int.from_bytes(s[-8:], "little") == blob_hash(bytes(s[:-8]))


def test_rank_checkpoint_is_written_whole(tmp_path):
    """dist.save_rank_checkpoint without a process group: rank 0's file, written through a temporary name"""
    from rainier_b200 import dist as rdist

    class Saved:
        def save(self):
            return bytearray(b"blob")

    path = rdist.save_rank_checkpoint(Saved(), str(tmp_path))
    assert path == str(tmp_path / "rank0.ckpt") and open(path, "rb").read() == b"blob"
    assert sorted(os.listdir(tmp_path)) == ["rank0.ckpt"]
