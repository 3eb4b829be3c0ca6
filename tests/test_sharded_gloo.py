"""N > 1 path on CPU: world_size-2 gloo run of the gene-sharded driver (deseq2_b200/sharded.py) with the oracle
engine; sharded == unsharded (the reference proves the same for its BiocParallel chunking,
tests/testthat/test_parallel.R:12-37)."""
import os
import sys

import numpy as np
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q, emu_lib=None):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="2")
    if emu_lib:
        os.environ["B200NB_LIB"] = emu_lib          # the product engine's own source, executed by the SIMT emulator
    import torch.distributed as dist
    from deseq2_b200 import sharded, synth
    if emu_lib:
        from deseq2_b200 import wrappers as O
    else:
        from oracle import oracle as O
    dist.init_process_group("gloo", rank=rank, world_size=world)
    d = synth.make_example_counts(301, 8, seed=77)
    r = sharded.sharded_DESeq(d["counts"], d["x"], d["sizeFactors"], engine=O)
    if rank == 0:
        q.put({k: np.asarray(v) for k, v in r.items()})
    dist.barrier()
    dist.destroy_process_group()


def test_shard_bounds_cover_everything():
    from deseq2_b200.sharded import shard_bounds
    for n in (0, 1, 7, 100, 1001):
        for world in (1, 2, 3, 8):
            b = [shard_bounds(n, world, r) for r in range(world)]
            assert b[0][0] == 0 and b[-1][1] == n
            assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            sizes = [hi - lo for lo, hi in b]
            assert max(sizes) - min(sizes) <= 1


def test_sharded_equals_whole(oracle):
    from deseq2_b200 import pipeline, synth
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    d = synth.make_example_counts(301, 8, seed=77)
    whole = pipeline.DESeq(d["counts"], d["x"], sizeFactors=d["sizeFactors"], engine=oracle)
    for k in ("dispGeneEst", "dispFit", "dispMAP", "dispersion", "betaMatrix", "betaSE", "WaldStatistic", "deviance"):
        assert np.allclose(got[k], whole[k], rtol=1e-12, atol=0, equal_nan=True), k
    assert abs(got["dispPriorVar"] - whole["dispPriorVar"]) < 1e-14


def test_sharded_equals_whole_with_the_emulated_engine(emu):
    """The same two-rank run with the PRODUCT engine (wrappers -> C ABI -> the CUDA kernels' source on the SIMT emulator)
    in every rank: what the multi-GPU deployment does, minus the GPUs.  Genes are independent, so the sharded result
    equals the single-process result of the same engine exactly."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build_emu
    from deseq2_b200 import pipeline, synth
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, build_emu.build())) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    d = synth.make_example_counts(301, 8, seed=77)
    whole = pipeline.DESeq(d["counts"], d["x"], sizeFactors=d["sizeFactors"], engine=emu)
    for k in ("dispGeneEst", "dispFit", "dispMAP", "dispersion", "betaMatrix", "betaSE", "WaldStatistic", "deviance"):
        assert np.allclose(got[k], whole[k], rtol=1e-12, atol=0, equal_nan=True), k


def _device_worker(rank, world, port, q, emu_lib):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="2", B200NB_LIB=emu_lib,
                      B200NB_TEST_EMULATOR="1")
    import ctypes as C
    import torch
    import torch.distributed as dist
    from deseq2_b200 import device as D, sharded, synth
    D._stream = lambda: C.c_void_p(0)          # emulated engine: host pointers, no CUDA stream
    dist.init_process_group("gloo", rank=rank, world_size=world)
    m = 12
    x = synth.design_condition(m)
    d = synth.make_example_counts(400, m, x=x, seed=91)
    lo, hi = sharded.shard_bounds(400, world, rank)
    y = D.to_gene_major(d["counts"][lo:hi], torch.device("cpu"))
    r = sharded.sharded_DESeq_device(y, x, d["sizeFactors"])
    if rank == 0:
        q.put({"trend": r["trendCoefs"].numpy(), "priorVar": r["dispPriorVar"],
               "beta": r["gathered"]["betaMatrix"].numpy(), "disp": r["gathered"]["dispersion"].numpy(),
               "pval": r["gathered"]["WaldPvalue"].numpy(), "n_local": int(r["idx"].numel())})
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_device_pipeline_equals_whole(emu):
    """The device-resident pipeline gene-sharded over two ranks (gloo; emulated engine, CPU tensors): the global step
    (trend + prior variance on ALL genes through one all-gather) makes every per-gene result equal to the
    single-process run, bit for bit."""
    import ctypes as C
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build_emu
    from deseq2_b200 import device as D, device_pipeline as DP, synth
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_device_worker, args=(r, 2, port, q, build_emu.build())) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=600)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    saved = D._stream
    D._stream = lambda: C.c_void_p(0)
    try:
        m = 12
        x = synth.design_condition(m)
        d = synth.make_example_counts(400, m, x=x, seed=91)
        whole = DP.DESeq_device(D.to_gene_major(d["counts"], torch.device("cpu")), x, d["sizeFactors"])
    finally:
        D._stream = saved
    assert np.array_equal(got["trend"], whole["trendCoefs"].numpy()) and got["priorVar"] == whole["dispPriorVar"]
    assert 0 < got["n_local"] < whole["idx"].numel()
    assert np.array_equal(got["disp"], whole["dispersion"].numpy())
    assert np.array_equal(got["beta"], whole["betaMatrix"].numpy(), equal_nan=True)
    assert np.array_equal(got["pval"], whole["WaldPvalue"].numpy(), equal_nan=True)
