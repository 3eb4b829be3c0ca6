"""The gene-sharded drivers (deseq2_b200/sharded.py) equal the single-process run: the host mirror sharded_DESeq on two
gloo ranks with the oracle or the emulated engine (the reference proves the same for its BiocParallel chunking,
tests/testthat/test_parallel.R:12-37), and the device-resident sharded_DESeq_device on two gloo ranks with the emulated
engine or on 2-4 GPUs over NCCL.  The feature-specific sharded runs (weights, nf, betaPrior, LRT, results,
fitType = "mean") live with their features' tests; every one of them goes through tests/ranks.py, checked here too."""
import multiprocessing
import time

import numpy as np
import pytest

from helpers import emu_dev, gm  # noqa: F401
from ranks import DEVICE, nccl_world, run_ranks


def test_shard_bounds_cover_everything():
    from deseq2_b200.sharded import shard_bounds
    for n in (0, 1, 7, 100, 1001):
        for world in (1, 2, 3, 8):
            b = [shard_bounds(n, world, r) for r in range(world)]
            assert b[0][0] == 0 and b[-1][1] == n
            assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            sizes = [hi - lo for lo, hi in b]
            assert max(sizes) - min(sizes) <= 1


# ---------------------------------------------------------------- the harness

def _raise_on_rank_1(rank, world, dev):
    import torch.distributed as dist
    if rank == 1:
        raise ValueError("rank 1 refuses")
    dist.barrier()                                  # never completes: rank 1 is gone


def test_run_ranks_fails_fast_and_cleans_up():
    """A rank that raises fails run_ranks at once with its traceback, though the other rank waits in a collective;
    no rank process is left."""
    t0 = time.monotonic()
    with pytest.raises(RuntimeError, match="rank 1 of 2 failed(.|\n)*ValueError: rank 1 refuses"):
        run_ranks(_raise_on_rank_1)
    assert time.monotonic() - t0 < 60
    assert multiprocessing.active_children() == []


# ---------------------------------------------------------------- the host mirror

def _host_mirror_rank(rank, world, dev, engine):
    from deseq2_b200 import sharded, synth
    if engine == "oracle":
        from oracle import oracle as O
    else:
        from deseq2_b200 import wrappers as O           # the emulated engine: run_ranks bound it in every rank
    d = synth.make_example_counts(301, 8, seed=77)
    return sharded.sharded_DESeq(d["counts"], d["x"], d["sizeFactors"], engine=O)


def _check_host_mirror(engine, name):
    from deseq2_b200 import pipeline, synth
    got = run_ranks(_host_mirror_rank, name)
    d = synth.make_example_counts(301, 8, seed=77)
    whole = pipeline.DESeq(d["counts"], d["x"], sizeFactors=d["sizeFactors"], engine=engine)
    for g in got:
        for k in ("dispGeneEst", "dispFit", "dispMAP", "dispersion", "betaMatrix", "betaSE", "WaldStatistic",
                  "deviance"):
            assert np.allclose(g[k], whole[k], rtol=1e-12, atol=0, equal_nan=True), k
    return got, whole


def test_sharded_equals_whole(oracle):
    got, whole = _check_host_mirror(oracle, "oracle")
    assert all(abs(g["dispPriorVar"] - whole["dispPriorVar"]) < 1e-14 for g in got)


def test_sharded_equals_whole_with_the_emulated_engine(emu):
    """The same two-rank run with the PRODUCT engine (wrappers -> C ABI -> the CUDA kernels' source on the SIMT emulator)
    in every rank: what the multi-GPU deployment does, minus the GPUs.  Genes are independent, so the sharded result
    equals the single-process result of the same engine exactly."""
    _check_host_mirror(emu, "emulated")


# ---------------------------------------------------------------- the device-resident pipeline

def _data(n, m):
    from deseq2_b200 import synth
    x = synth.design_condition(m)
    d = synth.make_example_counts(n, m, x=x, seed=91)
    return d["counts"], x, d["sizeFactors"]


def _device_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    K, x, sf = _data(n, m)
    lo, hi = sharded.shard_bounds(n, world, rank)
    r = sharded.sharded_DESeq_device(gm(K[lo:hi], dev), x, sf)
    return {"trendCoefs": r["trendCoefs"], "dispPriorVar": r["dispPriorVar"], "gathered": r["gathered"],
            "collectives": r["collectives"], "n_local": r["idx"].numel()}


def _check_device(backend, n, m, world=2):
    """The global step (trend + prior variance on ALL genes through one all-gather) makes every per-gene result equal
    to the single-process run, bit for bit; two per-gene collectives (+ one 8-byte all-reduce)."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_device_rank, n, m, world=world, backend=backend)
    K, x, sf = _data(n, m)
    whole = DP.DESeq_device(gm(K, DEVICE[backend]), x, sf)
    for g in got:
        assert np.array_equal(g["trendCoefs"], whole["trendCoefs"].cpu().numpy())
        assert g["dispPriorVar"] == whole["dispPriorVar"]
        assert 0 < g["n_local"] < whole["idx"].numel()
        assert g["collectives"] - 1 == 2
        assert np.array_equal(g["gathered"]["dispersion"], whole["dispersion"].cpu().numpy())
        for k in ("betaMatrix", "WaldPvalue"):
            assert np.array_equal(g["gathered"][k], whole[k].cpu().numpy(), equal_nan=True), k


def test_sharded_device_pipeline_equals_whole(emu_dev):
    _check_device("gloo", 400, 12)


@pytest.mark.gpu
def test_sharded_device_pipeline_over_nccl_equals_whole(engine):
    _check_device("nccl", 20000, 40, world=nccl_world(4))
