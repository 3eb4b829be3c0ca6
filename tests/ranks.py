"""The multi-rank harness of the gene-sharded tests: run_ranks runs one function on every rank of a torch.distributed
process group, one spawned process per rank, over gloo on the CPU or over NCCL with one GPU per rank.

With backend="gloo" every rank runs the emulated engine (the product's CUDA sources on the SIMT emulator, see
tests/test_emulated_kernels.py) with CPU tensors; with backend="nccl" rank r runs the real engine on cuda:r.  The ranks
meet through a file store in a temporary directory, so no port is taken.  A rank that raises, exits or runs past the
timeout fails the call at once with that rank's traceback; the other ranks, which may be blocked in a collective, are
terminated, and no rank process outlives the call."""
import ctypes as C
import multiprocessing as mp
import os
import queue
import sys
import tempfile
import time
import traceback

import torch

from helpers import DEV

DEVICE = {"gloo": "cpu", "nccl": "cuda"}          # where a test's single-process run goes, per backend


def nccl_world(most=2):
    """The NCCL world size of a `-m gpu` test: `most` ranks when that many GPUs are visible, else 2; skips below two
    GPUs (and on the emulated engine, which has none)."""
    import pytest
    n_gpu = torch.cuda.device_count() if DEV == "cuda" else 0
    if n_gpu < 2:
        pytest.skip("needs at least 2 GPUs")
    return most if n_gpu >= most else 2


def _numpy(v):
    if isinstance(v, torch.Tensor):
        return v.cpu().numpy()
    if isinstance(v, dict):
        return {k: _numpy(e) for k, e in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(_numpy(e) for e in v)
    return v


def _rank_main(rank, world, backend, init, emu_lib, q, fn, args):
    try:
        import torch.distributed as dist
        if backend == "gloo":
            os.environ.update(B200NB_LIB=emu_lib, B200NB_TEST_EMULATOR="1", OMP_NUM_THREADS="2")
            from deseq2_b200 import _lib, device as D
            _lib._SO, _lib._lib = emu_lib, None    # fn's module imported the package before B200NB_LIB was set
            D._stream = lambda: C.c_void_p(0)      # emulated engine: host pointers, no CUDA stream
            dev = torch.device("cpu")
            dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
        else:
            dev = torch.device("cuda", rank)
            torch.cuda.set_device(dev)
            dist.init_process_group("nccl", init_method=init, rank=rank, world_size=world, device_id=dev)
        out = _numpy(fn(rank, world, dev, *args))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, out, None))
    except BaseException:
        q.put((rank, None, traceback.format_exc()))


def _collect(procs, q, timeout):
    deadline = time.monotonic() + timeout
    got = {}
    while len(got) < len(procs):
        # ranks that exited before this get: whatever they sent is already in the queue
        gone = {r: p.exitcode for r, p in enumerate(procs) if r not in got and p.exitcode is not None}
        try:
            rank, out, err = q.get(timeout=0.5)
        except queue.Empty:
            if gone:
                r, code = min(gone.items())
                raise RuntimeError(f"rank {r} of {len(procs)} exited with code {code} before returning a result")
            if time.monotonic() > deadline:
                raise TimeoutError(f"ranks {sorted(set(range(len(procs))) - set(got))} returned nothing in {timeout} s")
            continue
        if err is not None:
            raise RuntimeError(f"rank {rank} of {len(procs)} failed:\n{err}")
        got[rank] = out
    return [got[r] for r in range(len(procs))]


def run_ranks(fn, *args, world=2, backend="gloo", timeout=900):
    """fn(rank, world, device, *args) on `world` ranks; returns the ranks' return values in rank order, tensors turned
    into numpy arrays.  fn must be a module-level function (the ranks are spawned and import it)."""
    assert backend in DEVICE, backend
    emu_lib = None
    if backend == "gloo":
        emu_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt_emu")
        if emu_dir not in sys.path:
            sys.path.insert(0, emu_dir)
        import build_emu
        emu_lib = build_emu.build()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        init = "file://" + os.path.join(tmp, "store")
        procs = [ctx.Process(target=_rank_main, args=(r, world, backend, init, emu_lib, q, fn, args))
                 for r in range(world)]
        try:
            for p in procs:
                p.start()
            return _collect(procs, q, timeout)
        finally:
            started = [p for p in procs if p.pid is not None]
            for p in started:
                if p.is_alive():
                    p.terminate()
            for p in started:
                p.join(10)
                if p.is_alive():
                    p.kill()
                    p.join()
            q.close()
