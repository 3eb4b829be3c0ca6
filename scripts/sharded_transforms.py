"""Times the gene-sharded size factors and vst (deseq2_b200/sharded.py: sharded_size_factors_device, sharded_vst_device)
against the single-device functions (device_pipeline.size_factors, vst_device) and prints one JSON line.  Run on the
GPU:  python scripts/sharded_transforms.py [--worlds 1,2,8] [--shapes C2,C5] [--out DIR]
  * shapes C2 (50 000 x 100) and C5 (1 000 000 x 200); int32 counts drawn on the device from one seeded generator,
    so every rank builds the same matrix and keeps its rows (shard_bounds);
  * one process per GPU over NCCL for each world size that fits the visible GPUs (a world that does not fit is reported
    as skipped); each call is timed on every rank with a host clock ending in a device synchronise, after a barrier and
    one warm-up call, and the slowest rank counts; the median of --reps calls is reported;
  * the single-device functions are timed in the world-1 process, alternated with the sharded calls;
  * the collectives of each sharded call and their payload bytes, computed from the shapes here (sent per rank:
    all-reduce buffers, and each rank's part of an all-gather).
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SHAPES = {"C2": (50000, 100), "C5": (1000000, 200)}
NSUB = 1000


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # pragma: no cover
        return f"unknown ({e})"


def counts(n, m, dev, seed=5):
    """NB counts (gene means exp(N(3, 1.5)), dispersion 0.05 + 1 / mean, size factors exp(N(0, 0.3))) as a gene-major
    int32 device tensor, the same on every device for one seed."""
    from deseq2_b200 import device as D
    g = torch.Generator(device=dev).manual_seed(seed)
    mean = torch.exp(3.0 + 1.5 * torch.randn(n, 1, generator=g, device=dev, dtype=torch.float64))
    sf = torch.exp(0.3 * torch.randn(1, m, generator=g, device=dev, dtype=torch.float64))
    disp = 0.05 + 1.0 / mean
    out = torch.empty((n, m), dtype=torch.int32, device=dev)
    step = 100000
    for lo in range(0, n, step):
        mu = mean[lo:lo + step] * sf
        shape = (1.0 / disp[lo:lo + step]).expand_as(mu)
        lam = torch._standard_gamma(shape.contiguous(), generator=g) * mu * disp[lo:lo + step]
        out[lo:lo + step] = torch.poisson(lam, generator=g).clamp(max=2 ** 31 - 1).to(torch.int32)
    y = torch.zeros((n, D.ld_for(m)), dtype=torch.int32, device=dev)      # the gene-major layout of to_gene_major
    y[:, :m] = out
    return y


def sf_bytes(m, world):
    """(collectives, bytes sent per rank) of sharded_size_factors_device."""
    return 9, (m + 2) * 8 + 8 * (2 * m * 256 * 8)


def vst_bytes(m, world, cap, cap_sub):
    """sharded_vst_device with estimated size factors: the estimate, the 8-byte size agreement, the baseMean gather
    ((1 + 1) x cap doubles per rank, cap = the largest shard) and the GeneEst gather ((1 + 2) x cap_sub doubles per
    rank, cap_sub = the most subset rows on one rank)."""
    c, b = sf_bytes(m, world)
    return c + 3, b + 8 + 2 * cap * 8 + 3 * cap_sub * 8


def timed(f):
    dist.barrier()
    torch.cuda.synchronize()
    t = time.perf_counter()
    f()
    torch.cuda.synchronize()
    ms = torch.tensor([(time.perf_counter() - t) * 1e3], dtype=torch.float64, device="cuda")
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)                # the slowest rank
    return float(ms.item())


def rank_main(rank, world, init, shapes, reps, q):
    try:
        from deseq2_b200 import device_pipeline as DP, sharded
        dev = torch.device("cuda", rank)
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", init_method=init, rank=rank, world_size=world, device_id=dev)
        out = {}
        for name in shapes:
            n, m = SHAPES[name]
            lo, hi = sharded.shard_bounds(n, world, rank)
            y = counts(n, m, dev)[lo:hi].contiguous()
            torch.cuda.empty_cache()
            calls = {"sharded_size_factors_device": lambda: sharded.sharded_size_factors_device(y, m),
                     "sharded_vst_device": lambda: sharded.sharded_vst_device(y, m, nsub=NSUB)}
            if world == 1:
                calls.update({"size_factors": lambda: DP.size_factors(y, m),
                              "vst_device": lambda: DP.vst_device(y, m, nsub=NSUB)})
            got = {k: f() for k, f in calls.items()}                  # warm-up
            runs = {k: [] for k in calls}
            for _ in range(reps):
                for k, f in calls.items():
                    runs[k].append(timed(f))
            bounds = [sharded.shard_bounds(n, world, r) for r in range(world)]
            cap = max(b - a for a, b in bounds)
            owner = np.searchsorted([b for _, b in bounds], got["sharded_vst_device"]["subset"].cpu().numpy(),
                                    side="right")
            cap_sub = int(np.bincount(owner, minlength=world).max())
            r = {"n": n, "m": m, "ms": {k: float(np.median(v)) for k, v in runs.items()}, "ms_all": runs,
                 "collectives": {k: got[k]["collectives"] for k in ("sharded_size_factors_device", "sharded_vst_device")},
                 "bytes_sent_per_rank": {"sharded_size_factors_device": sf_bytes(m, world)[1],
                                         "sharded_vst_device": vst_bytes(m, world, cap, cap_sub)[1]}}
            assert r["collectives"]["sharded_size_factors_device"] == sf_bytes(m, world)[0]
            assert r["collectives"]["sharded_vst_device"] == vst_bytes(m, world, cap, cap_sub)[0]
            if world == 1:
                r["same_as_single_device"] = {
                    "sizeFactors": bool(torch.equal(got["sharded_size_factors_device"]["sizeFactors"],
                                                    got["size_factors"]["sizeFactors"])),
                    "vst": bool(torch.equal(got["sharded_vst_device"]["vst"], got["vst_device"]["vst"]))}
            del got, y
            torch.cuda.empty_cache()
            out[name] = r
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, out, None))
    except BaseException as e:                               # pragma: no cover
        import traceback
        q.put((rank, None, f"{e!r}\n{traceback.format_exc()}"))


def run_world(world, shapes, reps):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        init = "file://" + os.path.join(tmp, "store")
        procs = [ctx.Process(target=rank_main, args=(r, world, init, shapes, reps, q)) for r in range(world)]
        for p in procs:
            p.start()
        try:
            res = [q.get(timeout=3600) for _ in range(world)]
        finally:
            for p in procs:
                p.join(60)
                if p.is_alive():
                    p.terminate()
                    p.join()
    errs = [e for _, _, e in res if e]
    if errs:
        raise RuntimeError(errs[0])
    return next(o for r, o, _ in res if r == 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="1,2,8")
    ap.add_argument("--shapes", default="C2,C5")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    shapes = a.shapes.split(",")
    n_gpu = torch.cuda.device_count()
    res = {"card": card(), "gpus": n_gpu, "worlds": {}}
    for world in (int(w) for w in a.worlds.split(",")):
        if world > n_gpu:
            res["worlds"][world] = f"skipped: needs {world} GPUs, {n_gpu} visible"
            continue
        res["worlds"][world] = run_world(world, shapes, a.reps)
        print(world, json.dumps(res["worlds"][world]), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sharded_transforms.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
