"""Times device_pipeline.size_factors with control genes and given geometric means against the plain call, and prints
one JSON line.  Run on the GPU:  python scripts/control_genes.py [--shapes C2,C5] [--reps 20] [--out DIR]
  * shapes C2 (50 000 x 100) and C5 (1 000 000 x 200); int32 NB counts drawn on the device from one seeded generator
    (scripts/sharded_transforms.py's counts);
  * calls: no control genes; 92 control rows (indices, as many as ERCC spike-ins); a 10 % row mask; given geoMeans
    (the plain call's own, so the answer is known); given geoMeans with the 92 control rows;
  * every call is timed with CUDA events on the current stream (each call ends in its one host read, the stop count),
    after one warm-up call of every kind; the calls are alternated and the median of --reps is reported;
  * with two or more visible GPUs, sharded_size_factors_device with the 10 % mask on 2 ranks over NCCL (host clock
    after a barrier, ending in a device synchronise; the slowest rank counts).
The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from sharded_transforms import SHAPES, card, counts  # noqa: E402


def calls(y, m, seed=3):
    from deseq2_b200 import device_pipeline as DP
    n = y.shape[0]
    g = torch.Generator(device=y.device).manual_seed(seed)
    idx = torch.randperm(n, generator=g, device=y.device)[:92]
    mask = torch.rand(n, generator=g, device=y.device, dtype=torch.float64) < 0.1
    geo = torch.exp(DP.size_factors(y, m)["loggeomeans"])
    return {"plain": lambda: DP.size_factors(y, m),
            "control_92": lambda: DP.size_factors(y, m, controlGenes=idx),
            "control_mask_10pct": lambda: DP.size_factors(y, m, controlGenes=mask),
            "geoMeans": lambda: DP.size_factors(y, m, geoMeans=geo),
            "geoMeans_control_92": lambda: DP.size_factors(y, m, controlGenes=idx, geoMeans=geo)}


def event_ms(f):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    f()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def single_device(shapes, reps):
    out = {}
    for name in shapes:
        n, m = SHAPES[name]
        y = counts(n, m, torch.device("cuda"))
        fs = calls(y, m)
        got = {k: f() for k, f in fs.items()}                       # warm-up
        plain = got["plain"]["sizeFactors"]
        want = plain / torch.exp(torch.log(plain).mean())
        runs = {k: [] for k in fs}
        for _ in range(reps):
            for k, f in fs.items():
                runs[k].append(event_ms(f))
        out[name] = {"n": n, "m": m, "ms": {k: float(np.median(v)) for k, v in runs.items()},
                     "ms_min": {k: float(np.min(v)) for k, v in runs.items()},
                     "geoMeans_round_trip_max_rel_err": float(((got["geoMeans"]["sizeFactors"] - want).abs()
                                                               / want).max().item())}
        del y, fs, got
        torch.cuda.empty_cache()
    return out


def rank_main(rank, world, init, shapes, reps, q):
    try:
        import torch.distributed as dist
        from deseq2_b200 import sharded
        dev = torch.device("cuda", rank)
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", init_method=init, rank=rank, world_size=world, device_id=dev)
        out = {}
        for name in shapes:
            n, m = SHAPES[name]
            lo, hi = sharded.shard_bounds(n, world, rank)
            y = counts(n, m, dev)[lo:hi].contiguous()
            g = torch.Generator(device=dev).manual_seed(3)
            mask = (torch.rand(n, generator=g, device=dev, dtype=torch.float64) < 0.1)[lo:hi]
            f = lambda: sharded.sharded_size_factors_device(y, m, controlGenes_local=mask)  # noqa: E731
            f()
            ms = []
            for _ in range(reps):
                dist.barrier()
                torch.cuda.synchronize()
                t = time.perf_counter()
                f()
                torch.cuda.synchronize()
                v = torch.tensor([(time.perf_counter() - t) * 1e3], dtype=torch.float64, device=dev)
                dist.all_reduce(v, op=dist.ReduceOp.MAX)
                ms.append(float(v.item()))
            out[name] = {"ms": float(np.median(ms)), "collectives": f()["collectives"]}
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, out, None))
    except BaseException as e:                               # pragma: no cover
        import traceback
        q.put((rank, None, f"{e!r}\n{traceback.format_exc()}"))


def sharded_two_ranks(shapes, reps):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        init = "file://" + os.path.join(tmp, "store")
        procs = [ctx.Process(target=rank_main, args=(r, 2, init, shapes, reps, q)) for r in range(2)]
        for p in procs:
            p.start()
        try:
            res = [q.get(timeout=1800) for _ in range(2)]
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
    ap.add_argument("--shapes", default="C2,C5")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    shapes = a.shapes.split(",")
    res = {"card": card(), "gpus": torch.cuda.device_count(), "single_device": single_device(shapes, a.reps)}
    res["sharded_mask_10pct_2_ranks"] = sharded_two_ranks(shapes, a.reps) if res["gpus"] >= 2 else \
        f"skipped: needs 2 GPUs, {res['gpus']} visible"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "control_genes.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
