"""Times the device transforms (vst_device, varianceStabilizingTransformation_device, normTransform_device and their
kernel b200nb_transform_dev) and prints one JSON line.  Run on the GPU:  python scripts/vst_pipeline.py [--out DIR]
  * the transform kernel alone (CUDA events around 200 launches after 10 warm-up launches) for each mode, int32
    counts and size factors, with its achieved bytes/s against the H100 SXM data-sheet 3.35 TB/s; the bytes are the
    algorithm's, computed from the shape: 4 B read + 8 B written per entry, plus the m size factors;
  * vst_device (nsub = 1000), varianceStabilizingTransformation_device(blind = True) and normTransform_device end to
    end (host clock ending in a device synchronise), alternated after one warm-up call of each;
  * DESeq_device on the same data in the same process, for scale;
at C2 (50 000 x 100, ~condition) and C4 (50 000 x 1000, 10-level factor).  The card name and power limit are read in
the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # pragma: no cover
        return f"unknown ({e})"


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from deseq2_b200 import _lib, device as D, device_pipeline as DP, synth
    dev = torch.device("cuda")
    res = {"card": card(), "shapes": {}}
    for name, n, m in (("C2", 50000, 100), ("C4", 50000, 1000)):
        x = synth.design_condition(m) if name == "C2" else synth.design_factor(m, 10)
        d = synth.make_example_counts(n, m, x=x, seed=4)
        y = D.to_gene_major(d["counts"].astype(np.int32), dev)
        sf = torch.as_tensor(d["sizeFactors"], device=dev)
        r = {"n": n, "m": m, "kernel": {}}
        nbytes = n * m * (4 + 8) + m * 8
        for mode, c0, c1 in (("parametric", 0.05, 2.0), ("mean", 0.07, 0.0), ("log2", 1.0, 0.0)):
            for _ in range(10):
                DP.transform(y, m, mode, c0, c1, sf)
            out = torch.empty((n, m), dtype=torch.float64, device=dev)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            L = _lib.lib()
            st = D._stream()
            mcode = DP._TRANSFORM_MODE[mode]
            e0.record()
            for _ in range(200):
                L.b200nb_transform_dev(D._p(y), 0, D._p(sf), None, n, m, y.shape[1], mcode, c0, c1, D._p(out), m,
                                       st)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 200
            r["kernel"][mode] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6,
                                 "share_of_3.35TB_per_s": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
        calls = {"vst_device": lambda: DP.vst_device(y, m),
                 "varianceStabilizingTransformation_device": lambda: DP.varianceStabilizingTransformation_device(y, m),
                 "normTransform_device": lambda: DP.normTransform_device(y, m),
                 "DESeq_device": lambda: DP.DESeq_device(y, x)}
        for f in calls.values():                                              # warm-up
            f()
        runs = {k: [] for k in calls}
        for _ in range(a.reps):
            for k, f in calls.items():
                runs[k].append(timed(f))
        r["end_to_end_ms"] = {k: float(np.median(v)) for k, v in runs.items()}
        r["end_to_end_ms_all"] = runs
        res["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vst_pipeline.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
