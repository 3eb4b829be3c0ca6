"""Bit-identity A/B of two engine builds on the bench's three calls (fitDisp MLE, fitDisp MAP, fitBeta).

The small-p kernels take a separate variant for indicator designs (column 0 all 1.0, every other entry +0.0 or 1.0):
it forms no design products and shares the (a, a) sums with the (a, 0) sums, and must compute exactly what the
general variant computes.  This script runs the bench's three calls through each library on the same inputs, for
  condition        ~condition               (p = 2, the bench's design; indicator variant)
  batch_condition  ~batch + condition       (p = 4, three batches; indicator variant)
  covariate        ~condition + covariate   (p = 3, a continuous covariate; general variant)
and requires every output to be identical byte for byte (NaN in the same places with the same bits).

    python scripts/indicator_ab.py LIB_A LIB_B [--genes 3000] [--samples 100]

The libraries are loaded one per child process through B200NB_LIB.  An emulated build (tests/simt_emu/build_emu.py)
runs on the CPU; it is loaded only with B200NB_TEST_EMULATOR=1, which this script sets for libraries whose name says
`emu`.  The inputs come from bench.py's workload builder with the CPU oracle as the engine.
"""
from __future__ import annotations

import argparse
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def designs(w, seed):
    """The bench's workload with three designs: its own ~condition, ~batch + condition, ~condition + covariate."""
    x = np.asarray(w["x"])
    m = x.shape[0]
    rng = np.random.default_rng(seed)
    batch = np.arange(m) % 3
    x4 = np.column_stack([x[:, 0], batch == 1, batch == 2, x[:, 1]]).astype(np.float64)
    x3 = np.column_stack([x[:, 0], x[:, 1], rng.normal(0.0, 1.0, m)])
    out = {"condition": w}
    norm = w["counts"] / w["sf"][None, :]
    for name, xd in (("batch_condition", x4), ("covariate", x3)):
        q, r = np.linalg.qr(xd)
        v = dict(w)
        v["x"] = np.asfortranarray(xd)
        v["beta0"] = np.asfortranarray(np.linalg.solve(r, q.T @ np.log(norm + 0.1).T).T)
        v["lam"] = np.full(xd.shape[1], 1e-6) / np.log(2) ** 2
        out[name] = v
    return out


def child(inputs: str, output: str) -> None:
    import bench
    from deseq2_b200 import wrappers as W
    with open(inputs, "rb") as f:
        ws = pickle.load(f)
    res = {}
    for name, w in ws.items():
        for call, r in zip(("fit_disp_mle", "fit_disp_map", "fit_beta"), bench.three_calls_host(w, W)):
            for k, v in r.items():
                res[f"{name}.{call}.{k}"] = np.asarray(v, dtype=np.float64)
    with open(output, "wb") as f:
        pickle.dump(res, f)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs=2)
    ap.add_argument("--genes", type=int, default=3000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--seed", type=int, default=20260925)
    a = ap.parse_args()
    import bench
    from oracle import oracle as O
    w = bench.build_workload(a.genes, a.samples, a.seed, O)
    with tempfile.TemporaryDirectory() as tmp:
        inputs = os.path.join(tmp, "inputs.pkl")
        with open(inputs, "wb") as f:
            pickle.dump(designs(w, a.seed), f)
        results = []
        for i, lib in enumerate(a.libs):
            env = dict(os.environ, B200NB_LIB=os.path.abspath(lib))
            if "emu" in os.path.basename(lib):
                env["B200NB_TEST_EMULATOR"] = "1"
            out = os.path.join(tmp, f"out{i}.pkl")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", inputs, out], env=env, check=True)
            with open(out, "rb") as f:
                results.append(pickle.load(f))
    ra, rb = results
    assert ra.keys() == rb.keys(), "the two libraries returned different result sets"
    bad = [k for k in sorted(ra) if ra[k].shape != rb[k].shape or ra[k].tobytes() != rb[k].tobytes()]
    for k in sorted(ra):
        print(f"{k:48s} {'identical' if k not in bad else 'DIFFERENT'}  nan={int(np.isnan(ra[k]).sum())}")
    print(f"{len(ra) - len(bad)} of {len(ra)} outputs identical byte for byte "
          f"({len(w['counts'])} genes x {a.samples} samples, seed {a.seed})")
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 4 and sys.argv[1] == "--child":
        child(sys.argv[2], sys.argv[3])
    else:
        sys.exit(main())
