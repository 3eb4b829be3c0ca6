"""Config-4 shape (m = 1000, 10-level factor, p = 10): the general-p kernels of fit_generic.cu (B200NB_GENERIC_SEG=0)
against the segmented kernels of fit_generic_seg.cuh at 8 / 12 / 16 warps per SM (B200NB_GENERIC_WARPS), same inputs,
CUDA events, best of 3; plus the 11-column expanded design (not saturated: Cholesky path) and the results' agreement.
usage: python scripts/c4_seg_ab.py [genes]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deseq2_b200 import device as D, device_pipeline as DP, synth  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
m = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
EMU = "libb200nb_emu" in os.environ.get("B200NB_LIB", "")   # dry run of this script on the CPU (tests/simt_emu)
if EMU:
    import ctypes
    import time
    D._stream = lambda: ctypes.c_void_p(0)
x = synth.design_factor(m, 10)
d = synth.make_example_counts(n, m, x=x, seed=11, betaSD=0.5)
dev = torch.device("cpu" if EMU else "cuda")
y = D.to_gene_major(d["counts"], dev)
os.environ["B200NB_PIPE_DEBUG"] = "1"      # a sync after every stage: per-stage wall times
res = DP.DESeq_device(y, x, d["sizeFactors"])
res = DP.DESeq_device(y, x, d["sizeFactors"])
os.environ.pop("B200NB_PIPE_DEBUG")
print("DESeq_device stages (segmented kernels):", res["stage_ms"])
pr = DP.prep(y, x, d["sizeFactors"])
la0 = torch.log(pr["alpha0"])
lfit = torch.log(res["dispFit"])
lam = torch.full((10,), 1e-6 / np.log(2) ** 2, dtype=torch.float64, device=dev)
con = torch.zeros(10, dtype=torch.float64, device=dev)
con[0] = 1
x11 = synth.design_factor_expanded(m, 10)
lam11 = torch.as_tensor(np.r_[1e-6, np.full(10, 1.0 / 0.7)] / np.log(2) ** 2, device=dev)
con11 = torch.zeros(11, dtype=torch.float64, device=dev)
con11[10] = 1
beta11 = torch.zeros((11, y.shape[0]), dtype=torch.float64, device=dev)
beta11[0] = torch.log(torch.clamp(pr["baseMean"], min=0.1))
ev = lambda: torch.cuda.Event(enable_timing=True)


def t(fn, reps=3):
    if EMU:
        t0 = time.perf_counter()
        out = fn()
        return (time.perf_counter() - t0) * 1e3, out
    out = fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        a, b = ev(), ev()
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
    return best, out


def clone(o):
    return {k: v.clone() for k, v in o.items() if torch.is_tensor(v)}


ref = None
MODES = (("1", "12"), ("1", "16")) if os.environ.get("C4_SEG_ONLY") else (("0", ""), ("1", "8"), ("1", "12"), ("1", "16"))
for seg, warps in MODES:
    os.environ["B200NB_GENERIC_SEG"] = seg
    if warps:
        os.environ["B200NB_GENERIC_WARPS"] = warps
    else:
        os.environ.pop("B200NB_GENERIC_WARPS", None)
    t1, o1 = t(lambda: D.fit_disp(y, pr["xd"], pr["mu_lin"], la0, la0, 1.0, float(np.log(1e-9)), 1.0, 1e-6, 100, False))
    o1 = clone(o1)
    t2, o2 = t(lambda: D.fit_disp(y, pr["xd"], pr["mu_lin"], torch.log(res["dispGeneEst"]), lfit, res["dispPriorVar"],
                                  float(np.log(1e-9)), 1.0, 1e-6, 100, True))
    o2 = clone(o2)
    t3, o3 = t(lambda: D.fit_beta(y, pr["xd"], pr["sfd"], res["dispersion"], con, pr["beta0"], lam, 1e-8, 100))
    o3 = clone(o3)
    line = f"seg={seg} warps<={warps or '-':>2s}: fitDisp MLE {t1:6.2f} ms, MAP {t2:6.2f} ms, fitBeta {t3:6.2f} ms"
    try:
        t4, o4 = t(lambda: D.fit_beta(y, x11, pr["sfd"], res["dispersion"], con11, beta11, lam11, 1e-8, 100))
        line += f", fitBeta expanded p=11 {t4:6.2f} ms"
    except Exception as e:   # the A/B of the main shape must not die on the extra case
        line += f" (p=11 skipped: {type(e).__name__}: {e})"
    three = t1 + t2 + t3
    line += f"  | three calls {three:6.2f} ms = {y.shape[0] / three / 1e3:.2f} M genes/s  ({y.shape[0]} genes x {m})"
    print(line)
    cur = (o1, o2, o3)
    if ref is None:
        ref = cur
    else:
        same = ((cur[0]["iter"] == ref[0]["iter"]) & (cur[0]["iter_accept"] == ref[0]["iter_accept"])).double().mean().item()
        dla = (cur[0]["log_alpha"] - ref[0]["log_alpha"]).abs().max().item()
        db = (cur[2]["beta_mat"] - ref[2]["beta_mat"]).abs().max().item()
        it = (cur[2]["iter"] == ref[2]["iter"]).double().mean().item()
        print(f"    vs seg=0: fitDisp identical iter/iter_accept on {100 * same:.2f} % of genes, max|dlog_alpha| {dla:.2e}; "
              f"fitBeta identical iter on {100 * it:.2f} %, max|dbeta| {db:.2e}")
os.environ.pop("B200NB_GENERIC_SEG", None)
os.environ.pop("B200NB_GENERIC_WARPS", None)
