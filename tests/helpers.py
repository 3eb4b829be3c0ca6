"""Shared helpers for the parity tests: realistic fitDisp / fitBeta inputs built with the host glue."""
import functools
import os

import numpy as np
import pytest

from deseq2_b200 import pipeline, synth

# `-m gpu` tests run on "cuda"; when B200NB_LIB points at the emulated engine (tests/simt_emu/_build/libb200nb_emu*.so,
# see tests/test_emulated_kernels.py) the same tests run with CPU tensors: in the emulator device pointers are host
# pointers (tests/conftest.py then also replaces the CUDA stream getters of the torch wrappers by a null stream).
EMULATED = "libb200nb_emu" in os.path.basename(os.environ.get("B200NB_LIB", ""))
DEV = "cpu" if EMULATED else "cuda"


@pytest.fixture(scope="module")
def emu_dev(emu):
    """The emulated engine with CPU tensors: device pointers are host pointers, there is no CUDA stream.  Every binding
    takes its stream from deseq2_b200.device._stream at call time, so replacing that one getter covers them all."""
    import ctypes as C
    from deseq2_b200 import device as D
    saved = D._stream
    D._stream = lambda: C.c_void_p(0)
    try:
        yield emu
    finally:
        D._stream = saved


def gm(a, dev, dtype=None):
    """(n, m) numpy matrix -> gene-major (n, ld) tensor on `dev`: int32 for integer input, float64 otherwise, or
    converted to `dtype` first."""
    import torch
    from deseq2_b200 import device as D
    return D.to_gene_major(np.asarray(a, dtype=dtype), torch.device(dev))


gm64 = functools.partial(gm, dtype=np.float64)          # counts as float64 too: the float64-count path of the kernels


DISP_KEYS = ("log_alpha", "last_change", "initial_lp", "initial_dlp", "last_lp", "last_dlp", "last_d2lp")


def make_case(n, m, x=None, seed=1, drop_zero=True, **kw):
    d = synth.make_example_counts(n, m, x=x, seed=seed, **kw)
    counts = d["counts"]
    if drop_zero:
        counts = counts[counts.sum(axis=1) > 0]
    sf = d["sizeFactors"]
    x = d["x"]
    mv = pipeline.getBaseMeansAndVariances(counts, sf)
    norm = counts / sf[None, :]
    rough = pipeline.roughDispEstimate(norm, x)
    mom = pipeline.momentsDispEstimate(mv["baseMean"], mv["baseVar"], sf)
    alpha0 = np.minimum(np.maximum(1e-8, np.minimum(rough, mom)), max(10, m))
    nf = np.broadcast_to(sf[None, :], counts.shape).copy()
    if pipeline.modelMatrixGroups(x) == x.shape[1]:
        mu = np.maximum(pipeline.linearModelMu(norm, x) * nf, 0.5)
    else:
        mu = None
    Q, R = np.linalg.qr(x)
    beta0 = np.linalg.solve(R, Q.T @ np.log(norm + 0.1).T).T
    return dict(counts=counts, x=x, sf=sf, nf=nf, mu=mu, alpha0=alpha0, beta0=beta0, baseMean=mv["baseMean"],
                trueDisp=d["trueDisp"])


def disp_args(c, mu, log_alpha, prior_mean=None, sigmasq=1.0, usePrior=False, tol=1e-6, maxit=100, weights=None,
              useWeights=False, useCR=True, y=None):
    return dict(ySEXP=c["counts"] if y is None else y, xSEXP=c["x"], mu_hatSEXP=mu, log_alphaSEXP=log_alpha,
                log_alpha_prior_meanSEXP=log_alpha if prior_mean is None else prior_mean,
                log_alpha_prior_sigmasqSEXP=sigmasq, min_log_alphaSEXP=np.log(1e-8 / 10), kappa_0SEXP=1.0,
                tolSEXP=tol, maxitSEXP=maxit, usePriorSEXP=usePrior, weightsSEXP=weights, useWeightsSEXP=useWeights,
                weightThresholdSEXP=1e-2, useCRSEXP=useCR)


def beta_args(c, alpha, beta0=None, lam=None, useQR=True, maxit=100, tol=1e-8, weights=None, useWeights=False,
              contrast=None, nf=None, x=None, y=None):
    x = c["x"] if x is None else x
    p = x.shape[1]
    return dict(ySEXP=c["counts"] if y is None else y, xSEXP=x, nfSEXP=c["nf"] if nf is None else nf,
                alpha_hatSEXP=alpha, contrastSEXP=np.r_[1.0, np.zeros(p - 1)] if contrast is None else contrast,
                beta_matSEXP=c["beta0"] if beta0 is None else beta0,
                lambdaSEXP=np.full(p, 1e-6) / np.log(2) ** 2 if lam is None else lam, weightsSEXP=weights,
                useWeightsSEXP=useWeights, tolSEXP=tol, maxitSEXP=maxit, useQRSEXP=useQR, minmuSEXP=0.5)


def rel_err(a, b, floor=1e-12):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return np.abs(a - b) / np.maximum(np.abs(b), floor)


REFERENCE_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "outputs.npz")
REF_ROWS, REF_COLS = 48, 8


class StoredReference:
    """Outputs of the reference's own src/DESeq2.cpp (compiled unchanged into oracle/_ref, see oracle/ref.py) on the
    tests' inputs, stored in tests/golden/reference/outputs.npz so that the comparisons run without the reference.

    Every call names its case.  The file keeps, per case, the outputs at a fixed seeded sample of REF_ROWS genes
    (`rows`; every gene for fitDispGrid) and, for the genes x samples hat diagonals, of REF_COLS samples (`cols`);
    `at(result, stored)` picks the same entries out of a full result.  tests/golden/reference/make.py rewrites the file: with
    DESEQ2_RECORD_REFERENCE=1 every call runs the reference library and records what it returned."""

    def __init__(self):
        self.record = os.environ.get("DESEQ2_RECORD_REFERENCE") == "1"
        self.stored = dict(np.load(REFERENCE_GOLDEN)) if os.path.exists(REFERENCE_GOLDEN) else {}
        if self.record:
            from oracle import ref as R
            R.build()
            self.R = R

    def _call(self, fn, case, kw):
        if self.record:
            out = getattr(self.R, fn)(**kw)
            n = len(out["log_alpha"] if "log_alpha" in out else out["beta_mat"])
            rng = np.random.default_rng(int.from_bytes(case.encode(), "little") % 2 ** 63)
            keep = n if fn == "fitDispGrid" else min(n, REF_ROWS)     # one small vector: kept whole
            rows = np.sort(rng.choice(n, keep, replace=False))
            m = np.asarray(kw["ySEXP"]).shape[1]
            cols = np.sort(rng.choice(m, min(m, REF_COLS), replace=False))
            for k, v in at(out, {"rows": rows, "cols": cols}).items():
                self.stored[f"{case}/{k}"] = v
            self.stored[f"{case}/rows"], self.stored[f"{case}/cols"] = rows.astype(np.int32), cols.astype(np.int32)
            np.savez_compressed(REFERENCE_GOLDEN, **self.stored)
        pre = case + "/"
        got = {k[len(pre):]: v for k, v in self.stored.items() if k.startswith(pre)}
        assert got, f"no stored reference outputs for case {case!r} (tests/golden/reference/make.py)"
        return got

    def fitDisp(self, case, **kw):
        return self._call("fitDisp", case, kw)

    def fitDispGrid(self, case, **kw):
        return self._call("fitDispGrid", case, kw)

    def fitBeta(self, case, **kw):
        return self._call("fitBeta", case, kw)


def at(res, stored):
    """The entries of a full fitDisp / fitBeta / fitDispGrid result that a StoredReference case holds."""
    rows, cols = stored["rows"], stored["cols"]
    out = {}
    for k, v in res.items():
        if k in ("rows", "cols"):
            continue
        v = np.asarray(v)
        out[k] = v[rows][:, cols] if k == "hat_diagonals" else v[rows]
    return out
