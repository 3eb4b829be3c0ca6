"""Every IRLS fit kernel against a 40-digit fitBeta, one iteration at a time.

fitBeta (src/DESeq2.cpp:283-465) gives every DESeq() result its coefficients, their sandwich variances, the hat
diagonals of Cook's distances, the contrast of getContrast and the deviance.  The device runs it on several kernel
families: the small-p kernels (P = 1..4; 8-, 16- and 32-lane groups; indicator and general variants: fit_beta.cu,
fit_beta_grp.cuh), the general-p kernel (fit_generic.cu, rows in shared memory or in global memory at rows_global 1
and 2), the segmented long-row kernel (fit_generic_seg.cuh) and rlog's O(m) arrow-matrix kernel (rlog.cuh, at the end
of this file: 8, 16 and 32 lanes, size factors or an nf matrix, fitted or frozen intercept).  This file checks each of
them against a plain
restatement of fitBeta at 40 digits (mpmath) that takes its float64 inputs as exact values:

  * one IRLS step from a given beta: mu = max(nf e^(x beta), minmu), w = [wt] mu / (1 + alpha mu),
    z = log(mu / nf) + (y - mu) / mu, (X'WX + Lambda) beta' = X'Wz;
  * the post-loop block at a given beta: hat diagonals, the sandwich (X'WX + L)^-1 X'WX (X'WX + L)^-1, contrast_num,
    contrast_denom, the clamped mean and the deviance -2 sum [wt] log NB;
  * the rules: |beta_k| > 30 -> iter = maxit with the diverged beta kept and the mean, post-loop block and deviance of
    the previous pass (deviance 0 at the first iteration); the stop test |dev - dev_old| / (|dev| + 0.1) < tol from the
    second iteration on; maxit = 0 -> iter 0, deviance 0 and the post-loop block at the start.

The kernels are deterministic (no floating-point atomics, a fixed order of arithmetic per gene), so a call with
maxit = k returns the k-th iterate of the full fit.  Each case runs k = 0, 1, ..., iter and checks run k against the
restatement evaluated at the device's own iterate k - 1: rounding errors never have to be carried through an iteration
(IRLS is not contractive for every NB gene, so carrying them would make any bound loose or wrong).  The run with
maxit = iter must reproduce the maxit = 100 run bit for bit.

Every bound is derived in _Bounds from per-sample error budgets of the kernel's arithmetic; the linear-algebra parts
are taken entrywise through |A^-1|, A = X'WX + Lambda, with the backward error of a Cholesky factorisation of the
Jacobi-equilibrated D A D, D = diag(A)^-1/2 (the matrix the kernels factor), so they scale with kappa(DAD) and not with
kappa(A).  Each test prints the largest ratio of error to bound per output.

Each case runs on the SIMT-emulated engine on every CPU run (backend "emu": the product's CUDA sources compiled by g++,
tests/simt_emu/), where the launch log shows which kernel ran it, and again on the H100 under -m gpu, which adds one
50 000 x 100 fit.  CPU run time of the emulated half: about 2 minutes on one core, once the emulated engine is built
(measured with `pytest tests/test_irls_reference.py -m "not gpu"`)."""
import math

import mpmath
import numpy as np
import pytest

from helpers import chol_backward, sandwich_bound
from test_optim_loglik_reference import (DPS, EPS, LN2, MINMU, RIDGE, _loglik_scale, _mp, _nb, _prior_lambda, _T,
                                         backend, ref_logdens, x_batch_condition, x_condition, x_covariate,
                                         x_expanded10, x_factor10, x_p32)
from test_sample_counts import LONG_ROWS, _emu_lib, generic_last, grp16_last, launch_log

__all__ = ["backend"]          # the fixture, shared with test_optim_loglik_reference

TOL = 1e-8                     # DESeq()'s betaTol
MAXIT = 100
LARGE = 30.0                   # src/DESeq2.cpp:316


# ---------------------------------------------------------------- the 40-digit restatement of fitBeta

def _finite(b):
    return bool(np.all(np.isfinite(b)))


class Gene:
    """One row of fitBeta: counts y (m), design x (m, p), normalization factors nf (m), weights w (m or None),
    dispersion alpha, ridge lam (p, natural-log scale), minmu."""

    def __init__(self, y, x, nf, w, alpha, lam, minmu=MINMU):
        self.y = np.asarray(y, dtype=np.float64)
        self.x = np.asarray(x, dtype=np.float64)
        self.nf = np.asarray(nf, dtype=np.float64)
        self.w = None if w is None else np.asarray(w, dtype=np.float64)
        self.alpha, self.lam, self.minmu = float(alpha), np.asarray(lam, dtype=np.float64), float(minmu)
        self.m, self.p = self.x.shape
        self._cache = {}
        with mpmath.workdps(DPS):
            self.mx = [[_mp(v) for v in row] for row in self.x]
            self.mnf = [_mp(v) for v in self.nf]
            self.mlnf = [mpmath.log(v) for v in self.mnf]
            self.mw = [mpmath.mpf(1)] * self.m if self.w is None else [_mp(v) for v in self.w]
            self.my = [_mp(v) for v in self.y]

    def state(self, b):
        """Everything fitBeta forms from mu at coefficients b (float64, taken as exact): the clamped mean, the
        working weights and response, B = X'WX, A = B + Lambda, r = X'Wz and the deviance, at 40 digits."""
        b = np.asarray(b, dtype=np.float64)
        key = b.tobytes()
        if key in self._cache:
            return self._cache[key]
        m, p = self.m, self.p
        with mpmath.workdps(DPS):
            a = _mp(self.alpha)
            mmin = _mp(self.minmu)
            mb = [_mp(v) for v in b]
            mu, eta, clamped = [], [], []
            for j in range(m):
                if not _finite(b):
                    # a NaN coefficient: x beta is NaN and fmax(NaN, minmu) = minmu (src/DESeq2.cpp:326)
                    e, v = mpmath.mpf(0), mmin
                    clamped.append(True)
                else:
                    e = mpmath.fsum(self.mx[j][k] * mb[k] for k in range(p))
                    v = self.mnf[j] * mpmath.exp(e)
                    clamped.append(v < mmin)
                    v = max(v, mmin)
                eta.append(e)
                mu.append(v)
            lmn = [mpmath.log(mu[j] / self.mnf[j]) if clamped[j] else eta[j] for j in range(m)]
            W = [self.mw[j] * mu[j] / (1 + a * mu[j]) for j in range(m)]
            z = [lmn[j] + (self.my[j] - mu[j]) / mu[j] for j in range(m)]
            B = mpmath.matrix(p, p)
            r = mpmath.matrix(p, 1)
            for k in range(p):
                r[k] = mpmath.fsum(self.mx[j][k] * W[j] * z[j] for j in range(m) if self.x[j, k] != 0)
                for q in range(k + 1):
                    B[k, q] = B[q, k] = mpmath.fsum(self.mx[j][k] * W[j] * self.mx[j][q] for j in range(m)
                                                    if self.x[j, k] != 0 and self.x[j, q] != 0)
            A = B + mpmath.diag([_mp(v) for v in self.lam])
            Ai = A ** -1
            dev = -2 * mpmath.fsum(self.mw[j] * ref_logdens(self.y[j], mu[j], self.alpha)
                                   for j in range(m) if self.mw[j] != 0)
        st = dict(mu=mu, W=W, z=z, eta=eta, clamped=clamped, B=B, A=A, Ai=Ai, r=r, dev=dev,
                  f=dict(mu=np.array([float(v) for v in mu]), W=np.array([float(v) for v in W]),
                         z=np.array([float(v) for v in z]), eta=np.array([float(v) for v in eta]),
                         B=_f(B), A=_f(A), Ai=_f(Ai), r=np.array([float(v) for v in r]), dev=float(dev)))
        self._cache[key] = st
        return st

    def step(self, b):
        """One IRLS step from b: (X'WX + Lambda)^-1 X'Wz at the mean of b, 40 digits."""
        st = self.state(b)
        with mpmath.workdps(DPS):
            return st["Ai"] * st["r"]

    def post(self, b, contrast):
        """The post-loop block at b (src/DESeq2.cpp:429-455): hat diagonals, sandwich, contrast, mean, deviance."""
        st = self.state(b)
        with mpmath.workdps(DPS):
            Ai, B = st["Ai"], st["B"]
            S = Ai * B * Ai
            c = mpmath.matrix([_mp(v) for v in contrast])
            hat = []
            for j in range(self.m):
                xj = mpmath.matrix(self.mx[j])
                hat.append(st["W"][j] * (xj.T * Ai * xj)[0])
            cd2 = (c.T * S * c)[0]
            cn = mpmath.fsum(c[k] * _mp(b[k]) for k in range(self.p)) if _finite(b) else mpmath.nan
            return dict(S=_f(S), var=np.array([float(S[k, k]) for k in range(self.p)]),
                        hat=np.array([float(v) for v in hat]), cn=float(cn), cd=float(mpmath.sqrt(cd2)),
                        mu=st["f"]["mu"], dev=st["f"]["dev"])


def _f(M):
    return np.array([[float(M[i, k]) for k in range(M.cols)] for i in range(M.rows)])


# ---------------------------------------------------------------- the bounds

class _Bounds:
    """Error budgets of the kernel's arithmetic at coefficients b (its own iterate), from the exact state there.

    Per sample: the kernel forms eta = x b by p FMAs and le = eta + fl(log nf), so |d le| <= (p + 2) eps (|x| |b| +
    |log nf|) (as _f64_err states); exp_fast is within 1 ulp (test_optim_loglik_reference), so mu carries a relative
    error dmu = dle + 2 eps, clamped or not (the clamp is 1-Lipschitz); w = mu rcp(1 + alpha mu) [wt] adds 4 roundings;
    z = (le - log nf) + (y rcp(mu) - 1) carries dle + 3 eps (|eta| + |log nf| + |log mu| + 1) + y / mu (dmu + 3 eps).
    Sums over the m samples, in any order: (m + 2) eps times the sum of the magnitudes of the terms.  So X'WX carries
    E_B = |X|' diag(w (dw + (m + 2) eps)) |X| and X'Wz e_r = |X|' (w |dz| + w |z| (dw + (m + 3) eps))."""

    def __init__(self, g, b, st, dle_extra=0.0):
        f = st["f"]
        m, p = g.m, g.p
        bb = np.nan_to_num(np.asarray(b, dtype=np.float64), nan=0.0)
        lnf = np.abs(np.log(g.nf))
        nanb = not _finite(b)
        self.xb = np.abs(g.x) @ np.abs(bb)
        dle = np.zeros(m) if nanb else (p + 2) * EPS * (self.xb + lnf) + dle_extra
        self.dmu = dle + 2 * EPS
        dw = self.dmu + 4 * EPS
        mu, W, z = f["mu"], f["W"], f["z"]
        dz = dle + 3 * EPS * (np.abs(f["eta"]) + lnf + np.abs(np.log(mu)) + 1) + g.y / mu * (self.dmu + 3 * EPS)
        cs = (m + 2) * EPS
        ax = np.abs(g.x)
        self.E_B = ax.T @ ((W * (dw + cs))[:, None] * ax)
        self.E_A = self.E_B + chol_backward(f["A"], p)
        self.e_r = ax.T @ (W * dz + W * np.abs(z) * (dw + cs + EPS))
        self.dw = dw


def _a_norm(d, A):
    return math.sqrt(max(float(d @ A @ d), 0.0))


def step_bound(g, b_prev, beta_star):
    """||beta_dev - beta*||_A for the kernel's step from b_prev: (A + dA) beta = r + dr to first order gives
    A (beta - beta*) = dr - dA beta*, and ||A^-1 v||_A = sqrt(v' A^-1 v) <= sqrt(|v|' |A^-1| |v|) with
    |v| <= e_r + E_A |beta*|.  The second-order rest is below 1% while kappa(DAD) (3p + 6) eps < 1e-2 (asserted).
    Plus the rounding of beta itself to float64 (2 ulp per coefficient: the solve's last division and scaling)."""
    st = g.state(b_prev)
    f = st["f"]
    bd = _Bounds(g, b_prev, st)
    bs = np.array([float(v) for v in beta_star])
    v = bd.e_r + bd.E_A @ np.abs(bs)
    d = 1.0 / np.sqrt(np.diag(f["A"]))
    kdad = np.linalg.cond(d[:, None] * f["A"] * d[None, :])
    assert kdad * (3 * g.p + 6) * EPS < 1e-2, kdad
    u = 2 * np.spacing(np.abs(bs))
    return 1.01 * math.sqrt(float(v @ np.abs(f["Ai"]) @ v)) + math.sqrt(float(u @ np.abs(f["A"]) @ u)), kdad


def post_bounds(g, b, contrast, ref, dle_extra=0.0):
    """Bounds of the post-loop outputs at b (see _Bounds and sandwich_bound):
      hat_j = w_j x_j' A^-1 x_j: w_j (q_j dw_j + (p^2 + 6) eps |x_j|' |A^-1| |x_j| + |x_j|' |A^-1| E_A |A^-1| |x_j|);
      beta_var: the diagonal of sandwich_bound; contrast_denom = sqrt(c' S c): e = |c|' dS |c| + 2 p eps |c|' |S| |c|,
      then min(e / cd, sqrt(e)) + eps cd; contrast_num = c' b by p FMAs: 2 p eps |c|' |b|;
      mu: mu dmu; deviance: 2 (m + 16) eps sum_j _loglik_scale (the bound of test_nb_loglik_against_40_digits, with
      m + 16 roundings for the two m-term sums of the direct form and the hoisted constant)."""
    st = g.state(b)
    f = st["f"]
    bd = _Bounds(g, b, st, dle_extra)
    p, m = g.p, g.m
    aAi = np.abs(f["Ai"])
    ax = np.abs(g.x)
    q = np.einsum("jk,kl,jl->j", g.x, f["Ai"], g.x)
    qa = np.einsum("jk,kl,jl->j", ax, aAi, ax)
    qe = np.einsum("jk,kl,jl->j", ax, aAi @ bd.E_A @ aAi, ax)
    hat = f["W"] * (np.abs(q) * bd.dw + (p * p + 6) * EPS * qa + qe)
    dS = sandwich_bound(f["Ai"], f["B"], ref["S"], bd.E_A, bd.E_B, p)
    ac = np.abs(contrast)
    e = ac @ dS @ ac + 2 * p * EPS * ac @ np.abs(ref["S"]) @ ac
    cd = ref["cd"]
    cdb = (min(e / cd, math.sqrt(e)) if cd > 0 else math.sqrt(e)) + EPS * cd
    bb = np.nan_to_num(np.asarray(b, dtype=np.float64), nan=0.0)
    cnb = 2 * p * EPS * float(ac @ np.abs(bb))
    w = np.ones(m) if g.w is None else g.w
    scale = sum(_loglik_scale(g.y[j], f["mu"][j], g.alpha, w[j], bd.xb[j], abs(math.log(g.nf[j])))
                for j in range(m))
    devb = 2 * (m + 16) * EPS * scale
    return dict(hat=hat, var=np.diag(dS).copy(), cd=cdb, cn=cnb, mu=f["mu"] * bd.dmu, dev=devb)


# ---------------------------------------------------------------- cases

def x_intercept(m):
    return np.ones((m, 1))


def x_collinear(m):
    """Two nearly collinear covariates: kappa(DAD) of X'X about 1e8."""
    rng = np.random.default_rng(7)
    u = rng.normal(0.0, 1.0, m)
    return np.c_[np.ones(m), u, u + 2e-4 * rng.normal(0.0, 1.0, m)]


def x_cov6(m):
    rng = np.random.default_rng(m)
    return np.c_[np.ones(m), rng.normal(0.0, 0.4, (m, 5))]        # p = 6, > 32 distinct rows: samplewise


DESIGNS = {"int": x_intercept, "cond": x_condition, "batch": x_batch_condition, "cov": x_covariate,
           "colin": x_collinear, "f10": x_factor10, "exp10": x_expanded10, "p32": x_p32, "cov6": x_cov6}

ALPHAS = (1e-8, 1e-3, 0.1, 1.0, 10.0, "m")
# row kinds: "qr" the QR start; "zero" beta = 0; "zcell" a cell of zeros (mu at minmu); "big" counts ~1e7 (hat near 1);
# "diverge" counts ~1e7 from beta = 0 (the first step passes |beta| > 30); "nan" a NaN start; "frac" non-integer counts
ROWS = ("qr", "zero", "zcell", "big", "diverge", "nan")

# The small-p lane widths: 8 up to m = 40 (group_lanes_beta), 16 up to grp16_last, then a warp.
L16_P2 = grp16_last("beta", 2, False, True)
L16_P4W = grp16_last("beta", 4, True, False)
ROWS2_M = generic_last(1, "beta", 6, 0, False, True, False) + 1      # rows_global 2: p = 6 samplewise, w, nf matrix

# (name, design, m, nf, weights, counts dtype, ridge, contrast, rows, environment, expected route)
#   nf: "sf" a size-factor vector, "matrix" a gene-major matrix, "tiny" a vector ~1e-3 (non-zero rows reach minmu);
#   weights: None, "unif" uniform(0.3, 1) with exact zeros, "group0" a whole condition at weight 0;
#   ridge: a number (natural-log lambda for every coefficient) or "prior" (estimate_beta_prior_var, expanded matrix);
#   contrast: "last" e_p, a list, or "exp" an expanded-matrix contrast; route: the kernel the emulator must launch
#   (kernel family, lanes or rows level, indicator variant).
CASES = [
    ("smallp-p1-int-l8", "int", 12, "sf", None, "i4", RIDGE, "last", ("qr", "zero", "big", "nan"), {},
     ("grp", 8, True)),
    ("smallp-p2-cond-l8-ind", "cond", 10, "sf", None, "i4", RIDGE, "last", ROWS, {}, ("grp", 8, True)),
    ("smallp-p2-cond-l8-w0", "cond", 16, "tiny", "group0", "f8", RIDGE, "last", ("qr", "zero", "zcell", "frac"), {},
     ("grp", 8, True)),
    ("smallp-p2-cov-l16-w", "cov", 48, "sf", "unif", "f8", RIDGE, "last", ("qr", "zero", "frac", "nan"), {},
     ("grp", 16, False)),
    ("smallp-p3-colin-l8", "colin", 20, "matrix", None, "f8", RIDGE, "last", ("qr", "zero", "frac"), {},
     ("grp", 8, False)),
    ("smallp-p4-batch-l32-w", "batch", L16_P4W + 1, "matrix", "unif", "i4", RIDGE, [0, 1, -1, 0],
     ("qr", "zcell", "big"), {}, ("warp", 32, True)),
    ("smallp-p2-cond-l32", "cond", L16_P2 + 1, "sf", None, "i4", RIDGE, "last", ("qr", "zcell"),
     {"B200NB_LONG_ROWS": "0"}, ("warp", 32, True)),
    ("smallp-p4-batch-l16", "batch", 60, "sf", None, "f8", RIDGE, [0, 1, -1, 0], ("qr", "zcell", "frac"), {},
     ("grp", 16, True)),
    ("generic-f10-grouped-w", "f10", 40, "sf", "unif", "i4", RIDGE, "last", ("qr", "zcell", "zero"), {},
     ("generic", 0, None)),
    ("generic-exp10-prior", "exp10", 40, "sf", None, "i4", "prior", "exp", ("qr", "zcell", "zero"),
     {"B200NB_GENERIC_SEG": "0"}, ("generic", 0, None)),
    ("generic-p32", "p32", 96, "matrix", "unif", "f8", RIDGE, "last", ("qr",), {}, ("generic", 0, None)),
    ("generic-cov6-rows1", "cov6", 60, "matrix", "unif", "i4", RIDGE, "last", ("qr", "zero", "nan"),
     {"B200NB_GENERIC_ROWS": "global"}, ("generic", 1, None)),
    ("generic-cov6-rows2", "cov6", ROWS2_M, "matrix", "unif", "i4", RIDGE, "last", ("qr",), {},
     ("generic", 2, None)),
    ("seg-cond-long", "cond", LONG_ROWS, "sf", None, "i4", RIDGE, "last", ("qr", "zcell"), {}, ("seg", None, None)),
    ("seg-exp10-prior", "exp10", 40, "sf", None, "i4", "prior", "exp", ("qr", "zcell", "diverge"), {},
     ("seg", None, None)),
]


def _contrast(kind, p):
    if kind == "last":
        return np.r_[np.zeros(p - 1), 1.0]
    if kind == "exp":                                  # level 2 against level 1 of the expanded matrix
        c = np.zeros(p)
        c[2], c[1] = 1.0, -1.0
        return c
    return np.asarray(kind, dtype=np.float64)


def _inputs(case, backend):
    name, design, m, nfk, wk, dt, ridge, ck, kinds = case[:9]
    D, DP, dev, _ = backend
    rng = np.random.default_rng(sum(map(ord, name)))
    x = DESIGNS[design](m)
    n = len(kinds)
    p = x.shape[1]
    sf = np.exp(rng.normal(0.0, 0.25, m))
    sf /= np.exp(np.mean(np.log(sf)))
    if nfk == "tiny":
        sf *= 1e-3
    nf = np.broadcast_to(sf, (n, m)).copy()
    if nfk == "matrix":
        nf *= np.exp(rng.normal(0.0, 0.2, (n, m)))
    am = [float(max(10, m)) if a == "m" else a for a in ALPHAS]
    alphas = np.array([am[(g + len(name)) % len(am)] for g in range(n)])
    y = np.zeros((n, m))
    start = np.zeros((n, p))
    last = x[:, -1] != 0
    Q, R = np.linalg.qr(x) if np.linalg.matrix_rank(x) == p else (None, None)
    for g, kind in enumerate(kinds):
        b_true = np.r_[rng.uniform(2.0, 6.0), rng.normal(0.0, 0.7, p - 1)]
        if p > 1 and x[:, 1:].std() > 100:
            b_true[1:] /= 1000.0
        if nfk == "tiny":
            b_true[0] = rng.uniform(4.0, 6.5)                # counts of a few; nf * e^(x beta) near or below minmu
        mu = nf[g] * np.exp(x @ b_true)
        y[g] = _nb(rng, mu, min(alphas[g], 1.0))
        if kind in ("big", "diverge"):
            y[g] = np.round(1e7 * np.exp(x @ np.r_[0.0, rng.normal(0.0, 0.3, p - 1)]) * rng.uniform(0.95, 1.05, m))
        if kind == "zcell":
            y[g, last] = 0.0
        if kind == "frac" or (dt == "f8" and kind not in ("big", "diverge")):
            y[g] = y[g] + np.where(y[g] > 0, rng.uniform(0.0, 1.0, m).round(3), 0.0)
        if kind in ("zero", "diverge"):
            start[g] = 0.0
        elif kind == "nan":
            start[g] = np.nan
        elif Q is not None:
            start[g] = np.linalg.solve(R, Q.T @ np.log(y[g] / nf[g] + 0.1))
        else:                                                # rank-deficient expanded matrix: fitNbinomGLMs' start
            start[g] = np.r_[np.log(np.mean(y[g] / nf[g]) + 0.1), np.zeros(p - 1)]
    if dt == "i4":
        assert np.all(y == np.round(y)) and y.max() < 2 ** 31
    w = None
    if wk == "unif":
        w = rng.uniform(0.3, 1.0, (n, m))
        w[:, 0] = 0.0
        w[:, 1] = 0.0
    elif wk == "group0":
        w = rng.uniform(0.3, 1.0, (n, m))
        w[:, last] = 0.0                                     # a whole group at weight 0: its coefficient is ridge-only
    lam = _prior_lambda(D, DP, dev, m) if ridge == "prior" else np.full(p, float(ridge))
    return x, y, nf, w, alphas, lam, _contrast(ck, p), start, sf


class _Run:
    """fit_beta on the device at any maxit, outputs as numpy."""

    def __init__(self, backend, x, y, nf, w, alphas, lam, contrast, start, dt, nf_vector):
        import torch
        D, DP, dev, _ = backend
        self.D, self.m = D, x.shape[0]
        self.yd = D.to_gene_major(y.astype(np.int32) if dt == "i4" else y, dev)
        self.xd = D.x_to_device(x, dev)
        self.nfd = _T(nf[0], dev) if nf_vector else D.to_gene_major(nf, dev)
        self.wd = None if w is None else D.to_gene_major(w, dev)
        self.ad, self.cd, self.ld = _T(alphas, dev), _T(contrast, dev), _T(lam, dev)
        self.bd = _T(np.ascontiguousarray(start.T), dev)
        self.torch = torch

    def __call__(self, maxit):
        r = self.D.fit_beta(self.yd, self.xd, self.nfd, self.ad, self.cd, self.bd, self.ld, TOL, maxit,
                            weights=self.wd)
        out = {k: v.cpu().numpy() for k, v in r.items() if v is not None}
        out["beta_mat"], out["beta_var_mat"] = out["beta_mat"].T.copy(), out["beta_var_mat"].T.copy()
        out["hat_diagonals"] = out["hat_diagonals"][:, :self.m].copy()
        out["mu"] = out["mu"][:, :self.m].copy()
        return out


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _routes(log):
    """(family, lanes or None, indicator variant or None) of the IRLS launches that did the work.  The small-p launches
    come in pairs (general, then indicator variant); the variant that does not fit the design returns after one
    collective (the last field of a log line), the other one runs the genes."""
    out = set()
    lines = [[s.strip() for s in ln.split(" | ")] for ln in log.splitlines() if ln.strip()]
    small = [ln for ln in lines if "launch_beta_grp" in ln[1] or "launch_beta_t" in ln[1]]
    for i in range(0, len(small) - 1, 2):
        gen, ind = small[i], small[i + 1]
        work = ind if int(ind[4]) > 1 else gen
        if "launch_beta_grp" in work[1]:
            lanes = int(work[1].split("int GL = ")[1].split(";")[0])
            out.add(("grp", lanes, work is ind))
        else:
            out.add(("warp", 32, work is ind))
    for ln in lines:
        if ln[0] == "fit_beta_generic_kernel":
            out.add(("generic", None, None))
        elif ln[0].startswith("fit_beta_seg_kernel") or "launch_beta_seg_t" in ln[1]:
            out.add(("seg", None, None))
    return out


RATIOS = {}


def _ratio(fam, key, err, bound):
    err, bound = np.atleast_1d(np.abs(err)), np.atleast_1d(bound)
    r = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))))
    RATIOS.setdefault(fam, {})
    RATIOS[fam][key] = max(RATIOS[fam].get(key, 0.0), r)
    return r


def check_chain(tag, fam, run, genes, contrast, full, sample=None):
    """The per-iteration checks of every gene in `sample` (all by default) against the 40-digit restatement.
    Returns the number of genes whose stop decision lay within the deviances' error bounds."""
    n = len(genes)
    sample = range(n) if sample is None else sample
    end = {}
    for g in sample:
        it = full["iter"][g]
        if it < MAXIT:
            end[g] = int(it)
        else:
            assert np.any(np.abs(full["beta_mat"][g]) > LARGE), f"{tag} gene {g}: neither converged nor diverged"
            end[g] = None                                    # found below: the first iterate past |beta| > 30
    open_ = set(sample)
    prev = None
    knife = 0
    k = 0
    while open_:
        assert k <= MAXIT
        cur = run(k)
        for g in sorted(open_):
            gt = f"{tag} gene {g} (alpha {genes[g].alpha:g}) k={k}"
            gene = genes[g]
            b = cur["beta_mat"][g]
            diverged = k >= 1 and _finite(b) and np.any(np.abs(b) > LARGE)     # the start is not tested
            assert cur["iter"][g] == k, (gt, cur["iter"][g])
            if k >= 1:
                bp = prev["beta_mat"][g]
                bs = gene.step(bp)
                with mpmath.workdps(DPS):
                    d = np.array([float(_mp(b[i]) - bs[i]) for i in range(gene.p)])
                A = gene.state(bp)["f"]["A"]
                bound, kdad = step_bound(gene, bp, bs)
                err = _a_norm(d, A)
                assert _ratio(fam, "beta", err, bound) <= 1.0, f"{gt}: ||beta - beta*||_A {err:.3e} > {bound:.3e}"
            if diverged:
                # |beta| > 30: the diverged beta is kept; the mean, the post-loop block and the deviance are those of
                # the previous pass, so they equal run k - 1's bit for bit (the deviance is 0 at k = 1, as in run 0)
                assert k >= 1, gt
                for key in ("beta_var_mat", "hat_diagonals", "mu", "contrast_denom", "deviance"):
                    assert _same(cur[key][g], prev[key][g]), (gt, key)
                if k == 1:
                    assert cur["deviance"][g] == 0.0, gt
                ref = gene.post(prev["beta_mat"][g], contrast)
                cn = float(mpmath.fsum(_mp(contrast[i]) * _mp(b[i]) for i in range(gene.p)))
                assert abs(cur["contrast_num"][g] - cn) <= 2 * gene.p * EPS * np.abs(contrast) @ np.abs(b), gt
                assert end[g] is None or end[g] == k, gt
                end[g] = k
            else:
                ref = gene.post(b, contrast)
                bnd = post_bounds(gene, b, contrast, ref)
                got = dict(hat=cur["hat_diagonals"][g], var=cur["beta_var_mat"][g], cd=cur["contrast_denom"][g],
                           cn=cur["contrast_num"][g], mu=cur["mu"][g],
                           dev=cur["deviance"][g])
                want = dict(ref)
                if k == 0:
                    want["dev"], bnd["dev"] = 0.0, 0.0               # maxit = 0: no pass is scored
                for key in ("hat", "var", "cd", "cn", "mu", "dev"):
                    if key == "cn" and not _finite(b):
                        assert np.isnan(got[key]), gt
                        continue
                    err = np.abs(np.asarray(got[key]) - np.asarray(want[key]))
                    r = _ratio(fam, key, err, bnd[key])
                    assert r <= 1.0, f"{gt}: {key} off by {np.max(err):.3e}, {r:.3g} x its bound"
                # the stop decision at k, from the exact deviances at the device's iterates k - 1 and k; the test does
                # not apply at the first iteration
                if k == 1:
                    assert end[g] != 1, f"{gt}: stopped at the first iteration"
                if k >= 2:
                    d0 = genes[g].state(prev["beta_mat"][g])["dev"]
                    d1 = gene.state(b)["dev"]
                    with mpmath.workdps(DPS):
                        conv = float(abs(d1 - d0) / (abs(d1) + mpmath.mpf("0.1")))
                    e0 = post_bounds(gene, prev["beta_mat"][g], contrast, gene.post(prev["beta_mat"][g], contrast))["dev"]
                    e1 = bnd["dev"]
                    econv = (e0 + e1) / (abs(float(d1)) + 0.1) * (1 + conv) * 1.01
                    stopped = end[g] == k
                    if abs(conv - TOL) <= econv:
                        knife += 1
                    else:
                        assert stopped == (conv < TOL), f"{gt}: stop {stopped}, 40-digit conv_test {conv:.3e}"
            if end[g] == k:
                # determinism: the run that stops here reproduces the maxit = 100 run bit for bit
                for key in ("beta_mat", "beta_var_mat", "hat_diagonals", "mu", "contrast_num", "contrast_denom",
                            "deviance"):
                    assert _same(cur[key][g], full[key][g]), (gt, key, "differs from the maxit = 100 run")
                if not diverged:
                    assert full["iter"][g] == k, gt
                open_.discard(g)
        prev = cur
        k += 1
    return knife


def _family(route):
    kind, lanes, ind = route
    if kind in ("grp", "warp"):
        return f"small-p {lanes} lanes {'ind' if ind else 'gen'}"
    if kind == "generic":
        return f"general-p rows_global {lanes}"
    return "segmented"


def _report(name, knife=0):
    print(f"\n{name}: largest error / bound per output")
    for fam, r in sorted(RATIOS.items()):
        print("  " + fam + ": " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(r.items())))
    print(f"  stop decisions within the deviances' error bounds: {knife}")


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_irls_chain_against_40_digits(backend, case, monkeypatch):
    name, design, m, nfk, wk, dt, ridge, ck, kinds, env, route = case
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    D, DP, dev, _ = backend
    x, y, nf, w, alphas, lam, contrast, start, sf = _inputs(case, backend)
    run = _Run(backend, x, y, nf, w, alphas, lam, contrast, start, dt, nfk != "matrix")
    emu = dev.type == "cpu"
    if emu:
        launch_log(_emu_lib())
    full = run(MAXIT)
    if emu:
        got = _routes(launch_log(_emu_lib()))
        want = (route[0], route[1] if route[0] in ("grp", "warp") else None, route[2])
        assert got == {want}, f"{name}: launched {got}, expected {want}"
    if route[0] == "generic" and env.get("B200NB_GENERIC_ROWS") is None:
        from test_sample_counts import generic_level
        G = len(np.unique(x, axis=0))
        grouped = G <= 32
        assert generic_level("beta", m, x.shape[1], G if grouped else 0, grouped, w is not None,
                             nfk != "matrix") == route[1], name
    genes = [Gene(y[g], x, nf[g], None if w is None else w[g], alphas[g], lam) for g in range(len(y))]
    fam = _family(route)
    knife = check_chain(name, fam, run, genes, contrast, full)
    kinds_div = [g for g, kd in enumerate(kinds) if kd == "diverge"]
    for g in kinds_div:
        assert full["iter"][g] == MAXIT and np.any(np.abs(full["beta_mat"][g]) > LARGE), f"{name} gene {g}"
    _report(name, knife)


# ---------------------------------------------------------------- the sandwich of DESeq_device and getContrast_device

def test_deseq_betase_and_contrast_se_are_the_sandwich(backend):
    """DESeq_device's betaSE and getContrast_device's lfcSE equal the 40-digit sandwich at the returned coefficients
    divided by ln 2, within post_bounds's bounds (and the roundings of the sqrt and of the division by ln 2).  The
    natural-log coefficients are recovered from the log2 ones as fl(fl(beta / ln 2) ln 2), within 3 ulp of the
    kernel's (two roundings and that of ln 2 itself), so the kernel's x beta is within 3 eps |x| |b| of the one the
    restatement uses: _Bounds adds that to its per-sample error of le, from where it reaches mu, w and the sums.  This is where the
    ridge scale, the normalised weights and the factors reach the kernel."""
    D, DP, dev, _ = backend
    rng = np.random.default_rng(90)
    m, n = 8, 40
    x = x_condition(m)
    sf = np.exp(rng.normal(0.0, 0.2, m))
    sf /= np.exp(np.mean(np.log(sf)))
    b_true = np.c_[rng.uniform(2.0, 7.0, n), rng.normal(0.0, 1.0, n)]
    y = np.array([_nb(rng, sf * np.exp(x @ b_true[g]), 0.1) for g in range(n)])
    y[3, 4:] = 0
    w = rng.uniform(0.3, 1.0, (n, m))
    yd = D.to_gene_major(y.astype(np.int32), dev)
    wd = D.to_gene_major(w, dev)
    res = DP.DESeq_device(yd, x, sf, weights=wd)
    idx = res["idx"].cpu().numpy()
    bm = res["betaMatrix"].cpu().numpy()
    se = res["betaSE"].cpu().numpy()
    disp = res["dispersion"].cpu().numpy()
    wn = w[idx] / w[idx].max(axis=1, keepdims=True)          # the weights DESeq() normalises by the row maximum
    contrast = np.r_[0.0, 1.0]
    gc = DP.getContrast_device(yd[_T(idx, dev)].contiguous(), x, sf, res["dispersion"], res["betaMatrix"], contrast,
                               weights=wd[_T(idx, dev)].contiguous())
    lse = gc["lfcSE"].cpu().numpy()
    lam = np.full(2, 1e-6 / LN2 ** 2)
    for i in range(len(idx)):
        b = bm[i] * LN2
        g = Gene(y[idx[i]], x, sf, wn[i], disp[i], lam)
        ref = g.post(b, contrast)
        bnd = post_bounds(g, b, contrast, ref, dle_extra=3 * EPS * (np.abs(x) @ np.abs(b)))
        vb = bnd["var"]
        for k in range(2):
            want = math.sqrt(ref["var"][k]) / LN2
            lim = (min(vb[k] / (2 * ref["var"][k] ** 0.5), vb[k] ** 0.5) / LN2 + 3 * EPS * want)
            assert abs(se[i, k] - want) <= lim, (i, k, se[i, k], want, lim)
        want = ref["cd"] / LN2
        lim = bnd["cd"] / LN2 + 3 * EPS * want
        assert abs(lse[i] - want) <= lim, (i, lse[i], want, lim)


# ---------------------------------------------------------------- C2 size on the H100

@pytest.mark.gpu
def test_irls_chain_at_c2_size(engine):
    """50 000 genes x 100 samples, every gene fitted in one call (the persistent grid's scheduling over many CTAs),
    the chain of a seeded sample of 64 genes checked against the 40-digit restatement."""
    import torch
    from deseq2_b200 import device as D, device_pipeline as DP
    be = (D, DP, torch.device("cuda"), torch.cuda.get_device_properties(0).multi_processor_count)
    m, n = 100, 50000
    rng = np.random.default_rng(50000)
    x = x_batch_condition(m)
    p = x.shape[1]
    sf = np.exp(rng.normal(0.0, 0.25, m))
    sf /= np.exp(np.mean(np.log(sf)))
    b_true = np.c_[rng.uniform(0.0, 9.0, n), rng.normal(0.0, 0.7, (n, p - 1))]
    alphas = np.exp(rng.uniform(np.log(1e-3), np.log(5.0), n))
    mu = sf[None, :] * np.exp(b_true @ x.T)
    r = 1.0 / alphas[:, None]
    y = rng.negative_binomial(r, r / (r + mu)).astype(np.float64)
    y[y.sum(axis=1) == 0, 0] = 1
    Q, R = np.linalg.qr(x)
    start = np.linalg.solve(R, Q.T @ np.log(y / sf + 0.1).T).T
    lam = np.full(p, RIDGE)
    contrast = np.r_[0.0, 1.0, -1.0, 0.0]
    nf = np.broadcast_to(sf, (n, m))
    run = _Run(be, x, y, nf, None, alphas, lam, contrast, start, "i4", True)
    full = run(MAXIT)
    sample = sorted(np.random.default_rng(64).choice(n, 64, replace=False).tolist())
    genes = [None] * n
    for g in sample:
        genes[g] = Gene(y[g], x, sf, None, alphas[g], lam)
    knife = check_chain("c2", "small-p 16 lanes (C2)", run, genes, contrast, full, sample=sample)
    _report("c2", knife)


# ---------------------------------------------------------------- rlog_fit_kernel: the arrow-matrix IRLS of rlog()
# rlogData's fit (R/rlog.R:249-253) of the design X = [1 | I_m] with Lambda = diag(lambda0, lambda, ..., lambda), or
# X = I_m on nf' = nf 2^intercept with a frozen intercept.  X'WX + Lambda is an arrow matrix and its solution is exactly
#   beta0 = sum_j c_j z_j / (lambda0 + sum_j c_j),  c_j = w_j lambda / (w_j + lambda),  beta_j = w_j (z_j - beta0) / (w_j + lambda)
# (eliminate beta_j from row j and substitute into row 0; w - w^2 / (w + lambda) = c), so the restatement evaluates that
# at 40 digits.  A step depends on the coefficients only through eta_j = beta0 + beta_j (the mean of sample j).
# The kernel returns only the log2 scale, fl(beta0 / ln2) and fl(fl(beta0 / ln2) + fl(beta_j / ln2)) (or
# fl(fl(beta_j / ln2) + intercept)), so eta_{k-1} is recovered from run k - 1's outputs, and the effect of the recovery
# error on the step is added to the bound through a 40-digit forward-difference Jacobian of the step in eta.

RLOG_TOL = 1e-4                # rlog's betaTol
LAMBDA0 = 1e-6 / LN2 ** 2      # capi.cu::b200nb_rlog_fit_dev: the intercept's ridge, natural-log scale


def rlog_lanes(m):
    """rlog.cuh::rlog_group_lanes."""
    return 8 if m <= 40 else (16 if m <= 160 else 32)


class RlogGene:
    """One row of rlog's fit: counts y, exact factors nfp (nf', mpf), dispersion alpha, sample ridge lam and intercept
    ridge lam0 (natural-log scale; lam0 None when the intercept is frozen)."""

    def __init__(self, y, nfp, alpha, lam, lam0, minmu=MINMU):
        self.y, self.m = np.asarray(y, dtype=np.float64), len(y)
        self.nfp = nfp
        self.alpha, self.lam, self.lam0, self.minmu = float(alpha), float(lam), lam0, float(minmu)

    def _work(self, j, e):
        """mu, w, z, c of sample j at eta_j = e (40 digits)."""
        a, lam = _mp(self.alpha), _mp(self.lam)
        raw = self.nfp[j] * mpmath.exp(e)
        mu = max(raw, _mp(self.minmu))
        lmn = mpmath.log(mu / self.nfp[j]) if raw < mu else e
        w = mu / (1 + a * mu)
        z = lmn + (_mp(self.y[j]) - mu) / mu
        return mu, w, z, w * lam / (w + lam)

    def step(self, eta):
        """(beta0', [beta_j']) of one step from eta, with the pieces the bounds use."""
        with mpmath.workdps(DPS):
            lam = _mp(self.lam)
            ws = [self._work(j, eta[j]) for j in range(self.m)]
            if self.lam0 is None:
                b0, S1, S2 = mpmath.mpf(0), None, None
            else:
                S1 = mpmath.fsum(c * z for _, _, z, c in ws)
                S2 = mpmath.fsum(c for _, _, _, c in ws)
                b0 = S1 / (_mp(self.lam0) + S2)
            bj = [w * (z - b0) / (w + lam) for _, w, z, _ in ws]
            return dict(b0=b0, bj=bj, ws=ws, S1=S1, S2=S2)

    def jacobian(self, eta, st):
        """40-digit forward differences of the step in each eta_i: d beta0 / d eta_i and the total d beta_i / d eta_i
        (sample i moves the intercept, and through it every beta_j by -w_j / (w_j + lambda) d beta0)."""
        with mpmath.workdps(DPS):
            lam = _mp(self.lam)
            d0, dd = [], []
            for i in range(self.m):
                h = mpmath.mpf("1e-22") * (1 + abs(eta[i]))
                mu, w, z, c = self._work(i, eta[i] + h)
                if self.lam0 is None:
                    b0 = mpmath.mpf(0)
                else:
                    _, _, z0, c0 = st["ws"][i]
                    b0 = (st["S1"] - c0 * z0 + c * z) / (_mp(self.lam0) + st["S2"] - c0 + c)
                d0.append(float((b0 - st["b0"]) / h))
                dd.append(float((w * (z - b0) / (w + lam) - st["bj"][i]) / h))
            return np.array(d0), np.array(dd)

    def dev(self, eta):
        with mpmath.workdps(DPS):
            return -2 * mpmath.fsum(ref_logdens(self.y[j], max(self.nfp[j] * mpmath.exp(eta[j]), _mp(self.minmu)),
                                                self.alpha) for j in range(self.m))


def rlog_step_bound(g, eta, st, e_eta, nfp_err):
    """Bounds of the kernel's beta0' and beta_j' for a step from eta (its own eta within e_eta of the given one).
    Arithmetic, per sample: the kernel's eta = beta0 + beta_j rounds once (eps |eta|); mu = nf' exp(eta) carries
    dmu = eps |eta| + 2 eps + nfp_err (exp within 1 ulp, the product; nfp_err = 2 eps for nf 2^intercept); w = mu
    rcp(fma(alpha, mu, 1)) adds 3 roundings, c = w lam rcp(w + lam) 5 more; z = lmn + fma(y, rcp(mu), -1) carries
    eps |eta| (or 3 eps (|log(minmu / nf')| + 1) + nfp_err on the clamp path) + y / mu (dmu + 2 eps) + eps |z|; the two
    m-term sums (m + 2) eps of the magnitudes of their terms; beta0' = S1 rcp(lambda0 + S2) 4 roundings and beta_j' =
    w (z - beta0') rcp(w + lambda) 5, plus w / (w + lambda) times the error of beta0'.  Recovery: first order through
    the forward-difference Jacobian, |d beta0| <= sum_i |d beta0 / d eta_i| e_i and |d beta_j| <= |d beta_j / d eta_j|
    e_j + w_j / (w_j + lambda) sum_i |d beta0 / d eta_i| e_i."""
    m = g.m
    lam = g.lam
    etaf = np.array([float(v) for v in eta])
    mu = np.array([float(v[0]) for v in st["ws"]])
    w = np.array([float(v[1]) for v in st["ws"]])
    z = np.array([float(v[2]) for v in st["ws"]])
    c = np.array([float(v[3]) for v in st["ws"]])
    nfp = np.array([float(v) for v in g.nfp])
    clamped = mu <= g.minmu
    dmu = EPS * np.abs(etaf) + 2 * EPS + nfp_err
    dw = dmu + 3 * EPS
    dc = dw + 5 * EPS
    dz = (np.where(clamped, 3 * EPS * (np.abs(np.log(g.minmu / nfp)) + 1) + nfp_err, EPS * np.abs(etaf))
          + g.y / mu * (dmu + 2 * EPS) + EPS * np.abs(z))
    cs = (m + 2) * EPS
    b0 = float(st["b0"])
    bj = np.array([float(v) for v in st["bj"]])
    if g.lam0 is None:
        e_b0 = 0.0
    else:
        S2 = float(st["S2"])
        e_S1 = float(np.sum(np.abs(c * z) * (dc + cs) + c * dz))
        e_S2 = float(np.sum(c * (dc + cs)))
        e_b0 = (e_S1 + abs(b0) * e_S2) / (g.lam0 + S2) + 4 * EPS * abs(b0)
    f = w / (w + lam)
    e_bj = np.abs(bj) * (dw + 5 * EPS) + f * (dz + e_b0 + EPS * np.abs(z - b0))
    d0, dd = g.jacobian(eta, st)
    E0 = float(np.sum(np.abs(d0) * e_eta))
    return e_b0 + E0, e_bj + np.abs(dd) * e_eta + f * E0


def _rlog_eta(out, icpt, frozen):
    """eta of the kernel's coefficients, recovered from its log2 outputs, and the recovery error: out_j = fl(fl(beta0 /
    L) + fl(beta_j / L)), L = fl(ln 2), so out_j ln 2 is within eps (2 |beta0| + 2 |beta_j| + |eta|) of beta0 + beta_j
    (three roundings and that of L); frozen, out_j = fl(fl(beta_j / L) + intercept) and eta_j = beta_j."""
    base = np.zeros_like(out) if frozen else np.full_like(out, icpt)
    with mpmath.workdps(DPS):
        l2 = mpmath.log(2)
        eta = [(_mp(o) - (_mp(icpt) if frozen else 0)) * l2 for o in out]
    e = 1.01 * LN2 * EPS * (2 * np.abs(base) + 3 * np.abs(out - (icpt if frozen else base)) + np.abs(out))
    return eta, e


RLOG_CASES = [
    # (name, m, nf "sf" | "matrix", frozen intercept, counts dtype, betaPriorVar)
    ("rlog-l8-sf", 10, "sf", False, "i4", 1.0),
    ("rlog-l8-nf-frozen", 24, "matrix", True, "f8", 0.05),
    ("rlog-l16-nf", 60, "matrix", False, "i4", 0.05),
    ("rlog-l16-sf-frozen", 100, "sf", True, "i4", 1.0),
    ("rlog-l32-sf", 170, "sf", False, "f8", 0.5),
    ("rlog-l32-nf-frozen", 200, "matrix", True, "i4", 2.0),
]


@pytest.mark.parametrize("case", RLOG_CASES, ids=[c[0] for c in RLOG_CASES])
def test_rlog_chain_against_40_digits(backend, case):
    """rlog_fit_kernel, one iteration at a time: run k (maxit = k) against one 40-digit step from the eta recovered
    from run k - 1 (from the start for k = 1), every output on the log2 scale; iter = k until the stop, whose decision
    is checked against the 40-digit deviances (within their error bounds, which add the recovery error through
    d dev / d eta_j = -2 (y - mu) / (1 + alpha mu)); the run that stops reproduces the maxit = 100 run bit for bit.
    Rows: ordinary, a row with most counts 0 (means at minmu: the clamp path of rl_working), counts ~1e5, and for a
    fitted intercept an all-zero row (R leaves it out: 0, intercept -Inf, iter 0)."""
    from deseq2_b200 import device as D
    name, m, nfk, frozen, dt, bpv = case
    _, DP, dev, _ = backend
    rng = np.random.default_rng(sum(map(ord, name)))
    alphas = np.array([1.0, 0.1, 1e-8, 10.0, 0.5])      # 1e-8 on the 1e5 row: w / lambda ~ 1e5
    n = len(alphas)
    sf = np.exp(rng.normal(0.0, 0.3, m))
    sf /= np.exp(np.mean(np.log(sf)))
    nf = np.broadcast_to(sf, (n, m)).copy()
    if nfk == "matrix":
        nf *= np.exp(rng.normal(0.0, 0.2, (n, m)))
    y = np.array([_nb(rng, nf[g] * np.exp(rng.uniform(1.0, 6.0) + rng.normal(0.0, 0.8, m)), min(alphas[g], 1.0))
                  for g in range(n)])
    y[1, : max(2, m - 3)] = 0                                   # the clamp path
    y[2] = np.round(1e5 * nf[2] * rng.uniform(0.5, 2.0, m))
    if not frozen:
        y[4] = 0                                                # all zero: not fitted
    if dt == "f8":
        y = y + np.where(y > 0, rng.uniform(0.0, 1.0, (n, m)).round(3), 0.0)
    icpt = rng.uniform(1.0, 5.0, n)
    yd = D.to_gene_major(y.astype(np.int32) if dt == "i4" else y, dev)
    sfd = _T(sf, dev) if nfk == "sf" else D.to_gene_major(nf, dev)
    icd = _T(icpt, dev) if frozen else None

    def run(maxit):
        r = DP.rlog_fit(yd, m, sfd, _T(alphas, dev), bpv, intercept=icd, betaTol=RLOG_TOL, maxit=maxit)
        return (r["rlog"].cpu().numpy(), None if frozen else r["intercept"].cpu().numpy(), r["betaIter"].cpu().numpy())

    full = run(MAXIT)
    lam = (1.0 / bpv) / LN2 ** 2
    fam = f"rlog {rlog_lanes(m)} lanes {'frozen' if frozen else 'fitted'}"
    nfp_err = 2 * EPS if frozen else 0.0
    knife = 0
    for g in range(n):
        gt = f"{name} gene {g} (alpha {alphas[g]:g})"
        if not frozen and g == 4:
            assert np.all(full[0][g] == 0) and full[1][g] == -np.inf and full[2][g] == 0, gt
            continue
        it = int(full[2][g])
        assert 1 <= it <= MAXIT, (gt, it)
        with mpmath.workdps(DPS):
            nfp = [_mp(v) * (mpmath.mpf(2) ** _mp(icpt[g]) if frozen else 1) for v in nf[g]]
            if frozen:
                eta = [mpmath.log(_mp(y[g, j]) / nfp[j] + mpmath.mpf("0.1")) for j in range(m)]
            else:
                eta = [mpmath.log(mpmath.fsum(_mp(y[g, j]) / nfp[j] for j in range(m)) / m)] * m
        eta_f = np.array([float(v) for v in eta])
        e_eta = (4 * EPS + 2 * EPS * np.abs(eta_f) + nfp_err) if frozen else ((m + 5) * EPS + 2 * EPS * np.abs(eta_f))
        gene = RlogGene(y[g], nfp, alphas[g], lam, None if frozen else LAMBDA0)
        dev_prev, edev_prev = None, None
        for k in range(1, MAXIT + 1):
            out, ic, itk = run(k)
            o, t = out[g], int(itk[g])
            assert t == k, (gt, k, t)
            st = gene.step(eta)
            e_b0, e_bj = rlog_step_bound(gene, eta, st, e_eta, nfp_err)
            b0s, bjs = float(st["b0"]), np.array([float(v) for v in st["bj"]])
            with mpmath.workdps(DPS):
                l2 = mpmath.log(2)
                if frozen:
                    want = np.array([float(v / l2 + _mp(icpt[g])) for v in st["bj"]])
                    lim = e_bj / LN2 + 2 * EPS * np.abs(bjs) / LN2 + EPS * np.abs(want)
                else:
                    want = np.array([float((st["b0"] + v) / l2) for v in st["bj"]])
                    lim = (e_b0 + e_bj) / LN2 + 3 * EPS * (abs(b0s) + np.abs(bjs)) / LN2 + EPS * np.abs(want)
                    wi = float(st["b0"] / l2)
                    li = e_b0 / LN2 + 2 * EPS * abs(wi)
                    assert _ratio(fam, "intercept", abs(ic[g] - wi), li) <= 1.0, (gt, k, ic[g], wi, li)
            assert _ratio(fam, "rlog", np.abs(o - want), lim) <= 1.0, (gt, k, np.max(np.abs(o - want) / lim))
            eta, e_eta = _rlog_eta(o, icpt[g] if frozen else ic[g], frozen)
            # |beta| > 30 (intercept included): iter = maxit, the diverged coefficients kept (they are run k's)
            bnat = (o - (icpt[g] if frozen else ic[g])) * LN2
            diverged = np.any(np.abs(bnat) > LARGE) or (not frozen and abs(ic[g] * LN2) > LARGE)
            if diverged:
                assert it == MAXIT, (gt, k, "diverged, but the full run reports", it)
                assert _same(out[g], full[0][g]) and (frozen or _same(ic[g], full[1][g])), (gt, "differs from maxit 100")
                break
            if k == MAXIT:                                      # 100 steps without converging: R's iter = maxit
                assert it == MAXIT and _same(out[g], full[0][g]), gt
                break
            # the stop decision at k from the 40-digit deviances at the recovered eta_{k-1} and eta_k
            eta_f = np.array([float(v) for v in eta])
            d1 = gene.dev(eta)
            mu = np.maximum(np.array([float(v) for v in gene.nfp]) * np.exp(eta_f), MINMU)
            sens = 2 * np.abs(y[g] - mu) / (1 + alphas[g] * mu) * (mu > MINMU)
            scale = sum(_loglik_scale(y[g, j], mu[j], alphas[g], 1.0, abs(eta_f[j]), 0.0) for j in range(m))
            edev = 2 * (m + 16) * EPS * scale + float(sens @ e_eta)
            if k >= 2:
                with mpmath.workdps(DPS):
                    conv = float(abs(d1 - dev_prev) / (abs(d1) + mpmath.mpf("0.1")))
                econv = (edev + edev_prev) / (abs(float(d1)) + 0.1) * (1 + conv) * 1.01
                if abs(conv - RLOG_TOL) <= econv:
                    knife += 1
                else:
                    assert (k == it and it < MAXIT) == (conv < RLOG_TOL), (gt, k, conv)
            else:
                assert it != 1, f"{gt}: stopped at the first iteration"
            dev_prev, edev_prev = d1, edev
            if k == it and it < MAXIT:
                assert _same(out[g], full[0][g]) and (frozen or _same(ic[g], full[1][g])), (gt, "differs from maxit 100")
                break
    _report(name, knife)
