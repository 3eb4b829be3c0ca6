"""beta_optim_kernel and nb_loglik_kernel against a 40-digit maximiser and a 40-digit likelihood.

Two kernels finish a DESeq() fit: beta_optim_kernel (fit_optim.cu, fitNbinomGLMsOptim, R/fitNbinomGLMs.R:340-407)
refits whatever the IRLS could not fit, and nb_loglik_kernel (fit_beta.cu, nbinomLogLike at the unclamped mean)
gives every log-likelihood the LRT, the deviance, Cook's distances and the refitted rows use.  Both are checked here
against plain high-precision references of the same operation, not against another optimiser:

  * The objective of the optim fallback is strictly concave and its box-constrained maximiser is unique, so any method
    that reaches that maximiser is a complete reference.  ref_maximise runs a float64 projected Newton with an active
    set, then polishes the free coordinates with Newton steps at 40 digits (mpmath) and certifies the result by the
    KKT conditions at 40 digits: free gradient below 1e-25 relative, gradient strictly outward at each bound
    coordinate.  The device result is then held to its own stop rule (the 40-digit projected gradient at the device's
    coefficients), to the objective gap that rule implies, to the exact bound on active coordinates, and to the
    fitted means the rule determines.
  * device_pipeline._optim_fallback is checked against R's post-optim formulas (:378-403) at 40 digits, evaluated at
    the device's coefficients.
  * nb_loglik is checked against dnbinom(log = TRUE) by loggamma at 40 digits on a grid of (y, mu, alpha) that crosses
    every switch of the kernel: exp_fast / exp at |le| = 700, subnormal and zero means, the 256-entry log-factorial
    table and its integer test, and lgamma_diff's r >= kShift branch on both sides of r = 10.

Each case runs on the SIMT-emulated engine on every CPU run (backend "emu": the product's CUDA sources compiled by g++,
tests/simt_emu/) and again on the H100 under -m gpu (backend "gpu").  CPU run time of the emulated half: about
30 seconds on one core, once the emulated engine is built (measured with `pytest tests/test_optim_loglik_reference.py -m "not gpu"`)."""
import ctypes as C
import math

import mpmath
import numpy as np
import pytest

from helpers import chol_backward, sandwich_bound
from test_sample_counts import _emu_lib

EPS = 2.0 ** -52
LN2 = math.log(2.0)
U = 30.0 * LN2               # capi.cu::b200nb_beta_optim_dev, a.bound: the box on the natural-log scale, in fp64
MAXIT = 200                  # device.beta_optim's default
MINMU = 0.5
DPS = 40
EMU_SMS = 2                  # tests/simt_emu/cuda_runtime.h::cudaDeviceGetAttribute: the emulator reports 2 SMs


# ---------------------------------------------------------------- backends

@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def backend(request):
    """(device module, device_pipeline module, torch device, SM count the engine sees).  The emulated engine is bound
    for the one test only, so that the gpu cases of a full run never see it."""
    import torch
    from deseq2_b200 import _lib, device as D, device_pipeline as DP
    if request.param == "gpu":
        request.getfixturevalue("engine")
        dev = torch.device("cuda")
        yield D, DP, dev, torch.cuda.get_device_properties(dev).multi_processor_count
        return
    lib = _emu_lib()
    saved, saved_stream, saved_dp = _lib._lib, D._stream, DP._stream
    _lib._lib, D._stream = lib, (lambda: C.c_void_p(0))
    DP._stream = D._stream
    try:
        yield D, DP, torch.device("cpu"), EMU_SMS
    finally:
        _lib._lib, D._stream, DP._stream = saved, saved_stream, saved_dp


def _T(a, dev):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device=dev)


# ---------------------------------------------------------------- the 40-digit reference

def _mp(v):
    return mpmath.mpf(float(v))


def ref_logdens(y, mu, alpha):
    """R's dnbinom(y, mu = mu, size = 1/alpha, log = TRUE) by loggamma at the working precision (the caller sets 40
    digits).  y, mu, alpha are taken as the exact values of their float64 arguments.  mu = 0 is the point mass at 0."""
    y, mu, a = _mp(y), (mu if isinstance(mu, mpmath.mpf) else _mp(mu)), _mp(alpha)
    if mu == 0:
        return mpmath.mpf(0) if y == 0 else mpmath.mpf("-inf")
    r = 1 / a
    return (mpmath.loggamma(y + r) - mpmath.loggamma(r) - mpmath.loggamma(y + 1) + r * mpmath.log(r / (r + mu))
            + (y * mpmath.log(mu / (r + mu)) if y != 0 else 0))


class Row:
    """One row of fitNbinomGLMsOptim: counts y (m), design x (m, p), normalization factors nf (m), weights w (m or
    None), dispersion alpha, ridge lam (p, natural-log scale).  The objective (R/fitNbinomGLMs.R:359-370) is taken in
    the natural-log coefficients the kernel uses, beta = ln 2 * p: nf * 2^(x p) = nf * e^(x beta) and
    dnorm(p, 0, sqrt(1/lambda), log = TRUE) = -1/2 (lambda / ln(2)^2) beta^2 + const, lam = lambda / ln(2)^2."""

    def __init__(self, y, x, nf, w, alpha, lam):
        self.y = np.asarray(y, dtype=np.float64)
        self.x = np.asarray(x, dtype=np.float64)
        self.nf = np.asarray(nf, dtype=np.float64)
        self.w = None if w is None else np.asarray(w, dtype=np.float64)
        self.alpha = float(alpha)
        self.lam = np.asarray(lam, dtype=np.float64)
        self.m, self.p = self.x.shape
        self._mpdata = None

    def mpdata(self):
        if self._mpdata is None:
            with mpmath.workdps(DPS):
                a = _mp(self.alpha)
                r = 1 / a
                ys = [_mp(v) for v in self.y]
                const = [mpmath.loggamma(y + r) - mpmath.loggamma(r) - mpmath.loggamma(y + 1) + r * mpmath.log(r)
                         for y in ys]
                self._mpdata = dict(a=a, r=r, y=ys, const=const, x=[[_mp(v) for v in row] for row in self.x],
                                    lnf=[mpmath.log(_mp(v)) for v in self.nf],
                                    w=[mpmath.mpf(1)] * self.m if self.w is None else [_mp(v) for v in self.w],
                                    lam=[_mp(v) for v in self.lam], lnr=mpmath.log(r))
        return self._mpdata

    # -- 40 digits
    def mp_eval(self, b, hessian=True):
        """At 40 digits: R's objective f (with every constant), the kernel's objective fk (the beta-dependent part
        fit_optim.cu::objective sums), the gradient, the negative Hessian (the closed forms of fit_optim.cu's header),
        and the fitted means."""
        d = self.mpdata()
        with mpmath.workdps(DPS):
            b = [v if isinstance(v, mpmath.mpf) else _mp(v) for v in b]
            a, r, p = d["a"], d["r"], self.p
            f = fk = mpmath.mpf(0)
            g = [mpmath.mpf(0)] * p
            gs = [mpmath.mpf(0)] * p
            Hn = [[mpmath.mpf(0)] * p for _ in range(p)] if hessian else None
            mus = []
            for j in range(self.m):
                xj = d["x"][j]
                le = mpmath.fsum(xj[k] * b[k] for k in range(p)) + d["lnf"][j]
                mu = mpmath.exp(le)
                mus.append(mu)
                y, w = d["y"][j], d["w"][j]
                l1p = mpmath.log1p(a * mu)
                fk += w * (y * le - (y + r) * l1p)
                # log dnbinom = const + y log mu - (y + r) log(r + mu), log(r + mu) = log r + log1p(alpha mu)
                f += w * (d["const"][j] + y * le - (y + r) * (d["lnr"] + l1p))
                u = 1 + a * mu
                g1 = w * (y - mu) / u
                h1 = w * mu * (1 + a * y) / (u * u)
                for k in range(p):
                    if xj[k]:
                        g[k] += xj[k] * g1
                        gs[k] += abs(xj[k]) * (abs(g1) + h1)
                if hessian:
                    for k in range(p):
                        if xj[k]:
                            t = xj[k] * h1
                            for q in range(k + 1):
                                if xj[q]:
                                    Hn[k][q] += t * xj[q]
            lam = d["lam"]
            for k in range(p):
                pen = lam[k] * b[k] * b[k] / 2
                f += -pen + (mpmath.log(lam[k] * mpmath.log(2) ** 2 / (2 * mpmath.pi)) / 2 if lam[k] > 0 else 0)
                fk -= pen
                g[k] -= lam[k] * b[k]
                gs[k] += 1 + lam[k] * abs(b[k])
                if hessian:
                    Hn[k][k] += lam[k]
                    for q in range(k):
                        Hn[q][k] = Hn[k][q]
            return dict(f=f, fk=fk, g=g, gs=gs, Hn=Hn, mu=mus)

    # -- float64, for the start of the reference and for the long rows
    def f64_eval(self, b):
        le = self.x @ b + np.log(self.nf)
        mu = np.exp(le)
        w = np.ones(self.m) if self.w is None else self.w
        a, r, y = self.alpha, 1.0 / self.alpha, self.y
        with np.errstate(over="ignore", invalid="ignore"):
            t = w * (y * le - (y + r) * np.log1p(a * mu))
            u = 1.0 + a * mu
            big = np.isinf(mu)                               # the limit mu -> inf, as fit_optim.cu takes it
            gt = (w * np.where(big, -r, (y - mu) / u))[:, None] * self.x
            h1 = w * np.where(big, 0.0, mu * (1.0 + a * y) / (u * u))
        f = math.fsum(t) - 0.5 * math.fsum(self.lam * b * b)
        g = np.array([math.fsum(gt[:, k]) for k in range(self.p)]) - self.lam * b
        Hn = self.x.T @ (h1[:, None] * self.x) + np.diag(self.lam)
        return dict(f=f, g=g, Hn=Hn, mu=mu, t=t, gt=gt, le=le)


def _active(b, g):
    """fit_optim.cu's active set: a coordinate on a bound whose gradient points out of the box."""
    return [(float(b[k]) >= U and g[k] > 0) or (float(b[k]) <= -U and g[k] < 0) for k in range(len(b))]


def _f64_newton(row, start, iters=300):
    """Projected Newton with an active set in float64, from the start the kernel gets (NaN -> 0, clipped)."""
    b = np.clip(np.nan_to_num(np.asarray(start, dtype=np.float64), nan=0.0), -U, U)
    if not np.isfinite(row.f64_eval(b)["f"]):
        b = np.zeros(row.p)                                   # a start whose means overflow: any start will do
    for _ in range(iters):
        e = row.f64_eval(b)
        fr = ~np.array(_active(b, e["g"]))
        if not fr.any():
            break
        step = np.zeros(row.p)
        step[fr] = np.linalg.solve(e["Hn"][np.ix_(fr, fr)], e["g"][fr])
        t, moved = 1.0, False
        for _ in range(80):
            trial = np.clip(b + t * step, -U, U)
            ft = row.f64_eval(trial)["f"]
            if ft > e["f"]:
                moved = True
                break
            t *= 0.5
        if not moved:
            break
        b = trial
    return b


def ref_maximise(row, start):
    """The box-constrained maximiser of the row's objective, certified at 40 digits.  Returns beta* (mpf list), f*
    (R's objective), fk* (the kernel's), the negative Hessian H* (float64), the active set and the 40-digit means."""
    b = _f64_newton(row, start)
    with mpmath.workdps(DPS):
        bm = [_mp(v) for v in b]
        for k in range(row.p):                       # the float64 stage may stop a rounding short of a bound
            if abs(bm[k]) >= U * (1 - 1e-14):
                bm[k] = _mp(math.copysign(U, b[k]))
        for _ in range(12):
            e = row.mp_eval(bm)
            act = _active(bm, e["g"])
            fr = [k for k in range(row.p) if not act[k]]
            gf = [e["g"][k] for k in fr]
            if max((abs(v) for v in gf), default=0) <= mpmath.mpf("1e-32") * (1 + abs(e["f"])):
                break
            H = mpmath.matrix([[e["Hn"][i][k] for k in fr] for i in fr])
            step = mpmath.lu_solve(H, mpmath.matrix(gf))
            for i, k in enumerate(fr):
                bm[k] = min(max(bm[k] + step[i], _mp(-U)), _mp(U))
        e = row.mp_eval(bm)
        act = _active(bm, e["g"])
        fr = [k for k in range(row.p) if not act[k]]
        # the KKT certificate at 40 digits: stationary in the free coordinates, strictly outward at the bounds
        gfree = max((abs(e["g"][k]) for k in fr), default=mpmath.mpf(0))
        assert gfree <= mpmath.mpf("1e-25") * (1 + abs(e["f"])), f"reference not certified: |g_free| = {gfree}"
        assert all(abs(bm[k]) < U for k in fr)
        assert all(abs(bm[k]) == U and e["g"][k] * bm[k] > 0 for k in range(row.p) if act[k])
        Hn = np.array([[float(v) for v in rw] for rw in e["Hn"]])
        return dict(beta=bm, f=e["f"], fk=e["fk"], Hn=Hn, active=act, free=fr, mu=e["mu"])


# ---------------------------------------------------------------- designs

def x_condition(m):
    return np.c_[np.ones(m), np.r_[np.zeros((m + 1) // 2), np.ones(m // 2)]]


def x_batch_condition(m):
    from deseq2_b200 import synth
    return synth.design_batch_condition(m, 3)                # p = 4


def x_factor10(m):
    from deseq2_b200 import synth
    return synth.design_factor(m, 10)                        # p = 10


def x_covariate(m):
    """test_optim.R: ~condition with condition <- rnorm(ncol(dds), 0, 1000), a large predictor to test scaling."""
    return np.c_[np.ones(m), np.random.default_rng(1).normal(0.0, 1000.0, m)]


def x_expanded10(m):
    from deseq2_b200 import synth
    return synth.design_factor_expanded(m, 10)               # p = 11, rank 10: only the ridge makes it identifiable


def x_p32(m):
    return np.c_[np.ones(m), np.random.default_rng(32).normal(0.0, 0.3, (m, 31))]    # p = kMaxP


DESIGNS = {"cond": x_condition, "batch": x_batch_condition, "f10": x_factor10, "cov": x_covariate,
           "exp10": x_expanded10, "p32": x_p32}


# ---------------------------------------------------------------- the beta_optim cases
# (name, design, m, nf, weights, counts dtype, ridge, rows).  nf: "sf" (size-factor vector) or "matrix"; ridge: the
# natural-log lambda (a number for every coefficient, "prior" for an estimate_beta_prior_var call); rows: the kinds of
# rows of the one call (see _row).  Every case cycles alpha over ALPHAS(m).

RIDGE = 1e-6 / LN2 ** 2           # DESeq()'s betaPrior = FALSE ridge
TEST_OPTIM_RIDGE = 2.0 / LN2 ** 2  # test_optim.R's lambda = c(2, 2)
ORDINARY = ("ordinary", "far", "nan", "outside")


def ALPHAS(m):
    return (1e-8, 0.1, float(max(10, m)))


OPTIM_CASES = [
    ("cond-m10-R", "cond", 10, "sf", False, "i4", RIDGE, ("R", "R3000", "R-one", "R-swap") + ORDINARY),
    ("cond-m6-bounds", "cond", 6, "matrix", False, "f8", 1e-10, ("lower", "lower", "upper", "upper") + ORDINARY),
    ("cond-m40-w", "cond", 40, "sf", True, "i4", RIDGE, ("zero-cell", "zero-cell", "lower-w") + ORDINARY),
    ("batch-p4-nf", "batch", 24, "matrix", False, "f8", RIDGE, ("zero-cell", "upper") + ORDINARY),
    ("f10-w", "f10", 60, "sf", True, "f8", RIDGE, ("zero-cell", "zero-cell") + ORDINARY),
    ("cov-sd1000", "cov", 20, "sf", False, "i4", TEST_OPTIM_RIDGE, ORDINARY + ORDINARY),
    ("exp10-prior", "exp10", 40, "sf", False, "i4", "prior", ("zero-cell", "zero-cell") + ORDINARY),
    ("p32", "p32", 64, "matrix", True, "f8", RIDGE, ("upper",) + ORDINARY),
]


def _nb(rng, mu, alpha):
    r = 1.0 / alpha
    return rng.negative_binomial(r, r / (r + mu)).astype(np.float64)


def _row(kind, x, nf, alpha, rng, dt):
    """(counts, start) of one row kind.  Starts are natural-log coefficients."""
    m, p = x.shape
    b_true = np.r_[rng.uniform(3.0, 6.0), rng.normal(0.0, 0.7, p - 1)]
    if x[:, 1:].std() > 100:                                  # the sd-1000 covariate: fold changes per unit are tiny
        b_true[1:] /= 1000.0
    mu = nf * np.exp(x @ b_true)
    y = _nb(rng, mu, min(alpha, 1.0))
    start = b_true + rng.normal(0.0, 0.3, p)
    last = x[:, -1] != 0
    if kind.startswith("R"):
        # test_optim.R's row and variations of it: a design cell of zeros, flat except for the ridge
        y = np.array([0, 0, 0, 0, 0, 1000, 1000, 0, 0, 0], dtype=np.float64)
        if kind == "R3000":
            y[5] = 3000
        elif kind == "R-one":
            y[9] = 1
        elif kind == "R-swap":
            y = y[::-1].copy()
        start = np.array([0.0, 25.0])                         # what the IRLS leaves: diverging, outside the box
    elif kind in ("zero-cell", "lower"):
        y[last] = 0.0                                         # the last design column's cell has no counts
        start = np.zeros(p)
    elif kind == "lower-w":
        y[last] = 0.0
        start = np.r_[b_true[0], -U * np.ones(p - 1)]
    elif kind == "upper":
        # f64 counts ~1e12 against nf ~1e-2: the unconstrained intercept would be ~ log(1e14) > 30 ln 2
        y = np.round(1e12 * np.exp(x @ np.r_[0.0, rng.normal(0.0, 0.5, p - 1)]) * rng.uniform(0.9, 1.1, m))
        start = np.r_[U, np.zeros(p - 1)]
    elif kind == "far":
        start = rng.normal(0.0, 5.0, p)
    elif kind == "nan":
        start = np.full(p, np.nan)
    elif kind == "outside":
        start = np.r_[40.0, -35.0 * np.ones(p - 1)]
        if x[:, 1:].std() > 100:
            # with x ~ 1000 the clipped corner overflows every mean and no step halving reaches a finite objective
            # (DESIGN.md section 10): outside the box in the intercept only
            start[1:] = 0.0
    if dt == "f8" and kind not in ("upper",):
        y = y + np.where(y > 0, rng.uniform(0.0, 1.0, m).round(3), 0.0)    # non-integer counts
    return y, start


def _optim_inputs(case, backend):
    name, design, m, nfk, wk, dt, ridge, kinds = case
    D, DP, dev, _ = backend
    rng = np.random.default_rng(sum(map(ord, name)))
    x = DESIGNS[design](m)
    p = x.shape[1]
    sf = np.exp(rng.normal(0.0, 0.25, m))
    sf /= np.exp(np.mean(np.log(sf)))
    n = len(kinds)
    nf = np.broadcast_to(sf, (n, m)).copy()
    if nfk == "matrix":
        nf *= np.exp(rng.normal(0.0, 0.2, (n, m)))
        for g, k in enumerate(kinds):
            if k == "upper":
                nf[g] *= 1e-2
    alphas = np.array([ALPHAS(m)[g % 3] for g in range(n)])
    ys, starts = zip(*(_row(k, x, nf[g], alphas[g], rng, dt) for g, k in enumerate(kinds)))
    y, start = np.array(ys), np.array(starts)
    if dt == "i4":
        assert np.all(y == np.round(y)) and y.max() < 2 ** 31
    w = None
    if wk:
        w = rng.uniform(0.2, 1.0, (n, m))
        w[:, 0] = 0.0                                         # exact zeros
        w[:, 1] = 1e-4
    if ridge == "prior":
        lam = _prior_lambda(D, DP, dev, m)
    else:
        lam = np.full(p, float(ridge))
    return x, y, nf, w, alphas, lam, start


def _prior_lambda(D, DP, dev, m):
    """estimate_beta_prior_var (the device's estimateBetaPriorVar) on the standard 10-level matrix, from MLE log2 fold
    changes of 40 genes: the expanded matrix's prior variances, as DESeq(betaPrior = TRUE) passes them to the MAP fit."""
    rng = np.random.default_rng(10)
    levels = (np.arange(m) * 10) // m
    n = 40
    B = np.c_[rng.uniform(3, 8, n), rng.normal(0.0, 1.0, (n, 9))]
    pv = DP.estimate_beta_prior_var(_T(B, dev), [levels], _T(rng.uniform(50, 500, n), dev),
                                    _T(np.full(n, 0.1), dev)).cpu().numpy()
    assert pv.shape == (11,) and np.all(pv > 0) and pv[0] == 1e6
    return 1.0 / (pv * LN2 ** 2)


def _run_optim(D, dev, x, y, nf, w, alphas, lam, start, dt):
    yd = D.to_gene_major(y.astype(np.int32) if dt == "i4" else y, dev)
    nfd = D.to_gene_major(nf, dev) if not np.all(nf == nf[:1]) else _T(nf[0], dev)
    wd = None if w is None else D.to_gene_major(w, dev)
    o = D.beta_optim(yd, x, nfd, _T(alphas, dev), _T(lam, dev), _T(start.T, dev), weights=wd)
    return o["beta_mat"].cpu().numpy().T, o["converged"].cpu().numpy(), o["iter"].cpu().numpy()


def _check_optim_row(tag, row, bdev, conv, it, start):
    """The five per-row assertions against the certified 40-digit maximiser."""
    ref = ref_maximise(row, start)
    assert conv == 1 and it < MAXIT, f"{tag}: converged {conv}, iter {it}"
    assert np.all(np.abs(bdev) <= U), tag                                      # inside the box
    for k in range(row.p):                                                     # an active bound is exactly +-30 ln 2
        if ref["active"][k]:
            assert bdev[k] == math.copysign(U, float(ref["beta"][k])), (tag, k, bdev[k])
    with mpmath.workdps(DPS):
        e = row.mp_eval(list(bdev))
        # (3) the kernel's own stop rule, fit_optim.cu `|grad_k| <= 1e-10 * gscale_k` on every free coordinate, with
        # gscale_k = 1 + sum_j |x_jk| (|g1_j| + h1_j) + lambda_k |beta_k| the size of the gradient's terms, held at 40
        # digits with a factor 4 for the rounding of the kernel's fp64 sums
        tol = np.array([1e-10 * float(v) for v in e["gs"]])
        act = _active(bdev, e["g"])
        pg = max((abs(float(e["g"][k])) / tol[k] for k in range(row.p) if not act[k]), default=0.0)
        assert pg <= 4.0, f"{tag}: projected gradient {pg:.3e} x the stop rule's tolerance (> 4)"
        # (2) objective gap.  The objective is strongly concave with modulus lam_min(H*_free) near beta*, so a point
        # on beta*'s face with free gradient g is at most |g|_2^2 / (2 lam_min) below f*, and |g_k| <= 4 tol_k by (3).
        # Floor: 64 ulp(|f*|), the resolution of the fp64 coefficients themselves (rounding beta* to fp64 alone costs
        # up to h ulp(beta)^2 / 2, far below it).
        fr = ref["free"]
        lmin = np.linalg.eigvalsh(ref["Hn"][np.ix_(fr, fr)])[0] if fr else np.inf
        gap = float(ref["f"] - e["f"])
        bound = max(0.5 * np.sum((4.0 * tol[fr]) ** 2) / lmin, 64.0 * np.spacing(abs(float(ref["f"]))))
        assert gap <= bound, f"{tag}: objective gap {gap:.3e} > {bound:.3e}"
        # (5) the fitted means the stop rule determines.  To second order beta* - beta_dev = H^-1 g (free
        # coordinates, g the 40-digit gradient at beta_dev), so by Cauchy-Schwarz in the H^-1 inner product
        # |x_j (beta* - beta_dev)| <= sqrt(x_j' H^-1 x_j) sqrt(g' H^-1 g); a factor 2 covers the third-order rest
        # while the Newton decrement g' H^-1 g is small (asserted), plus 4 ulp for the fp64 product x beta.
        if fr:
            Hf = ref["Hn"][np.ix_(fr, fr)]
            gf = np.array([float(e["g"][k]) for k in fr])
            dec = float(gf @ np.linalg.solve(Hf, gf))
            assert dec < 1e-6, f"{tag}: Newton decrement {dec:.3e}"
            xf = row.x[:, fr]
            lev = np.einsum("jk,jk->j", xf, np.linalg.solve(Hf, xf.T).T)
            for j in range(row.m):
                mus = ref["mu"][j]
                if mus >= MINMU:
                    rel = abs(float(e["mu"][j] / mus - 1))
                    lim = 2.0 * math.sqrt(max(lev[j], 0.0) * dec) + 4 * EPS * (np.abs(row.x[j]) @ np.abs(bdev) + 1)
                    assert rel <= lim, f"{tag}: mu[{j}] rel err {rel:.3e} > {lim:.3e}"
    return ref


@pytest.mark.parametrize("case", OPTIM_CASES, ids=[c[0] for c in OPTIM_CASES])
def test_beta_optim_reaches_the_maximiser(backend, case):
    D, DP, dev, _ = backend
    name, dt = case[0], case[5]
    x, y, nf, w, alphas, lam, start = _optim_inputs(case, backend)
    beta, conv, it = _run_optim(D, dev, x, y, nf, w, alphas, lam, start, dt)
    kinds = case[7]
    n_active = 0
    for g in range(len(y)):
        row = Row(y[g], x, nf[g], None if w is None else w[g], alphas[g], lam)
        ref = _check_optim_row(f"{name} row {g} ({kinds[g]}, alpha {alphas[g]:g})", row, beta[g], conv[g], it[g],
                               start[g])
        n_active += sum(ref["active"])
        if kinds[g] == "upper":
            assert ref["active"][0] and ref["beta"][0] > 0, f"{name} row {g}: not at the upper bound"
        if kinds[g] == "lower":
            assert ref["active"][-1] and ref["beta"][-1] < 0, f"{name} row {g}: not at the lower bound"
    if any(k in ("upper", "lower") for k in kinds):
        assert n_active > 0


# ---------------------------------------------------------------- long rows: the strided-CTA route

def _optim_smem(m, p):
    """fit_optim.cu::launch_beta_optim's shared-memory size; past 200 KB the two rows of m go to global memory and at
    most 8 CTAs per SM stride over the genes."""
    mpad = (m + 3) & ~3
    return (2 * mpad + 2 * p * p + 5 * p + 2) * 8


def test_beta_optim_long_rows_strided(backend):
    """m = 13 000 (past launch_beta_optim's 200 KB switch) with more rows than 8 CTAs per SM, so that one CTA fits
    several genes in turn.  mpmath at this m is too slow, so the KKT certificate of the reference and the per-row
    checks are made in float64 with math.fsum instead: every per-sample term is computed with at most 8 roundings of
    relative size eps, fsum adds them exactly, so each 40-digit quantity of the short-row test is known here to within
    8 eps times the sum of the magnitudes of its terms, which the bounds below add."""
    D, DP, dev, sms = backend
    m, p = 13000, 2
    assert _optim_smem(m, p) > 200 * 1024 and _optim_smem(m, p) - 2 * ((m + 3) & ~3) * 8 <= 200 * 1024
    n = 8 * sms + 3
    rng = np.random.default_rng(13000)
    x = x_condition(m)
    sf = np.exp(rng.normal(0.0, 0.25, m))
    b_true = np.c_[rng.uniform(1.0, 5.0, n), rng.normal(0.0, 1.0, n)]
    alphas = np.array([(0.05, 0.5, 2.0)[g % 3] for g in range(n)])
    y = np.array([_nb(rng, sf * np.exp(x @ b_true[g]), alphas[g]) for g in range(n)])
    y[1, x[:, 1] == 1] = 0                                   # a zero cell: the ridge-only direction
    start = b_true + rng.normal(0.0, 0.5, (n, p))
    start[2] = np.nan
    lam = np.full(p, RIDGE)
    nf = np.broadcast_to(sf, (n, m))
    beta, conv, it = _run_optim(D, dev, x, y, nf, None, alphas, lam, start, "i4")
    for g in range(n):
        tag = f"long row {g}"
        row = Row(y[g], x, sf, None, alphas[g], lam)
        b = _f64_newton(row, start[g])
        for _ in range(3):                                   # float64 Newton polish of the free coordinates
            e = row.f64_eval(b)
            fr = ~np.array(_active(b, e["g"]))
            b[fr] += np.linalg.solve(e["Hn"][np.ix_(fr, fr)], e["g"][fr])
        e = row.f64_eval(b)
        act = np.array(_active(b, e["g"]))
        fr = ~act
        assert np.all(np.abs(b[fr]) < U) and np.all(np.abs(b[act]) == U)
        assert np.all(np.abs(e["g"][fr]) <= _f64_err(row, b, e)[1][fr]), f"{tag}: reference not certified"
        assert conv[g] == 1 and it[g] < MAXIT, (tag, conv[g], it[g])
        assert np.all(beta[g][act] == b[act]), (tag, beta[g], b)
        ed = row.f64_eval(beta[g])
        ferr, gerr = _f64_err(row, beta[g], ed)
        # the stop rule of fit_optim.cu (see _check_optim_row), its scale summed exactly
        h1 = ed["mu"] * (1.0 + row.alpha * row.y) / (1.0 + row.alpha * ed["mu"]) ** 2
        gs = np.array([math.fsum(np.abs(row.x[:, k]) * (np.abs(ed["gt"][:, k] / np.where(row.x[:, k] == 0, 1.0,
                                                                                        row.x[:, k])) + h1))
                       for k in range(p)]) + 1.0 + row.lam * np.abs(beta[g])
        tol = 1e-10 * gs
        dact = np.array(_active(beta[g], ed["g"]))
        assert np.all(np.abs(ed["g"][~dact]) <= 4.0 * tol[~dact] + gerr[~dact]), \
            f"{tag}: projected gradient {ed['g']} > 4 tol = {4 * tol}"
        lmin = np.linalg.eigvalsh(e["Hn"][np.ix_(fr, fr)])[0]
        gap = e["f"] - ed["f"]
        bound = (max(0.5 * np.sum((4.0 * tol[fr]) ** 2) / lmin, 64.0 * np.spacing(abs(e["f"]))) + ferr
                 + _f64_err(row, b, e)[0])
        assert gap <= bound, f"{tag}: objective gap {gap:.3e} > {bound:.3e}"


# ---------------------------------------------------------------- the optim fallback of a DESeq() fit

def _f64_err(row, b, e):
    """Error bounds of Row.f64_eval's objective and gradient against their exact values at b.  le = x b + log nf
    carries at most (p + 2) eps (|x| |b| + |log nf|) absolute error, so mu a relative error of that plus one ulp; every
    other per-sample operation rounds once (at most 6 of them per term), and math.fsum adds the terms exactly.  So the
    objective term y le - (y + r) log1p(alpha mu) is off by at most c eps (|y le| + (y + r) log1p(alpha mu)) + (y + r)
    dle, the gradient term x (y - mu) / (1 + alpha mu) by c eps |x| (y + mu) / (1 + alpha mu), with c = 8 + dle / eps."""
    w = np.ones(row.m) if row.w is None else row.w
    dle = (row.p + 2) * EPS * (np.abs(row.x) @ np.abs(b) + np.abs(np.log(row.nf)))
    c = 8.0 * EPS + dle
    r = 1.0 / row.alpha
    mu = e["mu"]
    l1p = np.log1p(row.alpha * mu)
    ferr = math.fsum(w * (c * (np.abs(row.y * e["le"]) + (row.y + r) * l1p) + (row.y + r) * dle))
    ferr += 4 * EPS * math.fsum(row.lam * b * b) + 2 * EPS * abs(e["f"])
    gerr = (np.abs(row.x) * (c * w * (row.y + mu) / (1.0 + row.alpha * mu))[:, None]).sum(axis=0)
    gerr = gerr + 2 * EPS * np.abs(row.lam * b)
    return ferr, gerr


@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "weighted"])
def test_optim_fallback_against_R_formulas(backend, weighted):
    """device_pipeline._optim_fallback on a call that mixes planted rows (test_optim.R's row and variations: the IRLS
    cannot fit them) with ordinary rows.  Against R's post-optim formulas (R/fitNbinomGLMs.R:372-403) at 40 digits,
    evaluated at the device's coefficients: the stored mean is unclamped (:384-386), logLike is at the minmu-clamped
    mean (:387, 398-403, weighted when weights are given), betaSE is the sandwich at the clamped mean (:388-397),
    betaConv follows :378-380, and the rows not refitted keep the IRLS output bit for bit."""
    import torch
    D, DP, dev, _ = backend
    m, n = 10, 24
    rng = np.random.default_rng(240 + weighted)
    x = x_condition(m)
    sf = np.exp(rng.normal(0.0, 0.25, m))
    sf /= np.exp(np.mean(np.log(sf)))
    b_true = np.c_[rng.uniform(2.0, 6.0, n), rng.normal(0.0, 1.0, n)]
    alphas = np.array([(0.05, 0.1, 0.5, 10.0)[g % 4] for g in range(n)])
    y = np.array([_nb(rng, sf * np.exp(x @ b_true[g]), min(alphas[g], 1.0)) for g in range(n)])
    planted = np.arange(0, n, 4)
    y[planted] = [0, 0, 0, 0, 0, 1000, 1000, 0, 0, 0]
    y[planted[1], 5] = 3000
    y[planted[2], 9] = 2
    y[planted[3]] = y[planted[3], ::-1]
    w = rng.uniform(0.3, 1.0, (n, m)) if weighted else None
    if weighted:
        w[:, 3] = 1e-4
        w[planted[0], 2] = 0.0
    yd = D.to_gene_major(y.astype(np.int32), dev)
    wd = None if w is None else D.to_gene_major(w, dev)
    xd = D.x_to_device(x, dev)
    sfd = _T(sf, dev)
    ad = _T(alphas, dev)
    p = 2
    lam = np.full(p, RIDGE)
    lamd = _T(lam, dev)
    contrast = _T(np.r_[1.0, 0.0], dev)
    Q, R = np.linalg.qr(x)
    beta0 = _T(np.linalg.solve(R, Q.T @ np.log(y / sf + 0.1).T), dev)
    fb = D.fit_beta(yd, xd, sfd, ad, contrast, beta0, lamd, 1e-8, 100, weights=wd, want_hat=False, want_mu=False)
    ll = D.nb_loglik(yd, xd, sfd, ad, fb["beta_mat"], weights=wd, want_mu=True)
    before = {k: v.clone() for k, v in fb.items() if v is not None}
    ll_before = {k: v.clone() for k, v in ll.items()}
    # what _optim_fallback will refit, and the optim run it makes (the kernel is deterministic: the same call again)
    irls_conv = (before["iter"] < 100).cpu().numpy()
    stable = ~torch.isnan(before["beta_mat"]).any(dim=0).cpu().numpy()
    varpos = ~(before["beta_var_mat"] <= 0).any(dim=0).cpu().numpy()
    rows = np.flatnonzero(~irls_conv | ~stable | ~varpos)
    assert set(planted) <= set(rows) and len(rows) < n, rows
    bm = before["beta_mat"].cpu().numpy()
    usable = stable[rows] & np.all(np.abs(bm[:, rows] / LN2) < 30, axis=0)
    start = np.nan_to_num(np.where(usable[None, :], bm[:, rows], beta0.cpu().numpy()[:, rows]), nan=0.0)
    o = D.beta_optim(yd[rows].contiguous(), xd, sfd, ad[rows].contiguous(), lamd, _T(start, dev),
                     weights=None if wd is None else wd[rows].contiguous())
    conv, nopt = DP._optim_fallback(yd, xd, sfd, ad, fb, beta0, lamd, contrast, 100, MINMU, ll, weights=wd)
    assert nopt == len(rows)
    conv = conv.cpu().numpy()
    ob = o["beta_mat"].cpu().numpy()
    got_b = fb["beta_mat"].cpu().numpy()
    assert np.array_equal(got_b[:, rows], ob)                              # the refit stores optim's coefficients
    # betaConv (:378-380): TRUE where the IRLS converged or optim reports convergence
    assert np.array_equal(conv[rows], irls_conv[rows] | (o["converged"].cpu().numpy() != 0))
    assert np.array_equal(conv[np.setdiff1d(np.arange(n), rows)], irls_conv[np.setdiff1d(np.arange(n), rows)])
    # rows not refitted: the IRLS output, bit for bit
    keep = np.setdiff1d(np.arange(n), rows)
    for k, v in before.items():
        a, b = fb[k].cpu().numpy(), v.cpu().numpy()
        sl = (slice(None), keep) if a.ndim == 2 and a.shape[0] == p else keep
        assert np.array_equal(a[sl], b[sl], equal_nan=True), k
    for k in ("logLike", "mu"):
        assert np.array_equal(ll[k].cpu().numpy()[keep], ll_before[k].cpu().numpy()[keep], equal_nan=True), k
    got_mu = ll["mu"].cpu().numpy()[:, :m]
    got_ll = ll["logLike"].cpu().numpy()
    got_var = fb["beta_var_mat"].cpu().numpy()
    for i, g in enumerate(rows):
        b = got_b[:, g]
        wg = np.ones(m) if w is None else w[g]
        with mpmath.workdps(DPS):
            bm_ = [_mp(v) for v in b]
            mus = [_mp(sf[j]) * mpmath.exp(_mp(x[j, 0]) * bm_[0] + _mp(x[j, 1]) * bm_[1]) for j in range(m)]
            # (:384-386) the stored mean is unclamped.  The kernel's le = fl(x beta) + fl(log nf) is off the exact
            # value by at most 2 ulp of |x beta| + |log nf|, and its exp by 1 ulp (see the nb_loglik test)
            for j in range(m):
                rm = float(mus[j])
                lim = np.spacing(rm) + rm * 2 * EPS * (abs(x[j] @ b) + abs(math.log(sf[j])) + 1)
                assert abs(got_mu[g, j] - rm) <= lim, (g, j, got_mu[g, j], rm)
            # (:387, 398-403) logLike at the clamped mean, weighted; the bound is the one derived in
            # test_nb_loglik_against_40_digits for the kernel's sum
            cl = [max(v, _mp(MINMU)) for v in mus]
            ref_ll = mpmath.fsum(_mp(wg[j]) * ref_logdens(y[g, j], cl[j], alphas[g]) for j in range(m))
            scale = sum(_loglik_scale(y[g, j], float(cl[j]), alphas[g], wg[j], abs(x[j] @ b), abs(math.log(sf[j])))
                        for j in range(m))
            assert abs(got_ll[g] - float(ref_ll)) <= 1e-14 * scale, (g, got_ll[g], float(ref_ll), scale)
            # (:388-397) the sandwich (X'WX + ridge)^-1 X'WX (X'WX + ridge)^-1 at the clamped mean
            W = [_mp(wg[j]) / (1 / cl[j] + _mp(alphas[g])) for j in range(m)]
            XtWX = mpmath.matrix(p, p)
            for a_ in range(p):
                for c_ in range(p):
                    XtWX[a_, c_] = mpmath.fsum(_mp(x[j, a_]) * W[j] * _mp(x[j, c_]) for j in range(m))
            A = XtWX + mpmath.diag([_mp(v) for v in lam])
            Ai = A ** -1
            S = Ai * XtWX * Ai
            # fit_beta's covariance (maxit = 0): the sandwich bound of test_irls_reference, which scales with
            # kappa(DAD), D = diag(A)^-1/2 (the equilibrated matrix the kernel factors), not with kappa(A).  X'WX
            # carries the rounding of its m-term sums and of w, whose mean is off by the rounding of le (see above)
            f = lambda M_: np.array(M_.tolist(), dtype=np.float64)
            Wf = np.array([float(v) for v in W])
            dw = (p + 2) * EPS * (np.abs(x) @ np.abs(b) + np.abs(np.log(sf))) + 6 * EPS
            E_B = np.abs(x).T @ ((Wf * (dw + (m + 2) * EPS))[:, None] * np.abs(x))
            dS = sandwich_bound(f(Ai), f(XtWX), f(S), E_B + chol_backward(f(A), p), E_B, p)
            for a_ in range(p):
                rv = float(S[a_, a_])
                assert abs(got_var[a_, g] - rv) <= dS[a_, a_], (g, a_, got_var[a_, g], rv, dS[a_, a_])


# ---------------------------------------------------------------- nb_loglik

def _loglik_scale(y, mu, alpha, w, eta_abs, lnf_abs):
    """The sum of the magnitudes of what nb_loglik_kernel adds for one sample (fit_beta.cu, nb_logdens.cuh), times
    |w|: lgamma_diff (for r >= kShift its three addends y log(y + r), (r - 1/2) log1p(y / r), y and the Stirling tails;
    else lgamma(y + r) and lgamma(r)), log y!, y (le + log alpha), (y + r) log1p(alpha mu); plus the effect of the
    rounding of le = fl(x beta) + fl(log nf) through d t / d le = y - (y + r) alpha mu / (1 + alpha mu)."""
    r = 1.0 / alpha
    if r >= 10.0:
        lgd = abs(y * math.log(y + r)) + abs((r - 0.5) * math.log1p(y / r)) + y + 1.0 / r
    else:
        lgd = _lgamma_mag(y + r) + _lgamma_mag(r)
    le = math.log(mu) if mu > 0 else 0.0
    am = alpha * mu
    dle = y + (y + r) * am / (1.0 + am)
    return abs(w) * (lgd + _lgamma_mag(y + 1.0) + y * (abs(le) + abs(math.log(alpha))) + (y + r) * math.log1p(am)
                     + dle * (eta_abs + lnf_abs + 1.0))


def _lgamma_mag(x):
    """The magnitudes nbmath.cuh::lgamma_pos adds: below kShift = 10 it shifts x up to x + n >= 10 and subtracts
    log(x (x + 1) ... (x + n - 1)) from the Stirling value at x + n, so its rounding is relative to both (about 13 at
    x = 1, where the exact lgamma is 0: log 0! and log 1! carry an absolute error of a few 1e-14)."""
    if x >= 10.0:
        return abs(math.lgamma(x))
    xs = x + math.ceil(10.0 - x)
    return 2.0 * abs(math.lgamma(xs)) + abs(math.lgamma(x))


# le values of the exp tests: both sides of the exp_fast / exp switch at |le| = 700, the subnormal range, zero means,
# and a dense sweep over reduced arguments near +-ln2/2 where exp_fast's Taylor tail (1/13! r^13) is largest
_SWITCH = [np.nextafter(700.0, 0.0), 700.0, np.nextafter(700.0, 800.0), 699.5, 700.5, 705.0, 709.0]
LE_EDGES = np.array(_SWITCH + [-v for v in _SWITCH]
                    + [-708.0, -708.3, -708.5, -709.0, -709.5, -709.8, -710.0, -712.0, -720.0, -730.0, -740.0, -744.0,
                       -744.5, -745.0, -745.1, -745.5, -746.0, -750.0, -800.0, -1000.0])
LE_SWEEP = np.array([k * LN2 + s * (0.5 * LN2 - d) for k in (-1000, -700, -300, -40, -1, 0, 1, 40, 300, 700, 1000)
                     for s in (-1.0, 1.0) for d in (1e-9, 1e-6, 1e-3, 0.01)])
Y_VALUES = [0.0, 1.0, 255.0, 256.0, 1e6, 2.0 ** 31 - 1, 0.5, 255.5, 256.5, 1e6 + 0.25]
ALPHA_GRID = [1e-8, np.nextafter(0.1, 0.0), 0.1, np.nextafter(0.1, 1.0), 1.0, 24.0]    # max(10, m) with m = 24
M_LL = 24


def _loglik_inputs(rng):
    """Identity design (p = m = 24): sample j's le is beta_j + log nf_j exactly when nf_j = 1 (fma(1, b, 0) = b and
    fma(0, b, eta) = eta), so the exp tests see the le they are meant to."""
    genes = []                                                 # (y row, le row, alpha)
    le_all = np.r_[LE_EDGES, LE_SWEEP, rng.uniform(-699.0, 699.0, 48)]
    for i in range(0, len(le_all), M_LL):
        chunk = le_all[i:i + M_LL]
        chunk = np.r_[chunk, rng.uniform(-5, 5, M_LL - len(chunk))]
        for y0 in (0.0, 1.0):
            genes.append((np.full(M_LL, y0), chunk, 0.1 if y0 else 1.0))
    for y0 in Y_VALUES:                                        # mu around y: every term of the density of moderate size
        for a in ALPHA_GRID:
            le = math.log(max(y0, 0.5)) + rng.uniform(-3.0, 3.0, M_LL)
            genes.append((np.full(M_LL, y0), le, a))
    y = np.array([g[0] for g in genes])
    le = np.array([g[1] for g in genes])
    alpha = np.array([g[2] for g in genes])
    return y, le, alpha


@pytest.mark.parametrize("nf_kind", ["ones", "vector", "matrix"])
def test_nb_loglik_against_40_digits(backend, nf_kind):
    """nb_loglik_kernel's unclamped mean and log-likelihood against nf * exp(x beta) and dnbinom(log = TRUE) at 40
    digits, for minmu 0 and 0.5, with and without weights, int32 and float64 counts.

    mu: within 1 ulp of exp(le) where the result is normal or subnormal (np.spacing is the subnormal grid there):
    exp_fast rounds once at 1 + p (1/2 ulp) after p = r + r^2 poly(r) is rounded (at most 1/4 ulp of the result:
    |p| < 0.42) and its Taylor tail r^14/14! is below 1e-17; CUDA's exp is within 1 ulp.  With nf != 1 the kernel's le
    carries the rounding of fl(log nf) and of the sum, at most 2 eps (|log nf| + |le|), which the bound adds.
    logLike: within 1e-14 (= 45 eps) of the sum of the magnitudes of every addend the kernel forms (_loglik_scale):
    each addend is a product of at most three rounded factors, a log (<= 1.06 ulp, nbmath.cuh), an lgamma or Stirling
    tail (a few ulp) or the log1p correction, so at most ~8 eps of its magnitude, and the 32-lane strided sum of
    m = 24 samples adds at most one rounding per sample and five per butterfly level, each within eps of the running
    sum's magnitude: 8 + 24 + 5 < 45."""
    D, DP, dev, _ = backend
    rng = np.random.default_rng(700 + len(nf_kind))
    y, le, alpha = _loglik_inputs(rng)
    n, m = y.shape
    x = np.eye(m)
    if nf_kind == "ones":
        nf = np.ones((n, m))
    elif nf_kind == "vector":
        nf = np.broadcast_to(np.exp(rng.normal(0.0, 0.5, m)), (n, m)).copy()
    else:
        nf = np.exp(rng.normal(0.0, 0.5, (n, m)))
    lnf = np.log(nf)
    beta = le - lnf                                            # per gene: beta_j = target le_j - log nf_j
    nfd = _T(nf[0], dev) if nf_kind != "matrix" else D.to_gene_major(nf, dev)
    ad = _T(alpha, dev)
    bd = _T(beta.T, dev)
    with mpmath.workdps(DPS):
        mu_ref = [[_mp(nf[g, j]) * mpmath.exp(_mp(beta[g, j])) for j in range(m)] for g in range(n)]
    mu_f = np.array([[float(v) for v in r_] for r_ in mu_ref])
    w = rng.uniform(1e-4, 1.0, (n, m))
    w[:, 5] = 1e-4
    # exact zeros, where the density is finite (0 * -inf is NaN, in R as in the kernel)
    w[:, 7] = np.where((mu_f[:, 7] > 0) | (y[:, 7] == 0), 0.0, w[:, 7])
    # the kernel's le: exact for nf = 1; otherwise within 2 eps (|log nf| + |le|) of the exact x beta + log nf
    le_err = 0.0 if nf_kind == "ones" else 2 * EPS * (np.abs(lnf) + np.abs(le))
    cache = {}
    for dt in ("i4", "f8"):
        rows = np.all(y == np.round(y), axis=1) if dt == "i4" else np.ones(n, bool)
        yy = y[rows]
        yd = D.to_gene_major(yy.astype(np.int32) if dt == "i4" else yy, dev)
        sel = np.flatnonzero(rows)
        nfs = nfd if nf_kind != "matrix" else D.to_gene_major(nf[rows], dev)
        for minmu in (0.0, MINMU):
            for weighted in (False, True):
                wd = D.to_gene_major(w[rows], dev) if weighted else None
                r = D.nb_loglik(yd, x, nfs, ad[_T(sel, dev)].contiguous(), bd[:, _T(sel, dev)].contiguous(),
                                weights=wd, want_mu=True, minmu=minmu)
                got_mu = r["mu"].cpu().numpy()[:, :m]
                got_ll = r["logLike"].cpu().numpy()
                ref_mu = mu_f[rows]
                lim = np.spacing(ref_mu) + ref_mu * (le_err[rows] if nf_kind != "ones" else 0.0)
                bad = np.abs(got_mu - ref_mu) > lim
                assert not bad.any(), (f"{nf_kind} {dt} minmu {minmu}: mu off at le "
                                       f"{le[rows][bad][:4]}: {got_mu[bad][:4]} vs {ref_mu[bad][:4]}")
                for i, g in enumerate(sel):
                    wg = w[g] if weighted else np.ones(m)
                    key = (g, minmu, weighted)
                    if key not in cache:
                        with mpmath.workdps(DPS):
                            terms, scale = [], 0.0
                            for j in range(m):
                                # R's mu is the float64 nf * exp(x beta): where that underflows to 0 the density is
                                # the point mass at 0; elsewhere the exact mean (the kernel takes log mu as le, not as
                                # the log of a subnormal)
                                mu = mu_ref[g][j] if mu_f[g, j] > 0 else mpmath.mpf(0)
                                if minmu > 0 and mu < minmu:
                                    mu = _mp(minmu)
                                t = ref_logdens(y[g, j], mu, alpha[g])
                                terms.append(_mp(wg[j]) * t if wg[j] != 0 else mpmath.mpf(0))
                                scale += _loglik_scale(y[g, j], float(mu), alpha[g], wg[j], abs(beta[g, j]),
                                                       abs(lnf[g, j]))
                            cache[key] = (mpmath.fsum(terms), scale)
                    ref, scale = cache[key]
                    tag = (f"{nf_kind} {dt} minmu {minmu} w {weighted} gene {g}: y {y[g, 0]}, alpha {alpha[g]!r}, "
                           f"le {le[g, :3]}")
                    if mpmath.isinf(ref):
                        assert got_ll[i] == -np.inf, f"{tag}: {got_ll[i]} for a point mass at 0 with y > 0"
                    else:
                        err = abs(got_ll[i] - float(ref))
                        assert err <= 1e-14 * scale, f"{tag}: logLike {got_ll[i]!r} vs {float(ref)!r} ({err:.3e})"
