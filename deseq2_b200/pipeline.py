"""Host-side glue of DESeq()'s default Wald path around the three native calls.

The reference keeps all of this in R (it "stays R" in a real drop-in, SURVEY.md section 8); R is not in this
image, so the steps that prepare the inputs of fitDisp / fitBeta and consume their outputs are restated here in
numpy, one function per R function, same names, so the engine can be driven and measured end to end:

  estimateSizeFactorsForMatrix   R/core.R:535-578   (type="ratio")
  estimateSizeFactorsIterate     R/core.R:2589-2622 (sfType="iterate"; optim's L-BFGS-B on scipy's implementation)
  getBaseMeansAndVariances       R/core.R:2138-2157
  linearModelMu / roughDispEstimate / momentsDispEstimate   R/core.R:2454-2459, 2422-2437, 2439-2448
  estimateDispersionsGeneEst     R/core.R:657-860
  parametricDispersionFit        R/core.R:2166-2189  (Gamma GLM, identity link, glm.fit IRLS restated)
  fitType = "mean"               R/core.R:900-905    (trimmed mean of the gene-wise estimates)
  dispersionFunction<-           R/methods.R:142-190 (dispFit, varLogDispEsts = mad^2)
  estimateDispersionsPriorVar    R/core.R:1135-1208  (incl. the Monte-Carlo branch for 1..3 residual df, own RNG)
  estimateDispersionsMAP         R/core.R:943-1131
  fitNbinomGLMs / fitNbinomGLMsOptim   R/fitNbinomGLMs.R:29-236, 340-407 (L-BFGS-B fallback, useOptim=TRUE by default as in the reference)
  nbinomWaldTest                 R/core.R:1332-1565  (betas, SEs, Wald statistic and p-value)
  nbinomLRT                      R/core.R:1787-2012  (full vs reduced fit, 2 (l_full - l_reduced), chi-square p-value)
  getContrast                    R/results.R:760-827 (numeric contrasts through fitBeta's maxit = 0 mode)
  replaceOutliers / refit        R/core.R:2069-2115, 2484-2565 (opt-in: DESeq(minReplicatesForReplace=7))
  robustMethodOfMomentsDisp / trimmedCellVariance / calculateCooksDistance / recordMaxCooks   R/core.R:2277-2359
  fitGLMsWithPrior / estimateBetaPriorVar / Hmisc.wtd.quantile / addAllContrasts / averagePriorsOverLevels /
  makeExpandedModelMatrix (additive factor designs)   R/fitNbinomGLMs.R:242-337, R/core.R:1601-1689, 2762-2803, R/expanded.R
  DESeq                          R/core.R:280-432    (test="Wald", fitType="parametric", betaPrior=FALSE or TRUE)
  vst / varianceStabilizingTransformation / getVarianceStabilizedData / normTransform   R/vst.R, R/helper.R:421-435
                                 (fitType "parametric" / "mean"; vst's gene subset is vstSubsetPositions)
  rlog / rlogData / sparseTest   R/rlog.R  (the design [1 | I_m], or I_m with a frozen intercept, through fitNbinomGLMs)
  getAndCheckWeights             R/core.R:2697-2752  (observation weights: row-max normalisation, two rank tests per
                                 gene with a restatement of LINPACK dqrdc2, the rank routine of R's qr())

Observation weights (a "weights" assay) go through every step above that takes them in the reference, except
betaPrior=TRUE and outlier replacement, which raise with weights.
Gene-specific normalization factors (estimateNormFactors, R/core.R:2159-2163, or a user matrix): every function that
takes `sizeFactors` also takes an (n, m) matrix of the same rows, as getSizeOrNormFactors (R/core.R:2221-2228) hands
either to the code; DESeq(normalizationFactors=...) threads it through every step.

`engine` is any object with fitDisp / fitDispGrid / fitBeta taking the reference's argument names
(deseq2_b200.wrappers is the product engine and the default; tests and the bench's CPU baseline pass the
oracle).  Not restated (out of scope, SURVEY.md section 8f): the local trend fit, results()/lfcShrink().
"""
from __future__ import annotations

import numpy as np
from scipy import special as _sp

from . import wrappers as _default_engine
from .wrappers import fitBetaWrapper, fitDispGridWrapper, fitDispWrapper

LN2 = np.log(2.0)


def controlGeneRows(controlGenes, n):
    """estimateSizeFactorsForMatrix's `controlGenes` (R/core.R:564-571) as 0-based row indices: a boolean mask with one
    entry per row, or non-negative integer row indices (numpy, a list or a torch tensor), a duplicated index counting
    once per occurrence as counts[controlGenes, ] does.  R recycles a short mask, drops negative indices and turns an
    index past the end into an NA row; those are refused here (ValueError), as is any other type."""
    if hasattr(controlGenes, "detach"):
        controlGenes = controlGenes.detach().cpu().numpy()
    c = np.asarray(controlGenes)
    if c.ndim != 1:
        raise ValueError("controlGenes should be a 1-d boolean mask or integer row indices")
    if c.dtype == np.bool_:
        if c.shape[0] != n:
            raise ValueError(f"a controlGenes mask needs one entry per row ({n}), got {c.shape[0]}")
        return np.flatnonzero(c)
    if c.size == 0:
        return np.zeros(0, dtype=np.int64)
    if not np.issubdtype(c.dtype, np.integer):
        raise ValueError("controlGenes should be either a boolean mask or integer row indices")
    if c.min() < 0 or c.max() >= n:
        raise ValueError(f"controlGenes indices must lie in [0, {n})")
    return c.astype(np.int64)


def logGeoMeans(geoMeans, n):
    """log(geoMeans) with R's length check (R/core.R:551-556): a zero gives -Inf, a negative value or NaN gives NaN."""
    g = np.asarray(geoMeans, dtype=np.float64)
    if g.ndim != 1 or g.shape[0] != n:
        raise ValueError("geoMeans should be as long as the number of rows of counts")
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(g)


def checkGeoMeansType(type, geoMeans):
    """R's estimateSizeFactors replaces given geoMeans by geoMeanNZ for type "poscounts" while
    estimateSizeFactorsForMatrix uses them: the combination is refused rather than resolved one way."""
    if type not in ("ratio", "poscounts"):
        raise ValueError("type must be 'ratio' or 'poscounts'")
    if type == "poscounts" and geoMeans is not None:
        raise ValueError("type 'poscounts' computes its own geoMeans: give geoMeans with type 'ratio'")


def _selectedMedianSizes(logc, counts, loggeomeans, controlGenes):
    """R/core.R:560-572: per sample, exp(median(log K - loggeomeans)) over the (control) rows with a finite loggeomeans
    and K > 0; NaN for a sample without such a row."""
    rows = np.arange(counts.shape[0]) if controlGenes is None else controlGeneRows(controlGenes, counts.shape[0])
    lg, lc, cn = loggeomeans[rows], logc[rows], counts[rows]
    sf = np.empty(counts.shape[1])
    for j in range(counts.shape[1]):
        sel = np.isfinite(lg) & (cn[:, j] > 0)
        sf[j] = np.exp(np.median(lc[sel, j] - lg[sel])) if sel.any() else np.nan
    return sf


def estimateSizeFactorsForMatrix(counts, type="ratio", geoMeans=None, controlGenes=None):
    """R/core.R:535-578, locfunc=median.  type "ratio": loggeomeans = rowMeans(log K).  type "poscounts" (as
    estimateSizeFactors calls it, R/methods.R:377-390): geoMeans = geoMeanNZ per row, log(exp(sum(log K[K > 0]) / m))
    (0 for an all-zero row), passed as incoming geoMeans, so the factors are rescaled to geometric mean 1 (:573-576).
    geoMeans: one value per row; loggeomeans = log(geoMeans) and the factors are rescaled the same way (not together
    with "poscounts", checkGeoMeansType).  controlGenes (controlGeneRows): the median is over these rows only.  The
    stop "every gene contains at least one zero" looks at the loggeomeans of all rows, so control rows that all
    contain a zero (or all-negative geoMeans, whose log is NaN, not infinite) give NaN factors instead."""
    checkGeoMeansType(type, geoMeans)
    counts = np.asarray(counts, dtype=np.float64)
    with np.errstate(divide="ignore"):
        logc = np.log(counts)
    if geoMeans is not None:
        loggeomeans = logGeoMeans(geoMeans, counts.shape[0])
    elif type == "poscounts":
        pos = counts > 0
        s = np.where(pos, logc, 0.0).sum(axis=1)
        with np.errstate(divide="ignore"):
            loggeomeans = np.log(np.where(pos.any(axis=1), np.exp(s / counts.shape[1]), 0.0))
    else:
        loggeomeans = logc.mean(axis=1)
    if np.all(np.isinf(loggeomeans)):
        raise ValueError("every gene contains at least one zero, cannot compute log geometric means")
    sf = _selectedMedianSizes(logc, counts, loggeomeans, controlGenes)
    if type == "poscounts" or geoMeans is not None:
        sf = sf / np.exp(np.mean(np.log(sf)))
    return sf


def iterateObjective(counts, q, disps, par, h=1e-3, Q=0.05):
    """The objective of estimateSizeFactorsIterate (R/core.R:2598-2604) evaluated directly at par and at the 2m points
    of optim's central differences, in the column order of b200nb_sf_iterate_objective_dev: [fn(par), fn(par + h e_k)
    for k < m, fn(par - h e_k) for k < m], with fn(p) = sum(gene.ll[gene.ll > quantile(gene.ll, Q)]),
    gene.ll = nbinomLogLike(counts, q * exp(p - mean(p)), disps) -- 2m + 1 full log-likelihood sums."""
    counts = np.asarray(counts, dtype=np.float64)
    par = np.asarray(par, dtype=np.float64)
    m = len(par)
    pts = [par] + [par + h * np.eye(m)[k] for k in range(m)] + [par - h * np.eye(m)[k] for k in range(m)]
    out = np.empty(2 * m + 1)
    for c, p in enumerate(pts):
        ll = nbinomLogLike(counts, q * np.exp(p - np.mean(p))[None, :], disps)
        out[c] = ll[ll > np.quantile(ll, Q, method="linear")].sum()
    return out


def optimizeLogSizeFactors(evaluate, par0, h=1e-3):
    """optim(par0, fn, control = list(fnscale = -1), method = "L-BFGS-B") as estimateSizeFactorsIterate calls it
    (R/core.R:2605), on scipy's L-BFGS-B (not R's lbfgsb.c): minimise -fn with optim's defaults lmm = 5,
    factr = 1e7 (ftol = factr * eps), pgtol = 0, maxit = 100, no bounds, and optim's finite-difference gradient
    (fmingr, ndeps = h): -(fn(par + h e_k) - fn(par - h e_k)) / (2 h).  `evaluate(par)` returns the 2m + 1 values of
    iterateObjective's column order, one call per point.  Raises ValueError where optim stops on a non-finite value.
    Returns scipy's OptimizeResult (status 0 = converged; `nfev` = objective calls)."""
    from scipy import optimize as _so
    m = len(par0)

    def fg(p):
        v = np.asarray(evaluate(p), dtype=np.float64)
        if not np.isfinite(v[0]):
            raise ValueError("L-BFGS-B needs finite values of 'fn'")
        g = -(v[1:m + 1] - v[m + 1:]) / (2.0 * h)
        if not np.all(np.isfinite(g)):
            raise ValueError(f"non-finite finite-difference value [{int(np.flatnonzero(~np.isfinite(g))[0]) + 1}]")
        return -v[0], g

    return _so.minimize(fg, np.asarray(par0, dtype=np.float64), jac=True, method="L-BFGS-B",
                        options={"maxcor": 5, "ftol": 1e7 * np.finfo(float).eps, "gtol": 0.0, "maxiter": 100})


def iterateSizeFactors(m, step, niter=10, h=1e-3):
    """The outer loop of estimateSizeFactorsIterate (R/core.R:2589-2622), shared by the host mirror and the device
    path: `step(sf)` runs the dispersion chain at the size factors sf and returns (evaluate, info), the objective
    evaluator for optimizeLogSizeFactors and whatever the caller wants kept from the last iteration.  R's stops: the
    optimiser's status != 0, and niter iterations without sum((log sf_old - log sf)^2) < 1e-4 (tested from the second
    iteration on, so niter = 1 always stops).  Returns sizeFactors, iterations, evaluations (objective calls per
    iteration) and the last info."""
    sf = np.ones(m)
    evals = []
    info = None
    for i in range(1, niter + 1):
        evaluate, info = step(sf)
        sf_old = sf
        o = optimizeLogSizeFactors(evaluate, np.log(sf_old), h)
        evals.append(int(o.nfev))
        if o.status != 0:
            raise ValueError("iterative size factor normalization did not converge within an iteration")
        sf = np.exp(o.x - np.mean(o.x))
        if i > 1 and np.sum((np.log(sf_old) - np.log(sf)) ** 2) < 1e-4:
            break
        if i == niter:
            raise ValueError("iterative size factor normalization did not converge")
    return {"sizeFactors": sf, "iterations": i, "evaluations": evals, "last": info}


def estimateSizeFactorsIterate(counts, niter=10, Q=0.05, engine=None, minDisp=1e-8, minmu=0.5):
    """R/core.R:2589-2622: design ~1; each iteration estimateDispersions(fitType = "mean") at the current size
    factors, q = mu / sf of the gene-wise fit, and optim over the log size factors of the trimmed total
    log-likelihood (iterateObjective, evaluated directly).  Rows with a zero sum are left out.  Returns
    iterateSizeFactors' dict; "last" holds the last iteration's q and dispersions (and the dispersion results)."""
    counts = np.asarray(counts)
    cts = counts[counts.sum(axis=1) > 0]
    m = cts.shape[1]
    x = np.ones((m, 1))

    def step(sf):
        mv = getBaseMeansAndVariances(cts, sf)
        ge = estimateDispersionsGeneEst(cts, sf, x, engine=engine, mv=mv, minmu=minmu, minDisp=minDisp)
        tf = estimateDispersionsFit(ge["dispGeneEst"], ge["baseMean"], minDisp=minDisp, fitType="mean")
        dispPriorVar = estimateDispersionsPriorVar(tf["varLogDispEsts"], m, 1, ge["dispGeneEst"], tf["dispFit"],
                                                   minDisp)
        mp = estimateDispersionsMAP(cts, x, ge["mu"], ge["dispGeneEst"], tf["dispFit"], dispPriorVar,
                                    tf["varLogDispEsts"], engine=engine, minDisp=minDisp)
        q = ge["mu"] / sf[None, :]
        disps = mp["dispersion"]
        info = {"q": q, "dispersion": disps, "dispGeneEst": ge["dispGeneEst"], "meanDisp": tf["meanDisp"],
                "dispPriorVar": dispPriorVar}
        return (lambda par: iterateObjective(cts, q, disps, par, Q=Q)), info

    return iterateSizeFactors(m, step, niter=niter)


def _div(sizeFactors):
    """getSizeOrNormFactors: the (m,) size factors as a (1, m) row, or an (n, m) normalization-factor matrix as is."""
    sf = np.asarray(sizeFactors, dtype=np.float64)
    return sf if sf.ndim == 2 else sf[None, :]


def estimateNormFactors(counts, normMatrix, type="ratio", geoMeans=None, controlGenes=None):
    """R/core.R:2159-2163 as estimateSizeFactors calls it (R/methods.R:377-402), in the reference's formula order:
    the median-of-ratios size factors of counts / normMatrix -- for type "poscounts" with the geoMeans of the raw
    counts, log(exp(sum(log K[K > 0]) / m)), and the incoming-geoMeans rescaling sf / exp(mean(log sf))
    (R/core.R:573-576) -- then nf = normMatrix * sf divided by its row geometric mean.  geoMeans and controlGenes as
    in estimateSizeFactorsForMatrix: the given geoMeans are compared with counts / normMatrix, the median is over the
    control rows, and nf is formed for every row."""
    checkGeoMeansType(type, geoMeans)
    counts = np.asarray(counts, dtype=np.float64)
    nm = np.asarray(normMatrix, dtype=np.float64)
    if nm.shape != counts.shape or not np.all(np.isfinite(nm) & (nm > 0)):
        raise ValueError("normMatrix must be finite, positive and of the counts' shape")
    cnts = counts / nm
    m = counts.shape[1]
    with np.errstate(divide="ignore"):
        logc = np.log(cnts)
        if geoMeans is not None:
            loggeomeans = logGeoMeans(geoMeans, counts.shape[0])
        elif type == "poscounts":
            pos = counts > 0
            s = np.where(pos, np.log(np.where(pos, counts, 1.0)), 0.0).sum(axis=1)
            loggeomeans = np.log(np.where(pos.any(axis=1), np.exp(s / m), 0.0))
        else:
            loggeomeans = logc.mean(axis=1)
    if np.all(np.isinf(loggeomeans)):
        raise ValueError("every gene contains at least one zero, cannot compute log geometric means")
    sf = _selectedMedianSizes(logc, cnts, loggeomeans, controlGenes)
    if type == "poscounts" or geoMeans is not None:
        sf = sf / np.exp(np.mean(np.log(sf)))
    nf = nm * sf[None, :]
    return nf / np.exp(np.log(nf).mean(axis=1))[:, None]


def getBaseMeansAndVariances(counts, sizeFactors, weights=None):
    """R/core.R:2138-2157.  With weights: mean and variance of the RAW weights times the normalised counts; allZero
    stays the unweighted row sum.  sizeFactors: (m,) or an (n, m) normalization-factor matrix."""
    norm = np.asarray(counts, dtype=np.float64) / _div(sizeFactors)
    if weights is not None:
        norm = np.asarray(weights, dtype=np.float64) * norm
    return {"baseMean": norm.mean(axis=1), "baseVar": norm.var(axis=1, ddof=1),
            "allZero": np.asarray(counts).sum(axis=1) == 0}


def dqrdc2_rank(z, tol=1e-7):
    """The rank R's qr(z) reports: LINPACK dqrdc2 (R's src/appl/dqrdc2.f), Householder with limited column pivoting.
    Columns are taken in order; one whose norm after the transformations so far falls below tol times its original norm
    (1 for a zero column) is moved to the end and no longer counted.  The norms are downdated as dqrdc2 does, and
    recomputed when the downdate loses precision."""
    x = np.array(z, dtype=np.float64)
    n, p = x.shape
    if n == 0 or p == 0:
        return 0
    qraux = np.sqrt((x * x).sum(axis=0))
    work1 = qraux.copy()
    work2 = np.where(qraux == 0.0, 1.0, qraux)
    k = p + 1                                     # 1-based, as in the Fortran
    for l in range(min(n, p)):                    # 0-based column / row l
        while l + 1 < k and qraux[l] < work2[l] * tol:
            x[:, l:] = np.roll(x[:, l:], -1, axis=1)
            qraux[l:] = np.roll(qraux[l:], -1)
            work1[l:] = np.roll(work1[l:], -1)
            work2[l:] = np.roll(work2[l:], -1)
            k -= 1
        if l == n - 1:
            continue
        nrmxl = np.sqrt(np.sum(x[l:, l] ** 2))
        if nrmxl == 0.0:
            continue
        if x[l, l] != 0.0:
            nrmxl = np.copysign(nrmxl, x[l, l])
        x[l:, l] /= nrmxl
        x[l, l] += 1.0
        for j in range(l + 1, p):
            t = -np.dot(x[l:, l], x[l:, j]) / x[l, l]
            x[l:, j] += t * x[l:, l]
            if qraux[j] == 0.0:
                continue
            tt = max(1.0 - (abs(x[l, j]) / qraux[j]) ** 2, 0.0)
            if abs(tt) < 1e-6:
                qraux[j] = np.sqrt(np.sum(x[l + 1:, j] ** 2))
                work1[j] = qraux[j]
            else:
                qraux[j] = qraux[j] * np.sqrt(tt)
        qraux[l] = x[l, l]
        x[l, l] = -nrmxl
    return min(k - 1, n)


def check_test_args(x, test, reduced, betaPrior):
    """DESeq()'s checks of test / reduced for model matrices (R/core.R:318-344; checkFullRank :2624-2644 with R's qr
    rank).  Raises ValueError as R stops; returns reduced as a float64 matrix (None for the Wald test)."""
    if test not in ("Wald", "LRT"):
        raise ValueError("test must be 'Wald' or 'LRT'")
    if test == "Wald":
        if reduced is not None:
            raise ValueError("'reduced' ignored when test='Wald'")
        return None
    if reduced is None:
        raise ValueError("likelihood ratio test requires a 'reduced' design, see ?DESeq")
    if betaPrior:
        raise ValueError("test='LRT' does not support use of LFC shrinkage, use betaPrior=FALSE")
    reduced = np.asarray(reduced, dtype=np.float64)
    if reduced.ndim != 2 or reduced.shape[0] != x.shape[0] or reduced.shape[1] == 0:
        raise ValueError(f"reduced must be a model matrix with one row per sample ({x.shape[0]}), got shape "
                         f"{reduced.shape}")
    for name, mm in (("full", x), ("reduced", reduced)):
        if dqrdc2_rank(mm) < mm.shape[1]:
            raise ValueError(f"the {name} model matrix is not full rank, so the model cannot be fit as specified")
    if x.shape[1] <= reduced.shape[1]:
        raise ValueError("the number of columns of 'full' should be more than the number of columns of 'reduced'")
    return reduced


def getAndCheckWeights(weights, x, weightThreshold=1e-2):
    """R/core.R:2697-2752 for a full-rank model matrix.  Returns (weights / row maximum, weightsFail).  Raises
    ValueError where the reference stops: a negative or NaN weight (stopifnot), a row without a positive weight or an
    infinite weight (NaN after the normalisation, which qr() rejects).  A gene fails unless qr(w * X) has rank p and
    X on the samples with w > weightThreshold, all-zero columns dropped, has full column rank."""
    w = np.asarray(weights, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    if w.ndim != 2 or w.shape[1] != x.shape[0]:
        raise ValueError(f"weights must have one column per sample: shape {w.shape}, {x.shape[0]} samples")
    if not np.all(w >= 0):
        raise ValueError("weights must be non-negative and not NaN")
    wmax = w.max(axis=1) if w.shape[0] else np.zeros(0)
    if np.any(~(wmax > 0)) or np.any(~np.isfinite(wmax)):
        raise ValueError("every row of weights needs a positive, finite maximum")
    wn = w / wmax[:, None]
    p = x.shape[1]
    fail = np.zeros(len(wn), bool)
    for i in range(len(wn)):
        test1 = dqrdc2_rank(wn[i][:, None] * x) == p
        sub = x[wn[i] > weightThreshold]
        sub = sub[:, np.abs(sub).sum(axis=0) > 0]
        test2 = dqrdc2_rank(sub) == sub.shape[1]
        fail[i] = not (test1 and test2)
    return wn, fail


def linearModelMu(y, x):
    """R/core.R:2454-2459: (y Q)(x R^-1)'."""
    Q, R = np.linalg.qr(x)
    Rinv = np.linalg.inv(R)
    return (y @ Q) @ (x @ Rinv).T


def roughDispEstimate(y, x):
    """R/core.R:2422-2437."""
    mu = np.maximum(1.0, linearModelMu(y, x))
    m, p = x.shape
    est = (((y - mu) ** 2 - mu) / mu ** 2).sum(axis=1) / (m - p)
    return np.maximum(est, 0.0)


def momentsDispEstimate(baseMean, baseVar, sizeFactors):
    """R/core.R:2439-2448; with an (n, m) normalization-factor matrix xim = mean(1 / colMeans(nf)) over its rows."""
    sizeFactors = np.asarray(sizeFactors, dtype=np.float64)
    xim = np.mean(1.0 / (sizeFactors.mean(axis=0) if sizeFactors.ndim == 2 else sizeFactors))
    return (baseVar - xim * baseMean) / baseMean ** 2


def modelMatrixGroups(x):
    """R/core.R:2450-2452: number of distinct rows of the design."""
    return len({tuple(r) for r in np.asarray(x)})


def _stirling_tail(x):
    xi = 1.0 / x
    x2 = xi * xi
    return xi * (1.0 / 12 - x2 * (1.0 / 360 - x2 * (1.0 / 1260 - x2 * (1.0 / 1680 - x2 * (1.0 / 1188)))))


def _lgamma_diff(y, r):
    """lgamma(y + r) - lgamma(r) without the cancellation of two ~r log r numbers (r = 1/alpha reaches 1e8, where the
    direct difference loses ~1e-7 per sample): for r >= 10 the Stirling forms are subtracted analytically."""
    r = np.broadcast_to(r, y.shape)
    big = r >= 10.0
    out = np.empty(y.shape)
    rb, yb = r[big], y[big]
    out[big] = yb * np.log(yb + rb) + (rb - 0.5) * np.log1p(yb / rb) - yb + _stirling_tail(yb + rb) - _stirling_tail(rb)
    out[~big] = _sp.gammaln(y[~big] + r[~big]) - _sp.gammaln(r[~big])
    return out


def nbinomLogLike(counts, mu, disp, weights=None):
    """R/core.R:2208-2217: rowSums(weights * dnbinom(counts, mu = mu, size = 1/disp, log = TRUE)).  Evaluated in
    the cancellation-free direct form (the same as the device kernels), with dnbinom_mu's point mass at mu = 0."""
    y = np.asarray(counts, dtype=np.float64)
    mu = np.asarray(mu, dtype=np.float64)
    alpha = np.asarray(disp, dtype=np.float64)[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (_lgamma_diff(y, 1.0 / alpha) - _sp.gammaln(y + 1) + _sp.xlogy(y, mu * alpha)
             - (y + 1.0 / alpha) * np.log1p(mu * alpha))
    t = np.where(mu == 0, np.where(y == 0, 0.0, -np.inf), t)
    if weights is not None:
        t = np.asarray(weights, dtype=np.float64) * t
    return t.sum(axis=1)


def estimateDispersionsGeneEst(counts, sizeFactors, x, engine=None, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6,
                               maxit=100, useCR=True, weightThreshold=1e-2, minmu=0.5, mv=None, weights=None):
    """R/core.R:657-860 for niter=1.  `counts` holds only the non-all-zero rows; `weights` (optional) are the
    normalised weights of those rows (getAndCheckWeights).  With weights there is no linear mu (:738-741), mu comes
    from the weighted GLM fit, and fitDisp / fitDispGrid get pmax(weights, 1e-6) (:702)."""
    engine = engine or _default_engine
    counts = np.asarray(counts)
    n, m = counts.shape
    p = x.shape[1]
    if mv is None:
        mv = getBaseMeansAndVariances(counts, sizeFactors)      # with weights the caller passes the weighted pair
    norm = counts / _div(sizeFactors)
    useWeights = weights is not None
    wdisp = np.maximum(weights, 1e-6) if useWeights else None
    roughDisp = roughDispEstimate(norm, x)
    momentsDisp = momentsDispEstimate(mv["baseMean"], mv["baseVar"], sizeFactors)
    alpha_hat = np.minimum(roughDisp, momentsDisp)
    maxDisp = max(10, m)
    alpha_hat = alpha_init = np.minimum(np.maximum(minDisp, alpha_hat), maxDisp)
    linearMu = modelMatrixGroups(x) == p and not useWeights
    nf = np.broadcast_to(_div(sizeFactors), (n, m))
    if not linearMu:
        fit = fitNbinomGLMs(counts, nf, x, alpha_hat, engine=engine, weights=weights)
        fitMu = fit["mu"]
    else:
        fitMu = linearModelMu(norm, x) * nf
    fitMu = np.maximum(fitMu, minmu)
    dispRes = fitDispWrapper(ySEXP=counts, xSEXP=x, mu_hatSEXP=fitMu, log_alphaSEXP=np.log(alpha_hat),
                             log_alpha_prior_meanSEXP=np.log(alpha_hat), log_alpha_prior_sigmasqSEXP=1.0,
                             min_log_alphaSEXP=np.log(minDisp / 10), kappa_0SEXP=kappa_0, tolSEXP=dispTol,
                             maxitSEXP=maxit, usePriorSEXP=False, weightsSEXP=wdisp, useWeightsSEXP=useWeights,
                             weightThresholdSEXP=weightThreshold, useCRSEXP=useCR, engine=engine)
    dispIter = dispRes["iter"]
    dispGeneEst = np.minimum(np.exp(dispRes["log_alpha"]), maxDisp)
    noIncrease = dispRes["last_lp"] < dispRes["initial_lp"] + np.abs(dispRes["initial_lp"]) / 1e6
    dispGeneEst[noIncrease] = alpha_init[noIncrease]
    dispGeneEstConv = (dispIter < maxit) & ~(dispIter == 1)
    refitDisp = ~dispGeneEstConv & (dispGeneEst > minDisp * 10)
    if refitDisp.sum() > 0:
        dispGrid = fitDispGridWrapper(y=counts[refitDisp], x=x, mu=fitMu[refitDisp],
                                      logAlphaPriorMean=np.zeros(int(refitDisp.sum())), logAlphaPriorSigmaSq=1.0,
                                      usePrior=False, weightsSEXP=wdisp[refitDisp] if useWeights else None,
                                      useWeightsSEXP=useWeights,
                                      weightThresholdSEXP=weightThreshold, useCRSEXP=useCR, engine=engine)
        dispGeneEst[refitDisp] = dispGrid
    dispGeneEst = np.minimum(np.maximum(dispGeneEst, minDisp), maxDisp)
    return {"dispGeneEst": dispGeneEst, "dispGeneIter": dispIter, "mu": fitMu, "baseMean": mv["baseMean"],
            "baseVar": mv["baseVar"], "n_refit": int(refitDisp.sum()), "dispRes": dispRes}


def _gamma_glm_identity(y, xinv, start, maxit=25, epsilon=1e-8):
    """glm(y ~ I(1/means), family=Gamma(link='identity'), start=start) via glm.fit's IRLS:
    eta = mu, working weights 1/mu^2, working response y; converged when |dev-devold|/(|dev|+0.1) < epsilon."""
    X = np.c_[np.ones_like(xinv), xinv]
    coef = np.asarray(start, dtype=np.float64)
    mu = X @ coef
    dev_old = 2.0 * np.sum(-np.log(y / mu) + (y - mu) / mu)
    converged = False
    for _ in range(maxit):
        w = 1.0 / mu ** 2
        XtW = X.T * w
        coef = np.linalg.solve(XtW @ X, XtW @ y)
        mu = X @ coef
        if np.any(mu <= 0):
            raise FloatingPointError("parametric dispersion fit failed")
        dev = 2.0 * np.sum(-np.log(y / mu) + (y - mu) / mu)
        if abs(dev - dev_old) / (abs(dev) + 0.1) < epsilon:
            converged = True
            break
        dev_old = dev
    return coef, converged


def parametricDispersionFit(means, disps):
    """R/core.R:2166-2189.  Returns (asymptDisp, extraPois)."""
    coefs = np.array([0.1, 1.0])
    it = 0
    while True:
        residuals = disps / (coefs[0] + coefs[1] / means)
        good = (residuals > 1e-4) & (residuals < 15)
        oldcoefs = coefs
        coefs, converged = _gamma_glm_identity(disps[good], 1.0 / means[good], coefs)
        if not np.all(coefs > 0):
            raise FloatingPointError("parametric dispersion fit failed")
        if (np.sum(np.log(coefs / oldcoefs) ** 2) < 1e-6) and converged:
            break
        it += 1
        if it > 10:
            raise FloatingPointError("dispersion fit did not converge")
    return coefs


def _mad(x):
    """stats::mad: 1.4826 * median(|x - median(x)|)."""
    return 1.4826 * np.median(np.abs(x - np.median(x)))


def r_trimmed_mean(v, trim):
    """R's mean(v, trim = trim) for 0 < trim < 0.5 (mean.default): the order statistics floor(n trim) + 1 ..
    n - floor(n trim), averaged as .Internal(mean) does, a sum over n plus the mean of the residuals."""
    v = np.sort(np.asarray(v, dtype=np.float64))
    n = len(v)
    lo = int(np.floor(n * trim))
    v = v[lo:n - lo]
    s = v.sum() / len(v)
    return float(s + (v - s).sum() / len(v))


def meanDispersionFit(dispGeneEst, minDisp=1e-8):
    """fitType = "mean" (R/core.R:900-905): mean(dispGeneEst[dispGeneEst > 10 minDisp], trim = 0.001)."""
    d = np.asarray(dispGeneEst, dtype=np.float64)
    return r_trimmed_mean(d[d > 10 * minDisp], 0.001)


def estimateDispersionsFit(dispGeneEst, baseMean, minDisp=1e-8, fitType="parametric"):
    """R/core.R:864-940 (fitType 'parametric' or 'mean') + dispersionFunction<- (R/methods.R:142-190).  For "mean"
    `coefs` is (meanDisp, 0), so coefs[0] + coefs[1] / baseMean is the constant fit, and `meanDisp` is added."""
    if fitType not in ("parametric", "mean"):
        raise ValueError("fitType must be 'parametric' or 'mean'")
    useForFit = dispGeneEst > 100 * minDisp
    if useForFit.sum() == 0:
        raise ValueError("all gene-wise dispersion estimates are within 2 orders of magnitude from the minimum value")
    if fitType == "mean":
        meanDisp = meanDispersionFit(dispGeneEst, minDisp)
        coefs = np.array([meanDisp, 0.0])
        dispFit = np.full(len(baseMean), meanDisp)
    else:
        coefs = parametricDispersionFit(baseMean[useForFit], dispGeneEst[useForFit])
        dispFit = coefs[0] + coefs[1] / baseMean
    aboveMinDisp = dispGeneEst >= minDisp * 100
    dispResiduals = np.log(dispGeneEst) - np.log(dispFit)
    varLogDispEsts = _mad(dispResiduals[aboveMinDisp]) ** 2
    out = {"dispFit": dispFit, "coefs": coefs, "varLogDispEsts": varLogDispEsts}
    if fitType == "mean":
        out["meanDisp"] = coefs[0]
    return out


def _loess_quadratic(xg, yg, xnew, span):
    """stats::loess(y ~ x, span = span) with its defaults degree = 2, family = "gaussian", evaluated directly at xnew
    (R's default surface = "interpolate" evaluates the same local fits at kd-tree vertices and blends them; on a smooth
    200-point curve the two agree far inside the Monte-Carlo noise of the curve itself): local quadratic least squares
    over the q = floor(n * span + 1e-5) nearest points with tricube weights."""
    n = len(xg)
    q = max(int(np.floor(n * span + 1e-5)), 3)
    out = np.empty(len(xnew))
    for i, x0 in enumerate(xnew):
        d = np.abs(xg - x0)
        idx = np.argpartition(d, q - 1)[:q]
        h = d[idx].max()
        w = (1.0 - (d[idx] / h) ** 3) ** 3 if h > 0 else np.ones(q)
        w = np.maximum(w, 0.0)
        X = np.c_[np.ones(q), xg[idx] - x0, (xg[idx] - x0) ** 2]
        sw = np.sqrt(w)
        coef, *_ = np.linalg.lstsq(X * sw[:, None], yg[idx] * sw, rcond=None)
        out[i] = coef[0]
    return out


def estimateDispersionsPriorVar(varLogDispEsts, m, p, dispGeneEst=None, dispFit=None, minDisp=1e-8):
    """R/core.R:1135-1208.  m - p > 3: MAD-based variance minus the sampling variance trigamma((m-p)/2), floor 0.25.
    1 <= m - p <= 3 (2-vs-2, 3-vs-2 experiments, :1157-1193): the reference matches the histogram of the log
    dispersion residuals against simulated log(chisq_{m-p}/(m-p)) + N(0, v) on a grid of v by KL divergence, smooths
    the curve with loess(span = .2) and takes the argmin; needs dispGeneEst and dispFit.  The reference fixes R's RNG
    (set.seed(2): Mersenne-Twister + inversion) for reproducibility; R's generator is not restated here, numpy's
    PCG64(2) plays its role, so the value agrees with R's within the Monte-Carlo noise of 1e4 draws per grid point
    (a few grid steps of 0.008), not bit for bit -- host glue that stays R in a real drop-in.
    m == p: no sampling variance is subtracted."""
    if m - p <= 3 and m > p:
        if dispGeneEst is None or dispFit is None:
            raise ValueError("residual df <= 3: the Monte-Carlo branch needs dispGeneEst and dispFit")
        dispGeneEst = np.asarray(dispGeneEst, dtype=np.float64)
        resid = np.log(dispGeneEst) - np.log(np.asarray(dispFit, dtype=np.float64))
        above = dispGeneEst >= minDisp * 100
        if above.sum() == 0:
            raise ValueError("no data found which is greater than minDisp")
        rng = np.random.Generator(np.random.PCG64(2))
        brks = np.arange(-20, 21) / 2.0
        obs = resid[above]
        obs = obs[(obs > brks[0]) & (obs < brks[-1])]
        obsDens = np.histogram(obs, bins=brks)[0] / (max(len(obs), 1) * 0.5)
        grid = np.linspace(0.0, 8.0, 200)
        kl = np.empty(len(grid))
        df = m - p
        for i, v in enumerate(grid):
            r = np.log(rng.chisquare(df, 10000)) + rng.normal(0.0, np.sqrt(v), 10000) - np.log(df)
            r = r[(r > brks[0]) & (r < brks[-1])]
            rDens = np.histogram(r, bins=brks)[0] / (max(len(r), 1) * 0.5)
            z = np.r_[obsDens, rDens]
            small = z[z > 0].min()
            kl[i] = np.sum(obsDens * (np.log(obsDens + small) - np.log(rDens + small)))
        fine = np.linspace(0.0, 8.0, 1000)
        fitted = _loess_quadratic(grid, kl, fine, 0.2)
        return float(max(fine[int(np.argmin(fitted))], 0.25))
    if m > p:
        expVarLogDisp = _sp.polygamma(1, (m - p) / 2.0)
        return float(max(varLogDispEsts - expVarLogDisp, 0.25))
    return float(varLogDispEsts)


def estimateDispersionsMAP(counts, x, mu, dispGeneEst, dispFit, dispPriorVar, varLogDispEsts, engine=None,
                           outlierSD=2.0, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6, maxit=100, useCR=True,
                           weightThreshold=1e-2, weights=None):
    """R/core.R:943-1131, type='DESeq2'.  `weights`: the normalised weights, unclamped (:1001-1007, 1036, 1057)."""
    engine = engine or _default_engine
    n, m = np.asarray(counts).shape
    dispInit = np.where(dispGeneEst > 0.1 * dispFit, dispGeneEst, dispFit)
    dispResMAP = fitDispWrapper(ySEXP=counts, xSEXP=x, mu_hatSEXP=mu, log_alphaSEXP=np.log(dispInit),
                                log_alpha_prior_meanSEXP=np.log(dispFit), log_alpha_prior_sigmasqSEXP=dispPriorVar,
                                min_log_alphaSEXP=np.log(minDisp / 10), kappa_0SEXP=kappa_0, tolSEXP=dispTol,
                                maxitSEXP=maxit, usePriorSEXP=True, weightsSEXP=weights,
                                useWeightsSEXP=weights is not None, weightThresholdSEXP=weightThreshold,
                                useCRSEXP=useCR, engine=engine)
    dispMAP = np.exp(dispResMAP["log_alpha"])
    dispIter = dispResMAP["iter"]
    dispConv = dispIter < maxit
    refitDisp = ~dispConv
    if refitDisp.sum() > 0:
        dispGrid = fitDispGridWrapper(y=np.asarray(counts)[refitDisp], x=x, mu=mu[refitDisp],
                                      logAlphaPriorMean=np.log(dispFit)[refitDisp], logAlphaPriorSigmaSq=dispPriorVar,
                                      usePrior=True, weightsSEXP=None if weights is None else weights[refitDisp],
                                      useWeightsSEXP=weights is not None, weightThresholdSEXP=weightThreshold,
                                      useCRSEXP=True, engine=engine)
        dispMAP[refitDisp] = dispGrid
    maxDisp = max(10, m)
    dispMAP = np.minimum(np.maximum(dispMAP, minDisp), maxDisp)
    dispersionFinal = dispMAP.copy()
    dispOutlier = np.log(dispGeneEst) > np.log(dispFit) + outlierSD * np.sqrt(varLogDispEsts)
    dispersionFinal[dispOutlier] = dispGeneEst[dispOutlier]
    return {"dispersion": dispersionFinal, "dispIter": dispIter, "dispOutlier": dispOutlier, "dispMAP": dispMAP,
            "n_refit": int(refitDisp.sum()), "dispRes": dispResMAP}


def fitNbinomGLMsOptim(counts, nf, x, lambda_, rowsForOptim, rowStable, alpha_hat, betaMatrix, betaSE, betaConv,
                       beta_mat, mu, logLike, minmu=0.5, weights=None):
    """R/fitNbinomGLMs.R:340-407: L-BFGS-B on the penalised NB log-likelihood (log2 scale, box [-30, 30]) for the rows
    the IRLS left unconverged / unstable; standard errors from the sandwich at the optimum.  With weights the
    log-likelihood and the sandwich's working weights are multiplied by them."""
    from scipy import optimize as _so
    counts = np.asarray(counts, dtype=np.float64)
    lam = np.asarray(lambda_, dtype=np.float64)
    lamNat = lam / LN2 ** 2
    large = 30.0
    betaMatrix, betaSE, betaConv, mu, logLike = (betaMatrix.copy(), betaSE.copy(), betaConv.copy(), mu.copy(),
                                                 logLike.copy())
    for row in rowsForOptim:
        betaRow = betaMatrix[row] if (rowStable[row] and np.all(np.abs(betaMatrix[row]) < large)) else beta_mat[row]
        nfr, k, alpha = nf[row], counts[row], alpha_hat[row]
        wr = None if weights is None else weights[row][None, :]

        def objective(p_):
            mu_row = nfr * 2.0 ** (x @ p_)
            ll = nbinomLogLike(k[None, :], mu_row[None, :], np.array([alpha]), wr)[0]
            logPrior = np.sum(-0.5 * np.log(2 * np.pi / lam) - 0.5 * lam * p_ ** 2)   # dnorm(p, 0, sqrt(1/lambda), log=TRUE)
            v = -(ll + logPrior)
            return v if np.isfinite(v) else 1e300

        o = _so.minimize(objective, np.asarray(betaRow, dtype=np.float64), method="L-BFGS-B",
                         bounds=[(-large, large)] * x.shape[1])
        if o.status == 0:
            betaConv[row] = True
        betaMatrix[row] = o.x
        mu_row = nfr * 2.0 ** (x @ o.x)
        mu[row] = mu_row
        mu_row = np.maximum(mu_row, minmu)
        w = 1.0 / (1.0 / mu_row + alpha)
        if wr is not None:
            w = wr[0] * w
        xtwx = (x.T * w) @ x
        inv = np.linalg.inv(xtwx + np.diag(lamNat))
        sigma = inv @ xtwx @ inv
        betaSE[row] = np.sqrt(np.maximum(np.diag(sigma), 0.0)) / LN2
        logLike[row] = nbinomLogLike(k[None, :], mu_row[None, :], np.array([alpha]), wr)[0]
    return {"betaMatrix": betaMatrix, "betaSE": betaSE, "betaConv": betaConv, "mu": mu, "logLike": logLike}


def fitNbinomGLMs(counts, nf, x, alpha_hat, lambda_=None, engine=None, betaTol=1e-8, maxit=100, useQR=True,
                  minmu=0.5, useOptim=True, forceOptim=False, weights=None):
    """R/fitNbinomGLMs.R:29-236; `weights`: normalised observation weights (getAndCheckWeights), or None.  An
    intercept-only model with the default wide prior takes the closed form (_fit_intercept_only, :99-137).  As in the
    reference (:203-227) rows with NA coefficients or
    non-positive variances ALWAYS go to the L-BFGS-B fallback, and with useOptim=TRUE (the reference's default, :30)
    so do the rows whose IRLS did not converge (iter == maxit, which includes the |beta| > 30 sentinel).  Parity tests
    that need the engine's raw output pass useOptim=False."""
    engine = engine or _default_engine
    counts = np.asarray(counts)
    n, m = counts.shape
    p = x.shape[1]
    if lambda_ is None:
        lambda_ = np.full(p, 1e-6)
    if weights is not None and p == 1 and np.all(x == 1) and np.all(np.asarray(lambda_) <= 1e-6):
        return _fit_intercept_only(counts, nf, alpha_hat, weights)
    norm = counts / nf
    if np.linalg.matrix_rank(x) == p:
        Q, R = np.linalg.qr(x)
        ylog = np.log(norm + 0.1).T
        beta_mat = np.linalg.solve(R, Q.T @ ylog).T
    else:
        beta_mat = np.zeros((n, p))
        beta_mat[:, 0] = np.log(norm.mean(axis=1))
    lambdaNatLogScale = np.asarray(lambda_, dtype=np.float64) / LN2 ** 2
    betaRes = fitBetaWrapper(ySEXP=counts, xSEXP=x, nfSEXP=nf, alpha_hatSEXP=alpha_hat, beta_matSEXP=beta_mat,
                             lambdaSEXP=lambdaNatLogScale, weightsSEXP=weights, useWeightsSEXP=weights is not None,
                             tolSEXP=betaTol, maxitSEXP=maxit, useQRSEXP=useQR, minmuSEXP=minmu, engine=engine)
    mu = nf * np.exp(betaRes["beta_mat"] @ x.T)
    logLike = nbinomLogLike(counts, mu, alpha_hat, weights)
    betaConv = betaRes["iter"] < maxit
    betaMatrix = betaRes["beta_mat"] / LN2
    betaSE = np.sqrt(np.maximum(betaRes["beta_var_mat"], 0.0)) / LN2
    rowStable = ~np.isnan(betaRes["beta_mat"]).any(axis=1)
    rowVarPositive = ~(betaRes["beta_var_mat"] <= 0).any(axis=1)
    rows = np.flatnonzero((~betaConv | ~rowStable | ~rowVarPositive) if useOptim else (~rowStable | ~rowVarPositive))
    if forceOptim:
        rows = np.arange(n)
    if True:
        if rows.size:
            o = fitNbinomGLMsOptim(counts, np.broadcast_to(nf, counts.shape), x, lambda_, rows, rowStable, alpha_hat,
                                   betaMatrix, betaSE, betaConv, beta_mat / LN2, mu, logLike, minmu=minmu,
                                   weights=weights)
            betaMatrix, betaSE, betaConv, mu, logLike = (o["betaMatrix"], o["betaSE"], o["betaConv"], o["mu"],
                                                         o["logLike"])
    return {"logLike": logLike, "betaConv": betaConv, "betaMatrix": betaMatrix, "betaSE": betaSE, "mu": mu,
            "betaIter": betaRes["iter"], "hat_diagonals": betaRes["hat_diagonals"], "betaRes": betaRes}


def r_pt_upper(q, df):
    """pt(q, df, lower.tail = FALSE) for any real df > 0 (q and df broadcast): the upper tail at |q| by scipy's stdtr,
    or for |q| < 1 as (1 - I_y(1/2, df / 2)) / 2, y = q^2 / (df + q^2), by scipy's betainc (stdtr loses ~100 ulps
    at df = 1, q = 1e-3); the normal tail ndtr(-|q|) at df = Inf; q < 0 as one minus that; NaN where df is NaN or
    <= 0 (R's NA)."""
    q, df = np.broadcast_arrays(np.asarray(q, dtype=np.float64), np.asarray(df, dtype=np.float64))
    with np.errstate(invalid="ignore", divide="ignore"):
        ok = df > 0
        d = np.where(ok, df, 1.0)
        a = np.abs(q)
        body = 0.5 * (1.0 - _sp.betainc(0.5, 0.5 * d, a * a / (d + a * a)))
        up = np.where(a < 1.0, body, _sp.stdtr(d, -a))
        up = np.where(np.isinf(df), _sp.ndtr(-a), up)
        p = np.where(q >= 0, up, 1.0 - up)
    return np.where(ok, p, np.nan)


def waldPvalue(stat, df=None):
    """nbinomWaldTest's p-value: 2 pnorm(|stat|, lower.tail = FALSE), or with the t degrees of freedom df (one per
    row, broadcast along the columns) 2 pt(|stat|, df, lower.tail = FALSE) (R/core.R:1478-1508), whose df = Inf rows
    equal the normal ones."""
    if df is None:
        return 2.0 * _sp.ndtr(-np.abs(stat))
    d = np.asarray(df, dtype=np.float64)
    d = d[:, None] if np.ndim(stat) == 2 else d
    return np.where(np.isinf(d), 2.0 * _sp.ndtr(-np.abs(stat)), 2.0 * r_pt_upper(np.abs(stat), d))


def tDegreesFreedom(df, N, nz, m, p, weights=None):
    """nbinomWaldTest's t degrees of freedom over the rows nz of N (R/core.R:1478-1504): a given df (scalar, or one
    value per row, subset to nz), else m - p, or rowSums(weights) - p with the normalised weights of those rows; NA
    (NaN) where not > 0."""
    n = int(np.sum(nz))
    if df is None:
        d = (np.asarray(weights).sum(axis=1) if weights is not None else np.full(n, float(m))) - p
    else:
        d = np.asarray(df, dtype=np.float64).reshape(-1)
        if d.size == 1:
            d = np.full(n, d[0])
        elif d.size == N:
            d = d[nz]
        else:
            raise ValueError(f"df must be a scalar or have one value per row of the counts ({N}), got {d.size}")
    with np.errstate(invalid="ignore"):
        return np.where(d > 0, d, np.nan)


def nbinomWaldTest(counts, nf, x, dispersion, engine=None, betaTol=1e-8, maxit=100, useQR=True, minmu=0.5,
                   useOptim=True, weights=None, tdf=None):
    """R/core.R:1332-1565, betaPrior=FALSE; Cook's distances are not restated.  tdf: the t degrees of freedom of the
    rows (tDegreesFreedom) for useT = TRUE, added as "tDegreesFreedom"; None is useT = FALSE."""
    fit = fitNbinomGLMs(counts, nf, x, dispersion, engine=engine, betaTol=betaTol, maxit=maxit, useQR=useQR,
                        minmu=minmu, useOptim=useOptim, weights=weights)
    with np.errstate(divide="ignore", invalid="ignore"):
        WaldStatistic = fit["betaMatrix"] / fit["betaSE"]
    WaldPvalue = waldPvalue(WaldStatistic, tdf)
    fit.update({"WaldStatistic": WaldStatistic, "WaldPvalue": WaldPvalue, "deviance": -2.0 * fit["logLike"]})
    if tdf is not None:
        fit["tDegreesFreedom"] = tdf
    return fit


def _r_trimmed_mean(x, trim):
    """R's mean(x, trim=) along the last axis: drop floor(n*trim) order statistics from each end."""
    x = np.sort(np.asarray(x, dtype=np.float64), axis=-1)
    n = x.shape[-1]
    if trim >= 0.5:
        return np.median(x, axis=-1)
    lo = int(np.floor(n * trim))
    return x[..., lo:n - lo].mean(axis=-1)


def _trimfn(n):
    """as.integer(cut(n, breaks=c(0, 3.5, 23.5, Inf))) - 1  (R/core.R:2306)."""
    return 0 if n <= 3.5 else (1 if n <= 23.5 else 2)


_TRIMRATIO = (1.0 / 3.0, 1.0 / 4.0, 1.0 / 8.0)
_SCALE_C = (2.04, 1.86, 1.51)


def designCells(x):
    """Cell (distinct design row) id per sample, in order of first appearance, and the cell sizes."""
    seen, ids = {}, []
    for r in np.asarray(x):
        ids.append(seen.setdefault(tuple(r), len(seen)))
    ids = np.asarray(ids)
    return ids, np.bincount(ids)


def trimmedCellVariance(cnts, cells):
    """R/core.R:2302-2325."""
    levels = np.unique(cells)
    cellMeans = np.empty((cnts.shape[0], len(levels)))
    for k, lvl in enumerate(levels):
        sel = cells == lvl
        cellMeans[:, k] = _r_trimmed_mean(cnts[:, sel], _TRIMRATIO[_trimfn(sel.sum())])
    qmat = cellMeans[:, np.searchsorted(levels, cells)]
    sqerror = (cnts - qmat) ** 2
    varEst = np.empty_like(cellMeans)
    for k, lvl in enumerate(levels):
        sel = cells == lvl
        t = _trimfn(sel.sum())
        varEst[:, k] = _SCALE_C[t] * _r_trimmed_mean(sqerror[:, sel], _TRIMRATIO[t])
    return varEst.max(axis=1)


def trimmedVariance(x):
    """R/core.R:2327-2332."""
    rm = _r_trimmed_mean(x, 1.0 / 8.0)
    return 1.51 * _r_trimmed_mean((x - rm[:, None]) ** 2, 1.0 / 8.0)


def robustMethodOfMomentsDisp(counts, sizeFactors, x):
    """R/core.R:2277-2300."""
    cnts = np.asarray(counts, dtype=np.float64) / _div(sizeFactors)
    cells, sizes = designCells(x)
    three = sizes[cells] >= 3
    if three.any():
        v = trimmedCellVariance(cnts[:, three], cells[three])
    else:
        v = trimmedVariance(cnts)
    m = cnts.mean(axis=1)
    return np.maximum((v - m) / m ** 2, 0.04)


def calculateCooksDistance(counts, mu, H, sizeFactors, x):
    """R/core.R:2333-2340."""
    p = x.shape[1]
    disp = robustMethodOfMomentsDisp(counts, sizeFactors, x)
    V = mu + disp[:, None] * mu ** 2
    return (np.asarray(counts, dtype=np.float64) - mu) ** 2 / V / p * H / (1 - H) ** 2


def recordMaxCooks(x, cooks):
    """R/core.R:2349-2359: max Cook's distance over the samples that have >= 3 replicates in their cell."""
    cells, sizes = designCells(x)
    samplesForCooks = sizes[cells] >= 3
    m, p = x.shape
    if m > p and samplesForCooks.any():
        return cooks[:, samplesForCooks].max(axis=1)
    return np.full(cooks.shape[0], np.nan)


def nOrMoreInCell(x, n):
    """R/core.R:2366-2371: per sample, does its design cell (distinct design row) hold at least n samples?"""
    cells, sizes = designCells(x)
    return sizes[cells] >= n


def replaceOutliers(counts, cooks, sizeFactors, x, trim=0.2, cooksCutoff=None, minReplicates=7):
    """R/core.R:2069-2115 (size factors or an (n, m) normalization-factor matrix).  Returns (counts with the outlying entries of
    replaceable samples set to as.integer(trimmed mean of the normalised counts * size factor), per-gene `replace`
    flag, per-sample `replaceable` flag).  Like the reference, `replace` is raised by an outlier in ANY sample."""
    from scipy import stats as _st
    counts = np.asarray(counts)
    n, m = counts.shape
    p = x.shape[1]
    if minReplicates < 3:
        raise ValueError("at least 3 replicates are necessary in order to indentify a sample as a count outlier")
    if m <= p:
        return counts.copy(), np.zeros(n, bool), np.zeros(m, bool)
    if cooksCutoff is None:
        cooksCutoff = _st.f.ppf(0.99, p, m - p)
    with np.errstate(invalid="ignore"):
        over = cooks > cooksCutoff                      # NA > cutoff is NA in R and drops out of which()/any()
    replace = over.any(axis=1)
    trimBaseMean = _r_trimmed_mean(counts / _div(sizeFactors), trim)
    replacementCounts = np.trunc(trimBaseMean[:, None] * _div(sizeFactors)).astype(counts.dtype)   # as.integer
    newCounts = counts.copy()
    newCounts[over] = replacementCounts[over]
    whichSamples = nOrMoreInCell(x, minReplicates)
    out = counts.copy()
    out[:, whichSamples] = newCounts[:, whichSamples]
    return out, replace, whichSamples


def getContrast(counts, nf, x, dispersion, betaMatrix, contrast, betaPriorVar=None, engine=None, minmu=0.5,
                weights=None, useT=False, df=None):
    """R/results.R:760-827: a numeric contrast c of the fitted coefficients, batched over genes through fitBeta's
    maxit = 0 mode (no IRLS iteration: covariance at the given betas, c'beta and sqrt(c' Sigma c)).  `counts` are the
    counts the model was fitted to (replaceCounts after an outlier refit), `betaMatrix` is on the log2 scale; rows are
    the non-all-zero genes.  `weights` (optional, the same rows) are normalised by their row maximum and passed to
    fitBeta, without the rank tests (R/results.R:786-807).  Returns log2FoldChange, lfcSE, stat, pvalue; with useT the
    p-value is 2 pt(|stat|, df) with df the rows' tDegreesFreedom (R/results.R:812-816)."""
    if useT and df is None:
        raise ValueError("useT=True needs the t degrees of freedom (tDegreesFreedom) of the rows")
    engine = engine or _default_engine
    counts = np.asarray(counts)
    n, m = counts.shape
    p = x.shape[1]
    contrast = np.asarray(contrast, dtype=np.float64)
    if contrast.shape != (p,):
        raise ValueError("numeric contrast vector should have one element for every element of 'resultsNames(object)'")
    if betaPriorVar is None:
        betaPriorVar = np.full(p, 1e6)                                    # betaPrior = FALSE (R/core.R:1421)
    lam = 1.0 / (LN2 ** 2 * np.asarray(betaPriorVar, dtype=np.float64))
    if weights is not None:
        w = np.asarray(weights, dtype=np.float64)
        if w.shape != counts.shape:
            raise ValueError(f"weights have shape {w.shape}, expected {counts.shape}")
        if not np.all(w >= 0):
            raise ValueError("weights must be non-negative and not NaN")
        weights = w / w.max(axis=1)[:, None]
    r = engine.fitBeta(ySEXP=counts, xSEXP=x, nfSEXP=np.broadcast_to(nf, counts.shape), alpha_hatSEXP=dispersion,
                       contrastSEXP=contrast, beta_matSEXP=LN2 * np.asarray(betaMatrix, dtype=np.float64),
                       lambdaSEXP=lam, weightsSEXP=weights, useWeightsSEXP=weights is not None, tolSEXP=1e-8,
                       maxitSEXP=0,
                       useQRSEXP=False, minmuSEXP=minmu)
    est = np.asarray(r["contrast_num"]).reshape(n) / LN2
    se = np.asarray(r["contrast_denom"]).reshape(n) / LN2
    with np.errstate(divide="ignore", invalid="ignore"):
        stat = est / se
    return {"log2FoldChange": est, "lfcSE": se, "stat": stat, "pvalue": waldPvalue(stat, df if useT else None)}


def _fit_intercept_only(counts, nf, alpha_hat, weights=None):
    """R/fitNbinomGLMs.R:99-137: reduced model ~1 with the default wide prior needs no IRLS (no native call).  With
    weights: beta = log2(sum(w K/s) / sum(w)), and the log-likelihood and the working weights are multiplied by w."""
    norm = counts / nf
    if weights is None:
        betaMatrix = np.log2(norm.mean(axis=1))[:, None]
    else:
        betaMatrix = np.log2((weights * norm).sum(axis=1) / weights.sum(axis=1))[:, None]
    mu = nf * (2.0 ** betaMatrix)
    logLike = nbinomLogLike(counts, mu, alpha_hat, weights)
    w = 1.0 / (1.0 / mu + alpha_hat[:, None])
    if weights is not None:
        w = weights * w
    xtwx = w.sum(axis=1)
    return {"logLike": logLike, "betaConv": np.ones(len(counts), bool), "betaMatrix": betaMatrix,
            "betaSE": (np.sqrt(1.0 / xtwx) / LN2)[:, None], "mu": mu, "betaIter": np.ones(len(counts)),
            "hat_diagonals": w / xtwx[:, None]}


def fitReducedModel(counts, nf, reduced, dispersion, engine=None, betaTol=1e-8, maxit=100, useQR=True, minmu=0.5,
                    useOptim=True, weights=None):
    """nbinomLRT's reduced fit (R/core.R:1863-1873): the closed form for ~1 (_fit_intercept_only), else fitNbinomGLMs."""
    if reduced.shape[1] == 1 and np.all(reduced == 1):
        return _fit_intercept_only(counts, nf, dispersion, weights)
    return fitNbinomGLMs(counts, nf, reduced, dispersion, engine=engine, betaTol=betaTol, maxit=maxit, useQR=useQR,
                         minmu=minmu, useOptim=useOptim, weights=weights)


def lrtStatistic(logLikeFull, logLikeReduced, df):
    """LRTStatistic = 2 (logLike_full - logLike_reduced) and its pchisq upper tail (R/core.R:1877-1878); df = 1 and 2
    by the closed forms erfc(sqrt(s / 2)) and exp(-s / 2) (the first terms of device_pipeline.chisq_upper's sums):
    scipy's chi2.sf loses up to 130 ulps at df = 1 for s below about 5."""
    from scipy import stats as _st
    stat = 2.0 * (logLikeFull - logLikeReduced)
    half = np.maximum(stat, 0.0) / 2.0
    if df == 1:
        return stat, _sp.erfc(np.sqrt(half))
    if df == 2:
        return stat, np.exp(-half)
    return stat, _st.chi2.sf(stat, df)


def nbinomLRT(counts, nf, full, reduced, dispersion, engine=None, betaTol=1e-8, maxit=100, useQR=True, minmu=0.5,
              useOptim=True, weights=None):
    """R/core.R:1787-2012 with user-supplied model matrices, betaPrior=FALSE; Cook's distances are not restated.
    `full` / `reduced` are m x p model matrices (reduced nested in full); `weights`: normalised weights or None."""
    counts = np.asarray(counts)
    if reduced.shape[1] >= full.shape[1]:
        raise ValueError("less than one degree of freedom, perhaps full and reduced models are not in the correct order")
    fullModel = fitNbinomGLMs(counts, nf, full, dispersion, engine=engine, betaTol=betaTol, maxit=maxit, useQR=useQR,
                              minmu=minmu, useOptim=useOptim, weights=weights)
    reducedModel = fitReducedModel(counts, nf, reduced, dispersion, engine=engine, betaTol=betaTol, maxit=maxit,
                                   useQR=useQR, minmu=minmu, useOptim=useOptim, weights=weights)
    df = full.shape[1] - reduced.shape[1]
    LRTStatistic, LRTPvalue = lrtStatistic(fullModel["logLike"], reducedModel["logLike"], df)
    return {"LRTStatistic": LRTStatistic, "LRTPvalue": LRTPvalue, "deviance": -2.0 * fullModel["logLike"],
            "betaMatrix": fullModel["betaMatrix"], "betaSE": fullModel["betaSE"], "fullBetaConv": fullModel["betaConv"],
            "reducedBetaConv": reducedModel["betaConv"], "betaIter": fullModel["betaIter"], "mu": fullModel["mu"],
            "hat_diagonals": fullModel["hat_diagonals"], "df": df}


# ---------------------------------------------------------------- beta prior (config 4: betaPrior=TRUE, expanded matrix)

def factorDesign(factors, expanded=False):
    """Model matrix of an additive design of factors, ~f1 + f2 + ... (no interactions).
    factors: list of integer level-code vectors (0 = reference level).  standard: intercept + one indicator per
    non-reference level (model.matrix treatment contrasts); expanded: intercept + one indicator for EVERY level
    (makeExpandedModelMatrix, R/expanded.R:1-18).  Returns (matrix, names, factor index per column (-1 = intercept),
    level per column)."""
    factors = [np.asarray(f) for f in factors]
    m = len(factors[0])
    cols, names, fidx, lvl = [np.ones(m)], ["Intercept"], [-1], [-1]
    for k, f in enumerate(factors):
        for l in range(0 if expanded else 1, int(f.max()) + 1):
            cols.append((f == l).astype(np.float64))
            names.append(f"f{k}{l}")
            fidx.append(k)
            lvl.append(l)
    return np.stack(cols, axis=1), names, np.asarray(fidx), np.asarray(lvl)


def wtd_quantile(x, weights, prob):
    """Hmisc.wtd.quantile(x, weights, prob, type='quantile', normwt=TRUE)  (R/core.R:2762-2803)."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(weights, dtype=np.float64)
    keep = ~(np.isnan(w) | (w == 0))
    x, w = x[keep], w[keep]
    w = w * len(x) / w.sum()                       # normwt
    order = np.argsort(x, kind="stable")
    xs, ws = x[order], w[order]
    ux, inv = np.unique(xs, return_inverse=True)   # wtd.table: sum of weights per distinct x
    wts = np.bincount(inv, weights=ws)
    n = wts.sum()
    o = 1 + (n - 1) * prob
    low = max(np.floor(o), 1.0)
    high = min(low + 1, n)
    frac = o % 1
    cum = np.cumsum(wts)

    def at(v):      # approx(cumsum(wts), x, xout=v, method='constant', f=1, rule=2): smallest x with cum >= v
        i = np.searchsorted(cum, v - 1e-12 * max(1.0, v), side="left")
        return ux[min(i, len(ux) - 1)]

    return (1 - frac) * at(low) + frac * at(high)


def matchWeightedUpperQuantileForVariance(x, weights, upperQuantile=0.05):
    """R/core.R:2416-2419."""
    from scipy import stats as _st
    sdEst = wtd_quantile(np.abs(x), weights, 1 - upperQuantile) / _st.norm.ppf(1 - upperQuantile / 2)
    return sdEst ** 2


def estimateBetaPriorVar(betaMatrix, names, fidx, baseMean, dispFit, expandedType=True, upperQuantile=0.05):
    """R/core.R:1601-1689 (betaPriorMethod='weighted').  betaMatrix: MLE log2 fold changes on the STANDARD matrix
    (columns described by names / fidx from factorDesign(expanded=False)).  Returns the prior variances for the
    standard columns and, when expandedType, for the expanded matrix columns (averagePriorsOverLevels,
    R/expanded.R:20-73) given `levels_per_factor` inferred from fidx."""
    weights = 1.0 / (1.0 / baseMean + dispFit)
    cols = {nm: betaMatrix[:, k] for k, nm in enumerate(names)}
    colsets = [(nm, betaMatrix[:, k], fidx[k]) for k, nm in enumerate(names)]
    if expandedType:                                # addAllContrasts (R/expanded.R:76-100)
        for f in sorted(set(int(v) for v in fidx if v >= 0)):
            M = betaMatrix[:, fidx == f]
            nlev = M.shape[1]
            for j in range(nlev - 1):
                for i in range(j + 1, nlev):
                    colsets.append((f"f{f}Cntrst", M[:, i] - M[:, j], f))

    def one(x):
        if len(x) == 1:                             # a single gene: betaMatrix^2, no quantile (R/core.R:1648-1666)
            return float(x[0] ** 2)
        fin = np.abs(x) < 10
        if fin.sum() == 0:
            return 1e6
        return matchWeightedUpperQuantileForVariance(x[fin], weights[fin], upperQuantile)

    pv = [(nm, one(x) if nm != "Intercept" else 1e6, f) for nm, x, f in colsets]
    std = np.array([v for (nm, v, f) in pv[:len(names)]])
    if not expandedType:
        return std, None
    mean_by_factor = {}
    for f in sorted(set(int(v) for v in fidx if v >= 0)):
        mean_by_factor[f] = float(np.mean([v for (nm, v, ff) in pv if ff == f]))
    return std, mean_by_factor


def fitGLMsWithPrior(counts, nf, factors, dispersion, baseMean, dispFit, engine=None, betaTol=1e-8, maxit=100,
                     useQR=True, minmu=0.5, useOptim=True, betaPriorVar=None, modelMatrix=None, weights=None):
    """R/fitNbinomGLMs.R:242-337 for an additive factor design with the expanded model matrix (the default when
    betaPrior=TRUE): MLE fit on the standard matrix -> estimateBetaPriorVar -> MAP fit on the expanded matrix with
    lambda = 1 / betaPriorVar.  useOptim goes to both fits (fitNbinomGLMs).
    betaPriorVar given (lfcShrink): the MLE fit and the prior are skipped, as R skips them when the first fit's mu
    and H exist (:250, :289-305); the MAP fit is on modelMatrix (modelMatrixType "standard" or "user-supplied") or,
    when it is None, on the expanded matrix of the factors, and "H", "mu", "mleBetaMatrix" and "mle" are None.
    weights: normalised observation weights of the rows, for the MAP fit."""
    mle = None
    if betaPriorVar is None:
        x_std, names, fidx, _ = factorDesign(factors, expanded=False)
        mle = fitNbinomGLMs(counts, nf, x_std, dispersion, engine=engine, betaTol=betaTol, maxit=maxit, useQR=useQR,
                            minmu=minmu, useOptim=useOptim)
        _, mean_by_factor = estimateBetaPriorVar(mle["betaMatrix"], names, fidx, baseMean, dispFit, expandedType=True)
        x_exp, enames, efidx, _ = factorDesign(factors, expanded=True)
        betaPriorVar = np.array([1e6 if f < 0 else mean_by_factor[int(f)] for f in efidx])
    elif modelMatrix is None:
        x_exp, enames = factorDesign(factors, expanded=True)[:2]
    else:
        x_exp, enames = np.asarray(modelMatrix, dtype=np.float64), None
    betaPriorVar = np.asarray(betaPriorVar, dtype=np.float64)
    if betaPriorVar.shape != (x_exp.shape[1],):
        raise ValueError(f"betaPriorVar should have length {x_exp.shape[1]} to match the model matrix")
    if np.any(betaPriorVar == 0):
        raise ValueError("beta prior variances are equal to zero for some variables")
    fit = fitNbinomGLMs(counts, nf, x_exp, dispersion, lambda_=1.0 / betaPriorVar, engine=engine, betaTol=betaTol,
                        maxit=maxit, useQR=useQR, minmu=minmu, useOptim=useOptim, weights=weights)
    if mle is None:
        return {"fit": fit, "H": None, "mu": None, "betaPriorVar": betaPriorVar, "modelMatrix": x_exp,
                "mleBetaMatrix": None, "names": enames, "mle": None}
    return {"fit": fit, "H": mle["hat_diagonals"], "mu": mle["mu"], "betaPriorVar": betaPriorVar,
            "modelMatrix": x_exp, "mleBetaMatrix": mle["betaMatrix"], "names": enames, "mle": mle}


def DESeq(counts, x, sizeFactors=None, engine=None, minReplicatesForReplace=np.inf, useOptim=True, betaPrior=False,
          factors=None, weights=None, weightThreshold=1e-2, minmu=0.5, normalizationFactors=None, sfType="ratio",
          fitType="parametric", test="Wald", reduced=None, useT=False, df=None):
    """R/core.R:280-432 with test='Wald', fitType='parametric', betaPrior=FALSE by default.
    minReplicatesForReplace: the reference's default is 7 (outlier replacement + refit whenever a design cell has >= 7
    samples, R/core.R:419-426, refitWithoutOutliers :2484-2565); the default here is Inf = off, which is what the
    engine parity tests and bench.py's `full_pipeline` exercise.  With a finite value the result also carries
    `replace` (genes refitted), `replaceable` (samples) and `replaceCounts`.
    betaPrior=True (additive factor designs only; x must be factorDesign(factors)[0], no outlier replacement): the
    Wald test goes through fitGLMsWithPrior -- coefficients, SEs, statistics and deviance of the MAP fit on the
    expanded matrix, Cook's distances from the MLE fit -- and the result also carries `mleBetaMatrix`,
    `betaPriorVar` and `modelMatrix` (the expanded matrix).
    weights: an (N, m) matrix of observation weights (the "weights" assay).  getAndCheckWeights normalises each row by
    its maximum and flags the rows whose weights leave the design rank deficient; those rows are treated as all-zero
    rows (NaN results) and reported in `weightsFail`.  baseMean / baseVar use the raw weights, every fit the
    normalised ones.  Not supported with betaPrior=True or outlier replacement (ValueError).
    minmu: the lower bound on the fitted mean (R's minmu; 1e-6 is the usual single-cell setting).
    normalizationFactors: an (N, m) matrix of gene-specific normalization factors in place of sizeFactors, used by
    every step (getSizeOrNormFactors); the moments dispersion's xim is over the non-all-zero rows.  Returned under
    `normalizationFactors`.  Not with sizeFactors or weights (ValueError).
    sfType: the estimator used when neither sizeFactors nor normalizationFactors is given: "ratio" (the default),
    "poscounts" or "iterate" (estimateSizeFactorsIterate; not with weights: ValueError).  The iterate run's outer
    iteration and objective-call counts are returned under `sfIterate`.
    fitType: "parametric" (the default; `trendCoefs`) or "mean" (R/core.R:900-905; `meanDisp` instead of
    `trendCoefs`).  Both are reported under `fitType`.
    test='LRT', reduced=<m x p_r model matrix>: nbinomLRT with the Wald path's full fit (the same fitNbinomGLMs call)
    and fitReducedModel on the same rows; adds `LRTStatistic`, `LRTPvalue`, `df`, `fullBetaConv`, `reducedBetaConv`
    and `reducedModelMatrix`, and the refitted rows of an outlier replacement get their LRT columns from the refit.
    The test is reported under `test`.  R's stops raise ValueError (check_test_args).
    useT=True, df (test='Wald' only; the LRT ignores both): Student t Wald p-values with tDegreesFreedom
    (tDegreesFreedom: df given as a scalar or per row, else m - p or rowSums(normalised weights) - p); the rows an
    outlier refit replaces get normal p-values and keep the first fit's df (refitWithoutOutliers does not pass useT).
    Returns per-gene vectors over ALL rows; all-zero rows carry NaN (buildDataFrameWithNARows, R/core.R:2232)."""
    engine = engine or _default_engine
    counts = np.asarray(counts)
    N, m = counts.shape
    p = x.shape[1]
    reduced = check_test_args(np.asarray(x, dtype=np.float64), test, reduced, betaPrior)
    if sfType not in ("ratio", "poscounts", "iterate"):
        raise ValueError("sfType must be 'ratio', 'poscounts' or 'iterate'")
    if fitType not in ("parametric", "mean"):
        raise ValueError("fitType must be 'parametric' or 'mean'")
    if sfType == "iterate" and sizeFactors is None and (weights is not None or normalizationFactors is not None):
        raise ValueError("sfType='iterate' is not supported with observation weights or normalization factors")
    sfIterate = None
    if betaPrior:
        if factors is None:
            raise ValueError("betaPrior=True needs the design factors (factors=...)")
        if not np.array_equal(np.asarray(x, dtype=np.float64), factorDesign(factors)[0]):
            raise ValueError("betaPrior=True: x must be the standard model matrix of the factors, factorDesign(factors)[0]")
        if np.isfinite(minReplicatesForReplace):
            raise ValueError("outlier replacement (finite minReplicatesForReplace) is not supported with betaPrior=True")
    if weights is not None:
        if np.shape(weights) != counts.shape:
            raise ValueError(f"weights have shape {np.shape(weights)}, expected {counts.shape}")
        if betaPrior:
            raise ValueError("observation weights are not supported with betaPrior=True")
        if np.isfinite(minReplicatesForReplace):
            raise ValueError("observation weights are not supported with outlier replacement "
                             "(finite minReplicatesForReplace)")
        wnAll, weightsFail = getAndCheckWeights(weights, x, weightThreshold)
    if normalizationFactors is not None:
        if sizeFactors is not None or weights is not None:
            raise ValueError("normalizationFactors are not supported together with sizeFactors or weights")
        sizeFactors = np.asarray(normalizationFactors, dtype=np.float64)
        if sizeFactors.shape != counts.shape or not np.all(np.isfinite(sizeFactors) & (sizeFactors > 0)):
            raise ValueError("normalizationFactors must be finite, positive and of the counts' shape")
    if sizeFactors is None:
        if sfType == "iterate":
            sfIterate = estimateSizeFactorsIterate(counts, engine=engine)
            sizeFactors = sfIterate["sizeFactors"]
        elif sfType == "poscounts":
            sizeFactors = estimateSizeFactorsForMatrix(counts, type="poscounts")
        else:
            sizeFactors = estimateSizeFactorsForMatrix(counts)
    sizeFactors = np.asarray(sizeFactors, dtype=np.float64)
    mvAll = getBaseMeansAndVariances(counts, sizeFactors, weights)
    nz = ~mvAll["allZero"]
    wnz = None
    if weights is not None:
        nz = nz & ~weightsFail
        wnz = wnAll[nz]
        if weightsFail.any():
            import warnings
            warnings.warn(f"for {int(weightsFail.sum())} row(s), the weights as supplied won't allow parameter "
                          "estimation, producing a degenerate design matrix. These rows have been flagged in "
                          "weightsFail and treated as if the row contained all zeros.")
    cnz = counts[nz]
    sfAll = sizeFactors
    if sizeFactors.ndim == 2:
        sizeFactors = sizeFactors[nz]                                   # the nf rows of the non-all-zero genes
    mv = {k: v[nz] for k, v in mvAll.items()}
    ge = estimateDispersionsGeneEst(cnz, sizeFactors, x, engine=engine, mv=mv, weights=wnz,
                                    weightThreshold=weightThreshold, minmu=minmu)
    tf = estimateDispersionsFit(ge["dispGeneEst"], ge["baseMean"], fitType=fitType)
    dispPriorVar = estimateDispersionsPriorVar(tf["varLogDispEsts"], m, p, ge["dispGeneEst"], tf["dispFit"])
    mp = estimateDispersionsMAP(cnz, x, ge["mu"], ge["dispGeneEst"], tf["dispFit"], dispPriorVar,
                                tf["varLogDispEsts"], engine=engine, weights=wnz, weightThreshold=weightThreshold)
    nf = np.broadcast_to(_div(sizeFactors), cnz.shape)
    tdf = tDegreesFreedom(df, N, nz, m, p, wnz) if useT and test == "Wald" else None
    prior = {}
    if betaPrior:
        gp = fitGLMsWithPrior(cnz, nf, factors, mp["dispersion"], mv["baseMean"], tf["dispFit"], engine=engine,
                              useOptim=useOptim)
        wt = dict(gp["fit"])
        with np.errstate(divide="ignore", invalid="ignore"):
            wt["WaldStatistic"] = wt["betaMatrix"] / wt["betaSE"]
        wt.update(WaldPvalue=waldPvalue(wt["WaldStatistic"], tdf), deviance=-2.0 * wt["logLike"])
        cooks = calculateCooksDistance(cnz, gp["mu"], gp["H"], sizeFactors, x)             # MLE mu / H (R/core.R:1416-1460)
        prior = {"betaPriorVar": gp["betaPriorVar"], "modelMatrix": gp["modelMatrix"]}
    else:
        wt = nbinomWaldTest(cnz, nf, x, mp["dispersion"], engine=engine, useOptim=useOptim, minmu=minmu,
                            weights=wnz, tdf=tdf)
        cooks = calculateCooksDistance(cnz, wt["mu"], wt["hat_diagonals"], sizeFactors, x)  # R/core.R:1457-1460
    per_gene = {"baseMean": mv["baseMean"], "dispGeneEst": ge["dispGeneEst"], "dispFit": tf["dispFit"],
                "dispMAP": mp["dispMAP"], "dispersion": mp["dispersion"], "dispOutlier": mp["dispOutlier"].astype(float),
                "betaMatrix": wt["betaMatrix"], "betaSE": wt["betaSE"], "WaldStatistic": wt["WaldStatistic"],
                "WaldPvalue": wt["WaldPvalue"], "betaConv": wt["betaConv"].astype(float), "betaIter": wt["betaIter"],
                "deviance": wt["deviance"], "dispGeneIter": ge["dispGeneIter"].astype(float),
                "dispIter": mp["dispIter"].astype(float), "maxCooks": recordMaxCooks(x, cooks)}
    if betaPrior:
        per_gene["mleBetaMatrix"] = gp["mleBetaMatrix"]
    if tdf is not None:
        per_gene["tDegreesFreedom"] = tdf
    if test == "LRT":
        red = fitReducedModel(cnz, nf, reduced, mp["dispersion"], engine=engine, minmu=minmu, useOptim=useOptim,
                              weights=wnz)
        df = p - reduced.shape[1]
        per_gene["LRTStatistic"], per_gene["LRTPvalue"] = lrtStatistic(wt["logLike"], red["logLike"], df)
        per_gene["reducedBetaConv"] = red["betaConv"].astype(float)
    extra = dict(prior)
    if np.isfinite(minReplicatesForReplace) and nOrMoreInCell(x, minReplicatesForReplace).any():
        # ---- refitWithoutOutliers (R/core.R:2484-2565) on the rows that had a count replaced
        newc, replace, replaceable = replaceOutliers(cnz, cooks, sizeFactors, x, minReplicates=minReplicatesForReplace)
        nrefit = int(replace.sum())
        newAllZero = replace & (newc.sum(axis=1) == 0)
        if nrefit > 0:
            mvNew = getBaseMeansAndVariances(newc, sizeFactors)
            per_gene["baseMean"] = mvNew["baseMean"]
        if nrefit > 0 and nrefit > int(newAllZero.sum()):
            rr = replace & ~newAllZero
            sub = newc[rr]
            sfSub = sizeFactors[rr] if sizeFactors.ndim == 2 else sizeFactors
            ge2 = estimateDispersionsGeneEst(sub, sfSub, x, engine=engine)
            dispFit2 = tf["coefs"][0] + tf["coefs"][1] / ge2["baseMean"]       # dispersionFunction(object)(baseMean)
            mp2 = estimateDispersionsMAP(sub, x, ge2["mu"], ge2["dispGeneEst"], dispFit2, dispPriorVar,
                                         tf["varLogDispEsts"], engine=engine)
            wt2 = nbinomWaldTest(sub, np.broadcast_to(_div(sfSub), sub.shape), x, mp2["dispersion"],
                                 engine=engine, useOptim=useOptim)
            upd = {"dispGeneEst": ge2["dispGeneEst"], "dispFit": dispFit2, "dispMAP": mp2["dispMAP"],
                   "dispersion": mp2["dispersion"], "dispOutlier": mp2["dispOutlier"].astype(float),
                   "betaMatrix": wt2["betaMatrix"], "betaSE": wt2["betaSE"], "WaldStatistic": wt2["WaldStatistic"],
                   "WaldPvalue": wt2["WaldPvalue"], "betaConv": wt2["betaConv"].astype(float),
                   "betaIter": wt2["betaIter"], "deviance": wt2["deviance"],
                   "dispGeneIter": ge2["dispGeneIter"].astype(float), "dispIter": mp2["dispIter"].astype(float)}
            resultsCols = ["betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "betaConv", "betaIter", "deviance"]
            if tdf is not None:                                                  # kept for rr, a "results" column
                resultsCols.append("tDegreesFreedom")
            if test == "LRT":                                                    # nbinomLRT(objectSub) (:2530-2531)
                red2 = fitReducedModel(sub, np.broadcast_to(_div(sfSub), sub.shape), reduced, mp2["dispersion"],
                                       engine=engine, useOptim=useOptim)
                upd["LRTStatistic"], upd["LRTPvalue"] = lrtStatistic(wt2["logLike"], red2["logLike"], df)
                upd["reducedBetaConv"] = red2["betaConv"].astype(float)
                resultsCols += ["LRTStatistic", "LRTPvalue", "reducedBetaConv"]
            for k, v in upd.items():
                per_gene[k] = per_gene[k].copy()
                per_gene[k][rr] = v
            for k in resultsCols:
                per_gene[k][newAllZero] = np.nan                                 # "results" columns (:2534)
            if replaceable.all():
                per_gene["maxCooks"] = np.full(len(cnz), np.nan)
            else:
                rc = cooks.copy()
                rc[:, replaceable] = 0.0
                per_gene["maxCooks"] = recordMaxCooks(x, rc)
        full_counts = counts.copy()
        full_counts[nz] = newc
        rep_all = np.zeros(N, bool)
        rep_all[nz] = replace
        extra = {"replace": rep_all, "replaceable": replaceable, "replaceCounts": full_counts, "n_replaced": nrefit}

    def full(v):
        out = np.full((N,) + v.shape[1:], np.nan)
        out[nz] = v
        return out

    res = {k: full(np.asarray(v, dtype=np.float64)) for k, v in per_gene.items()}
    res.update({"sizeFactors": None if sfAll.ndim == 2 else sfAll, "allZero": mvAll["allZero"], "dispPriorVar": dispPriorVar,
                "varLogDispEsts": tf["varLogDispEsts"], "n_refit_geneest": ge["n_refit"],
                "n_refit_map": mp["n_refit"], "fitType": fitType, "test": test})
    if test == "LRT":
        res.update(df=df, fullBetaConv=res["betaConv"], reducedModelMatrix=reduced)
    if fitType == "mean":
        res["meanDisp"] = tf["meanDisp"]
    else:
        res["trendCoefs"] = tf["coefs"]
    if sfIterate is not None:
        res["sfIterate"] = {"iterations": sfIterate["iterations"], "evaluations": sfIterate["evaluations"]}
    res["baseMean"] = np.where(nz, res["baseMean"], 0.0)
    if weights is not None:
        res["baseMean"] = np.where(mvAll["allZero"], 0.0, mvAll["baseMean"])    # weightsFail rows keep theirs
        res["weightsFail"] = weightsFail
        res["weights"] = wnz
        res["idx"] = np.flatnonzero(nz)
    if sfAll.ndim == 2:
        res["normalizationFactors"] = sfAll
        res["idx"] = np.flatnonzero(nz)
    res.update(extra)
    return res


def vstSubsetPositions(L, nsub):
    """The 0-based positions, into order(baseMean) of the L genes with baseMean > 5, of the nsub genes vst() fits its
    dispersion function on (R/vst.R:244-247): round(seq(from = 1, to = L, length.out = nsub)).  seq.default gives
    c(1, 1 + k ((L - 1) / (nsub - 1)) for k = 1 .. nsub - 2, L) (c(1, L) for nsub = 2, 1 for nsub = 1), and round()
    rounds half to even (L = 4, nsub = 3: 1, 2.5, 4 -> 1, 2, 4).  The one statement of this rule: the host mirror and
    the device path both use it."""
    L, nsub = int(L), int(nsub)
    if not 1 <= nsub <= L:
        raise ValueError(f"nsub={nsub} must lie in [1, {L}]")
    if nsub == 1:
        pos = np.array([1.0])
    elif nsub == 2:
        pos = np.array([1.0, float(L)])
    else:
        pos = np.r_[1.0, 1.0 + np.arange(1, nsub - 1) * ((L - 1.0) / (nsub - 1.0)), float(L)]
    return np.round(pos).astype(np.int64) - 1


def getVarianceStabilizedData(counts, sizeFactors, dispersionFunction):
    """R/vst.R:145-196 for fitType "parametric" ({"fitType", "trendCoefs": (asymptDisp, extraPois)}) and "mean"
    ({"fitType", "meanDisp"}), in R's operand order, on counts / sizeFactors (an (m,) vector or an (n, m) nf
    matrix).  "local" has no trend fit here: ValueError."""
    q = np.asarray(counts, dtype=np.float64) / _div(sizeFactors)
    fitType = dispersionFunction.get("fitType")
    if fitType == "parametric":
        a0, a1 = (float(v) for v in np.asarray(dispersionFunction["trendCoefs"], dtype=np.float64)[:2])
        return np.log((1 + a1 + 2 * a0 * q + 2 * np.sqrt(a0 * q * (1 + a1 + a0 * q))) / (4 * a0)) / np.log(2)
    if fitType == "mean":
        alpha = float(dispersionFunction["meanDisp"])
        return (2 * np.arcsinh(np.sqrt(alpha * q)) - np.log(alpha) - np.log(4)) / np.log(2)
    raise ValueError(f"fitType {fitType!r}: only 'parametric' and 'mean' dispersion functions are supported")


def _fitDispersionFunction(counts, sizeFactors, x, fitType, engine):
    """estimateDispersionsGeneEst + estimateDispersionsFit (quiet, defaults) on rows none of which is all zero."""
    ge = estimateDispersionsGeneEst(counts, sizeFactors, x, engine=engine)
    tf = estimateDispersionsFit(ge["dispGeneEst"], ge["baseMean"], fitType=fitType)
    if fitType == "mean":
        return {"fitType": "mean", "meanDisp": float(tf["meanDisp"])}
    return {"fitType": "parametric", "trendCoefs": tf["coefs"]}


def _vstDesign(x, m, blind):
    if blind:
        return np.ones((m, 1))
    if x is None:
        raise ValueError("blind=False needs the design x or a dispersionFunction")
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 2 or x.shape[0] != m:
        raise ValueError(f"x must be a design matrix with one row per sample ({m}), got shape {x.shape}")
    return x


def _vstResult(counts, sizeFactors, fn):
    return dict(fn, vst=getVarianceStabilizedData(counts, sizeFactors, fn), sizeFactors=sizeFactors)


def varianceStabilizingTransformation(counts, x=None, blind=True, fitType="parametric", sizeFactors=None,
                                      dispersionFunction=None, engine=None):
    """R/vst.R:112-142.  sizeFactors: (m,) or an (n, m) nf matrix; estimated (ratio) when None.  The dispersion
    function is fitted on the non-all-zero rows (design ~1 when blind, x otherwise) unless blind=False and
    dispersionFunction is given.  Returns {"vst", the dispersion keys, "sizeFactors"}."""
    counts = np.asarray(counts)
    m = counts.shape[1]
    if sizeFactors is None:
        sizeFactors = estimateSizeFactorsForMatrix(counts)
    if blind or dispersionFunction is None:
        x = _vstDesign(x, m, blind)
        nz = counts.sum(axis=1) > 0
        sf = np.asarray(sizeFactors, dtype=np.float64)
        dispersionFunction = _fitDispersionFunction(counts[nz], sf[nz] if sf.ndim == 2 else sf, x, fitType, engine)
    return _vstResult(counts, sizeFactors, dispersionFunction)


def vst(counts, x=None, blind=True, nsub=1000, fitType="parametric", sizeFactors=None, engine=None):
    """R/vst.R:219-267: the dispersion function fitted on nsub genes with baseMean > 5 (vstSubsetPositions of a stable
    ordering of baseMean, in that row order), then the VST of all rows.  Returns varianceStabilizingTransformation's
    dict plus "subset" (the row indices, in fit order)."""
    counts = np.asarray(counts)
    n, m = counts.shape
    if n < nsub:
        raise ValueError("less than 'nsub' rows, it is recommended to use varianceStabilizingTransformation directly")
    if sizeFactors is None:
        sizeFactors = estimateSizeFactorsForMatrix(counts)
    sf = np.asarray(sizeFactors, dtype=np.float64)
    baseMean = (counts / _div(sf)).mean(axis=1)
    keep = np.flatnonzero(baseMean > 5)
    if len(keep) < nsub:
        raise ValueError("less than 'nsub' rows with mean normalized count > 5, it is recommended to use "
                         "varianceStabilizingTransformation directly")
    o = np.argsort(baseMean[keep], kind="stable")
    subset = keep[o[vstSubsetPositions(len(keep), nsub)]]
    fn = _fitDispersionFunction(counts[subset], sf[subset] if sf.ndim == 2 else sf, _vstDesign(x, m, blind),
                                fitType, engine)
    return dict(_vstResult(counts, sizeFactors, fn), subset=subset)


def normTransform(counts, sizeFactors=None, pc=1.0):
    """R/helper.R:421-435 with f = log2: log2(counts / sizeFactors + pc); sizeFactors (m,) or (n, m), estimated
    (ratio) when None."""
    if sizeFactors is None:
        sizeFactors = estimateSizeFactorsForMatrix(counts)
    return np.log2(np.asarray(counts, dtype=np.float64) / _div(sizeFactors) + pc)


def sparseTest(normCounts, p=0.9, t1=100, t2=0.1):
    """R/rlog.R:274-287: warns when, among the rows whose sum of normalized counts exceeds t1, more than a fraction t2
    have one sample holding more than p of the row sum."""
    import warnings
    rs = normCounts.sum(axis=1)
    rmx = normCounts.max(axis=1)
    if np.all(rs <= t1):
        return
    total = np.mean((rmx / rs)[rs > t1] > p)
    if total > t2:
        warnings.warn(f"the rlog assumes that data is close to a negative binomial distribution: for "
                      f"{round(total, 3) * 100}% of genes with a sum of normalized counts above {t1}, a single "
                      f"sample's normalized count made up more than {p * 100}% of the sum", stacklevel=3)


def rlogData(counts, sizeFactors, dispFit, baseMean, intercept=None, betaPriorVar=None, engine=None):
    """R/rlog.R:172-272.  sizeFactors: (m,) or an (n, m) nf matrix; dispFit, baseMean: (n,).  The design is
    [1 | I_m] with lambda = (1e-6, 1 / betaPriorVar, ...) or, with a frozen intercept (n log2 values), I_m on
    nf 2^intercept; rows that are all zero (or whose intercept is not finite) are left out and get 0.  betaPriorVar,
    when None, is matchWeightedUpperQuantileForVariance of the log fold changes over an intercept.  One fitNbinomGLMs
    call (betaTol = 1e-4, useQR, useOptim = FALSE).  Returns {"rlog", "betaPriorVar", "intercept" (None when frozen),
    "betaIter"}."""
    counts = np.asarray(counts)
    n, m = counts.shape
    nf = np.broadcast_to(_div(sizeFactors), (n, m)).astype(np.float64)
    dispFit = np.asarray(dispFit, dtype=np.float64)
    baseMean = np.asarray(baseMean, dtype=np.float64)
    if intercept is None:
        allZero = counts.sum(axis=1) == 0
        x = np.c_[np.ones(m), np.eye(m)]            # model.matrix(~samples)[-1, ] with a "null_level" row first
    else:
        intercept = np.array(intercept, dtype=np.float64).reshape(-1)
        if len(intercept) != n:
            raise ValueError("intercept should be as long as the number of rows of object")
        infiniteIntercept = ~np.isfinite(intercept)
        intercept[infiniteIntercept] = -10.0
        nf = nf * 2.0 ** intercept[:, None]
        allZero = infiniteIntercept
        x = np.eye(m)
    nz = ~allZero
    if np.any(np.isnan(dispFit[nz])):
        raise ValueError("dispFit is NA on a row the rlog fits")
    if betaPriorVar is None:
        logFoldChangeMatrix = np.log2(counts[nz] / nf[nz] + 0.5) - np.log2(baseMean[nz] + 0.5)[:, None]
        weights = 1.0 / (1.0 / baseMean[nz] + dispFit[nz])
        betaPriorVar = matchWeightedUpperQuantileForVariance(logFoldChangeMatrix.ravel(order="F"), np.tile(weights, m))
    lam = np.full(x.shape[1], 1.0 / betaPriorVar)
    if intercept is None:
        lam[0] = 1e-6
    fit = fitNbinomGLMs(counts[nz], nf[nz], x, dispFit[nz], lambda_=lam, engine=engine, betaTol=1e-4, useQR=True,
                        useOptim=False)
    out = np.zeros((n, m))
    out[nz] = fit["betaMatrix"] @ x.T
    it = np.zeros(n)
    it[nz] = fit["betaIter"]
    res = {"betaPriorVar": betaPriorVar, "betaIter": it, "intercept": None}
    if intercept is not None:
        out = out + np.where(allZero, 0.0, intercept)[:, None]
    else:
        icpt = np.full(n, -np.inf)
        icpt[nz] = fit["betaMatrix"][:, 0]
        res["intercept"] = icpt
    res["rlog"] = out
    return res


def rlog(counts, x=None, blind=True, intercept=None, betaPriorVar=None, fitType="parametric", sizeFactors=None,
         dispFit=None, engine=None):
    """R/rlog.R:108-164 for a count matrix.  sizeFactors: (m,) or an (n, m) nf matrix, estimated (ratio) when None.
    sparseTest runs when no intercept is given.  With blind=True or without dispFit, the dispersion function is
    fitted on the non-all-zero rows (design ~1 when blind, x otherwise) and dispFit is it at baseMean.  Returns
    rlogData's dict plus "dispFit", "sizeFactors" and the dispersion keys when they were estimated."""
    counts = np.asarray(counts)
    m = counts.shape[1]
    if sizeFactors is None:
        sizeFactors = estimateSizeFactorsForMatrix(counts)
    sf = np.asarray(sizeFactors, dtype=np.float64)
    norm = counts / _div(sf)
    if intercept is None:
        sparseTest(norm)
    baseMean = norm.mean(axis=1)
    extra = {}
    if blind or dispFit is None:
        if not blind and x is None:
            raise ValueError("blind=False needs the design x or dispFit")
        nz = counts.sum(axis=1) > 0
        extra = _fitDispersionFunction(counts[nz], sf[nz] if sf.ndim == 2 else sf, _vstDesign(x, m, blind), fitType,
                                       engine)
        with np.errstate(divide="ignore"):
            if fitType == "mean":
                dispFit = np.full(len(counts), extra["meanDisp"])
            else:
                a = np.asarray(extra["trendCoefs"], dtype=np.float64)
                dispFit = a[0] + a[1] / baseMean
    res = rlogData(counts, sf, dispFit, baseMean, intercept=intercept, betaPriorVar=betaPriorVar, engine=engine)
    res.update(extra)
    res.update(dispFit=np.asarray(dispFit, dtype=np.float64), sizeFactors=sizeFactors)
    return res


# ---------------------------------------------------------------- results() and pvalueAdjustment() (R/results.R)

P_ADJUST_METHODS = ("BH", "fdr", "BY", "holm", "hochberg", "bonferroni", "none")
ALT_HYPOTHESES = ("greaterAbs", "lessAbs", "greater", "less", "greaterAbs2014")


def quantile7(x, probs):
    """quantile(x, probs, type = 7) (R's quantile.default): index = 1 + (n - 1) p, lo = floor(index); x[lo], replaced by
    (1 - h) x[lo] + h x[hi] (h = index - lo, hi = ceiling(index)) only where index > lo and x[hi] != x[lo].  numpy's
    default lerp is another formula.  x must not contain NaN (R stops)."""
    x = np.sort(np.asarray(x, dtype=np.float64))
    probs = np.atleast_1d(np.asarray(probs, dtype=np.float64))
    n = len(x)
    index = 1.0 + max(n - 1, 0) * probs
    lo = np.floor(index)
    hi = np.ceil(index)
    qs = x[lo.astype(np.int64) - 1]
    xhi = x[hi.astype(np.int64) - 1]
    i = (index > lo) & (xhi != qs)
    h = (index - lo)[i]
    qs = qs.copy()
    qs[i] = (1.0 - h) * qs[i] + h * xhi[i]
    return qs


def p_adjust(p, method="BH"):
    """R's p.adjust(p, method) restated literally (stats/R/p.adjust.R).  NaN is NA: it stays NaN and does not count;
    n = the number of non-NA p-values (the lazy default n = length(p) is forced after the NAs are dropped).  hommel is
    not supported (ValueError)."""
    if method == "fdr":
        method = "BH"
    if method not in ("BH", "BY", "holm", "hochberg", "bonferroni", "none"):
        raise ValueError(f"p.adjust method {method!r} is not supported (BH/fdr, BY, holm, hochberg, bonferroni, none)")
    p0 = np.array(p, dtype=np.float64)
    nna = ~np.isnan(p0)
    p = p0[nna]
    lp = len(p)
    n = lp
    if n <= 1:
        return p0
    with np.errstate(over="ignore"):
        if method == "bonferroni":
            v = np.minimum(1.0, n * p)
        elif method == "holm":
            i = np.arange(1, lp + 1)
            o = np.argsort(p, kind="stable")
            v = np.empty(lp)
            v[o] = np.minimum(1.0, np.maximum.accumulate((n - i + 1) * p[o]))
        elif method in ("hochberg", "BH", "BY"):
            i = np.arange(lp, 0, -1)
            o = np.argsort(-p, kind="stable")                     # order(p, decreasing = TRUE)
            if method == "hochberg":
                t = (n + 1 - i) * p[o]
            elif method == "BH":
                t = n / i * p[o]
            else:
                q = float(np.sum(1.0 / np.arange(1, n + 1)))
                t = q * n / i * p[o]
            v = np.empty(lp)
            v[o] = np.minimum(1.0, np.minimum.accumulate(t))
        else:
            v = p
    p0[nna] = v
    return p0


def _lowest(x, y, n, xs, nleft, nright, w, userw, rw):
    """clowess' local fit at xs from the points nleft..nright (1-based, ties on the right picked up); returns (ys, ok)."""
    rng = x[n] - x[1]
    h = max(xs - x[nleft], x[nright] - xs)
    h9, h1 = 0.999 * h, 0.001 * h
    a = 0.0
    j = nleft
    while j <= n:
        w[j] = 0.0
        r = abs(x[j] - xs)
        if r <= h9:
            w[j] = 1.0 if r <= h1 else (1.0 - (r / h) ** 3) ** 3
            if userw:
                w[j] *= rw[j]
            a += w[j]
        elif x[j] > xs:
            break
        j += 1
    nrt = j - 1
    if a <= 0.0:
        return 0.0, False
    for j in range(nleft, nrt + 1):
        w[j] /= a
    if h > 0.0:
        a = 0.0
        for j in range(nleft, nrt + 1):
            a += w[j] * x[j]
        b = xs - a
        c = 0.0
        for j in range(nleft, nrt + 1):
            c += w[j] * (x[j] - a) * (x[j] - a)
        if np.sqrt(c) > 0.001 * rng:
            b /= c
            for j in range(nleft, nrt + 1):
                w[j] *= (b * (x[j] - a) + 1.0)
    ys = 0.0
    for j in range(nleft, nrt + 1):
        ys += w[j] * y[j]
    return ys, True


def lowess(x, y, f=2.0 / 3.0, iter=3, delta=None):
    """R's lowess(x, y, f, iter, delta = 0.01 * diff(range(x))): the points sorted by x, then clowess (Cleveland 1979,
    R's src/library/stats/src/lowess.c) restated: tricube-weighted local linear fits over the ns = max(2, min(n,
    floor(f n + 1e-7))) nearest points, points within delta of the last fit interpolated, and `iter` robustness
    passes with bisquare weights of the residuals over 6 MAD.  Returns {"x": sorted x, "y": fitted values}."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    o = np.argsort(x, kind="stable")
    x, y = x[o], y[o]
    n = len(x)
    if delta is None:
        delta = 0.01 * (x[-1] - x[0]) if n else 0.0
    if n < 2:
        return {"x": x, "y": y.copy()}
    X = np.r_[0.0, x]                                           # 1-based, as the C code
    Y = np.r_[0.0, y]
    ys = np.zeros(n + 1)
    rw = np.zeros(n + 1)
    res = np.zeros(n + 1)
    ns = max(2, min(n, int(f * n + 1e-7)))
    it = 1
    while it <= iter + 1:
        nleft, nright, last, i = 1, ns, 0, 1
        while True:
            if nright < n:
                d1 = X[i] - X[nleft]
                d2 = X[nright + 1] - X[i]
                if d1 > d2:
                    nleft += 1
                    nright += 1
                    continue
            v, ok = _lowest(X, Y, n, X[i], nleft, nright, res, it > 1, rw)
            ys[i] = v if ok else Y[i]
            if last < i - 1:
                denom = X[i] - X[last]
                for j in range(last + 1, i):
                    alpha = (X[j] - X[last]) / denom
                    ys[j] = alpha * ys[i] + (1.0 - alpha) * ys[last]
            last = i
            cut = X[last] + delta
            i = last + 1
            while i <= n:
                if X[i] > cut:
                    break
                if X[i] == X[last]:
                    ys[i] = ys[last]
                    last = i
                i += 1
            i = max(last + 1, i - 1)
            if last >= n:
                break
        res[1:] = Y[1:] - ys[1:]
        sc = float(np.sum(np.abs(res[1:]))) / n
        if it > iter:
            break
        r = np.abs(res[1:])
        s = np.sort(r)
        m1 = n // 2
        cmad = 3.0 * (s[m1] + s[n - m1 - 1]) if n % 2 == 0 else 6.0 * s[m1]
        if cmad < 1e-7 * sc:
            break
        c9, c1 = 0.999 * cmad, 0.001 * cmad
        with np.errstate(divide="ignore", invalid="ignore"):     # cmad = 0: every r <= c1, the quotient is unused
            rw[1:] = np.where(r <= c1, 1.0, np.where(r <= c9, (1.0 - (r / cmad) ** 2) ** 2, 0.0))
        it += 1
    return {"x": x, "y": ys[1:].copy()}


def filtered_p(filter, test, theta, method="none"):
    """filtered_p (R/results.R:721-740) with a filter vector: the n x len(theta) matrix of p.adjust over the genes with
    filter >= quantile(filter, theta[i]) (NA elsewhere)."""
    filter = np.asarray(filter, dtype=np.float64)
    test = np.asarray(test, dtype=np.float64)
    cutoffs = quantile7(filter, theta)
    result = np.full((len(filter), len(cutoffs)), np.nan)
    for i, c in enumerate(cutoffs):
        use = filter >= c
        if use.any():
            result[use, i] = p_adjust(test[use], method)
    return result


def filter_default_theta(filter):
    """pvalueAdjustment's default theta: seq(mean(filter == 0), .95 or 1, length = 50), R's seq.default: the end
    points exact, the interior lo + k * ((hi - lo) / 49)."""
    lo = float(np.mean(np.asarray(filter) == 0))
    hi = 0.95 if lo < 0.95 else 1.0
    by = (hi - lo) / 49.0
    theta = lo + np.arange(50) * by
    theta[-1] = hi
    return theta


def filter_choose(numRej, fit_y):
    """pvalueAdjustment's choice of the theta index j (R/results.R:662-692), 0-based."""
    numRej = np.asarray(numRej, dtype=np.float64)
    if np.max(numRej) <= 10:
        return 0
    residual = 0.0 if np.all(numRej == 0) else numRej[numRej > 0] - fit_y[numRej > 0]
    maxFit = np.max(fit_y)
    rmse = np.sqrt(np.mean(np.asarray(residual) ** 2))
    thresh = maxFit - rmse
    for cond in (numRej > thresh, numRej > 0.9 * maxFit, numRej > 0.8 * maxFit):
        if cond.any():
            return int(np.flatnonzero(cond)[0])
    return 0


def check_filter_args(N, filter, theta, alpha, pAdjustMethod):
    """pvalueAdjustment's stops and this restatement's limits, shared by the host mirror and the device path.  Returns
    (filter as float64 numpy or None, theta as float64 numpy or None)."""
    if not (0.0 < alpha < 1.0):
        raise ValueError("alpha must be in (0, 1)")
    if pAdjustMethod not in P_ADJUST_METHODS:
        raise ValueError(f"pAdjustMethod {pAdjustMethod!r} is not supported (hommel and others are out of scope): "
                         f"use one of {', '.join(P_ADJUST_METHODS)}")
    if callable(filter):
        raise ValueError("a filter function is not supported: pass the filter values")
    if filter is not None:
        filter = np.asarray(filter.cpu() if hasattr(filter, "cpu") else filter, dtype=np.float64).reshape(-1)
        if len(filter) != N:
            raise ValueError(f"filter must have one value per row ({N}), got {len(filter)}")
        if np.isnan(filter).any():
            raise ValueError("missing values are not allowed in the filter")
    if theta is not None:
        theta = np.asarray(theta, dtype=np.float64).reshape(-1)
        if len(theta) < 2:
            raise ValueError("theta must have length > 1")
        if not np.all((theta >= 0) & (theta <= 1)):
            raise ValueError("theta must be probabilities in [0, 1]")
    return filter, theta


def pvalueAdjustment(pvalue, baseMean, independentFiltering=True, filter=None, theta=None, alpha=0.1,
                     pAdjustMethod="BH"):
    """pvalueAdjustment (R/results.R:638-718): returns (padj, metadata)."""
    N = len(pvalue)
    filter, theta = check_filter_args(N, filter, theta, alpha, pAdjustMethod)
    meta = {"alpha": alpha}
    if not independentFiltering:
        return p_adjust(pvalue, pAdjustMethod), meta
    if filter is None:
        filter = np.asarray(baseMean, dtype=np.float64)
    if theta is None:
        theta = filter_default_theta(filter)
    filtPadj = filtered_p(filter, pvalue, theta, pAdjustMethod)
    numRej = np.sum(filtPadj < alpha, axis=0)
    lo_fit = lowess(theta, numRej, f=1.0 / 5.0)
    j = filter_choose(numRej, lo_fit["y"])
    cutoffs = quantile7(filter, theta)
    meta.update(filterThreshold=float(cutoffs[j]), filterTheta=float(theta[j]), filterNumRej={"theta": theta,
                "numRej": numRej.astype(np.int64)}, lo_fit=lo_fit, j=j, cutoffs=cutoffs)
    return filtPadj[:, j].copy(), meta


def _column_names(x, factors, expanded):
    if factors is None:
        return None
    return factorDesign(factors, expanded=expanded)[1]


def _col_index(name, names, p):
    if isinstance(name, (bool, np.bool_)) or not isinstance(name, (int, np.integer, str)):
        raise ValueError("the argument 'name' should be a column index or one column name")
    if isinstance(name, str):
        if names is None or name not in names:
            raise ValueError(f"name {name!r} is not a column of the model matrix")
        return names.index(name)
    if not 0 <= int(name) < p:
        raise ValueError(f"column index {name} out of range (p = {p})")
    return int(name)


def resultsSelection(x, name=None, contrast=None, listValues=(1, -1), factors=None, betaPrior=False,
                     modelMatrix=None):
    """cleanContrast / getCoef (R/results.R:389-463, 832-1040): which column results() reports.  Returns a dict:
    {"kind": "coef", "col": k, "negate": bool} (a coefficient of the fitted matrix, negated when the numerator is the
    reference level) or {"kind": "contrast", "vec": numeric contrast over the fitted matrix's columns}, each with
    "mask": the samples of contrastAllZero (a bool (m,) array) or None.  Contrasts: `(k, num, den)` (a tuple of three
    ints: factor k of `factors`, numerator and denominator level codes), a list `[numerator names, denominator names]`
    (column names of factorDesign, weighted by listValues), or a numeric vector.  With betaPrior the fitted matrix is
    `modelMatrix` (the expanded one) and, without name and contrast, the default is the last factor's last level vs its
    first."""
    x = np.asarray(x, dtype=np.float64)
    xf = np.asarray(modelMatrix, dtype=np.float64) if betaPrior else x
    p = xf.shape[1]
    names = _column_names(x, factors, betaPrior)
    lv = np.asarray(listValues, dtype=np.float64)
    if lv.shape != (2,) or not (lv[0] > 0 and lv[1] < 0):
        raise ValueError("listValues must be two numbers, the first positive and the second negative")
    if betaPrior and contrast is None and name is None:
        f = np.asarray(factors[-1])
        contrast = (len(factors) - 1, int(f.max()), 0)
    if contrast is None:
        k = p - 1 if name is None else _col_index(name, names, p)
        return {"kind": "coef", "col": k, "negate": False, "mask": None}
    if isinstance(contrast, tuple) and len(contrast) == 3 and all(isinstance(v, (int, np.integer)) for v in contrast):
        if factors is None:
            raise ValueError("a factor-level contrast needs the design factors (factors=...)")
        k, num, den = (int(v) for v in contrast)
        if not 0 <= k < len(factors):
            raise ValueError(f"{k} should be the index of a factor of the design")
        f = np.asarray(factors[k])
        nlev = int(f.max()) + 1
        if num == den:
            raise ValueError(f"{num} and {den} should be different level names")
        if not (0 <= num < nlev and 0 <= den < nlev):
            raise ValueError(f"{num} and {den} should be levels of factor {k}")
        mask = np.isin(f, (num, den))
        _, _, fidx, lvl = factorDesign(factors, expanded=betaPrior)
        col = {int(l): c for c, (fi, l) in enumerate(zip(fidx, lvl)) if fi == k}
        if not betaPrior and den == 0:
            return {"kind": "coef", "col": col[num], "negate": False, "mask": mask}
        if not betaPrior and num == 0:
            return {"kind": "coef", "col": col[den], "negate": True, "mask": mask}
        vec = np.zeros(p)
        vec[col[num]] = 1.0
        vec[col[den]] = -1.0
        return {"kind": "contrast", "vec": vec, "mask": mask}
    if isinstance(contrast, list):
        if len(contrast) == 1:
            contrast = [contrast[0], []]
        if len(contrast) != 2:
            raise ValueError("'contrast', as a list, should have length 2, or, if length 1, an empty vector will be "
                             "added for the second element")
        num, den = ([v] if isinstance(v, str) else list(v) for v in contrast)
        if not all(isinstance(v, str) for v in num + den):
            raise ValueError("'contrast', as a list of length 2, should have column names as elements")
        if names is None or not all(v in names for v in num + den):
            raise ValueError("all elements of the contrast as a list of length 2 should be column names of the model "
                             "matrix")
        if set(num) & set(den):
            raise ValueError("elements in the contrast list should only appear in the numerator or the denominator, "
                             "but not both")
        if not num + den:
            raise ValueError("one of the two elements in the list should be a character vector of non-zero length")
        vec = np.zeros(p)
        vec[[names.index(v) for v in num]] = lv[0]
        vec[[names.index(v) for v in den]] = lv[1]
    else:
        if isinstance(contrast, (bool, np.bool_, str)) or isinstance(contrast, tuple):
            raise ValueError("'contrast' should be a (factor, numerator level, denominator level) tuple, a list of "
                             "two lists of column names, or a numeric vector")
        vec = np.asarray(contrast, dtype=np.float64).reshape(-1)
        if len(vec) != p:
            raise ValueError("numeric contrast vector should have one element for every column of the model matrix")
        if np.all(vec == 0):
            raise ValueError("numeric contrast vector cannot have all elements equal to 0")
    mask = None
    if not (np.all(vec >= 0) or np.all(vec <= 0)):          # contrastAllZeroNumeric (R/results.R:1248-1270)
        mask = (xf @ (vec != 0).astype(np.float64)) != 0
    return {"kind": "contrast", "vec": vec, "mask": mask}


def results_checks(lfcThreshold, altHypothesis, lrt, betaPrior, alpha, useT=False):
    """results()' stops (R/results.R:318-345, 465-470) and this restatement's limits."""
    if useT:
        raise ValueError("useT is not supported (there are no t degrees of freedom)")
    if altHypothesis not in ALT_HYPOTHESES:
        raise ValueError(f"altHypothesis must be one of {', '.join(ALT_HYPOTHESES)}")
    if not (np.isfinite(lfcThreshold) and lfcThreshold >= 0):
        raise ValueError("lfcThreshold must be finite and >= 0")
    if not (0.0 < alpha < 1.0):
        raise ValueError("alpha must be in (0, 1)")
    if lfcThreshold == 0 and altHypothesis == "lessAbs":
        raise ValueError("when testing altHypothesis='lessAbs', set the argument lfcThreshold to a positive value")
    thresholded = not (lfcThreshold == 0 and altHypothesis == "greaterAbs")
    if thresholded and lrt:
        raise ValueError("tests of log fold change above or below a theshold must be Wald tests")
    if thresholded and altHypothesis == "lessAbs" and betaPrior:
        raise ValueError("testing altHypothesis='lessAbs' requires setting the DESeq() argument betaPrior=FALSE")
    return thresholded


def r_pnorm_upper(q):
    """pnorm(q, lower.tail = FALSE)."""
    from scipy import stats as _st
    return _st.norm.sf(q)


def thresholdTest(LFC, SE, T, altHypothesis, df=None):
    """results()' lfcThreshold / altHypothesis step (R/results.R:464-518, pnorm; pnorm(q, sd = se) = pnorm(q / se)).
    df: the genes' t degrees of freedom (useT: pt(q, df) in place of pnorm).  Returns (stat, pvalue)."""
    from scipy import stats as _st
    up = r_pnorm_upper if df is None else (lambda q: r_pt_upper(q, df))
    low = _st.norm.cdf if df is None else (lambda q: r_pt_upper(-q, df))
    with np.errstate(divide="ignore", invalid="ignore"):
        if altHypothesis == "greaterAbs":
            return LFC / SE, low((-np.abs(LFC) + T) / SE) + low((-np.abs(LFC) - T) / SE)
        if altHypothesis == "greaterAbs2014":
            q = (np.abs(LFC) - T) / SE
            return np.sign(LFC) * np.maximum(q, 0), np.minimum(1.0, 2.0 * up(q))
        if altHypothesis == "lessAbs":
            qa, qb = (T - LFC) / SE, (LFC + T) / SE
            return np.minimum(np.maximum(qa, 0), np.maximum(qb, 0)), np.maximum(up(qa), up(qb))
        if altHypothesis == "greater":
            q = (LFC - T) / SE
            return np.maximum(q, 0), up(q)
        return np.minimum((LFC + T) / SE, 0), up((-T - LFC) / SE)


def results(dds, counts, x, name=None, contrast=None, listValues=(1, -1), lfcThreshold=0.0,
            altHypothesis="greaterAbs", cooksCutoff=None, independentFiltering=True, alpha=0.1, filter=None, theta=None,
            pAdjustMethod="BH", factors=None, lrt=None, minmu=0.5, cooks=None, engine=None, useT=False):
    """results() + pvalueAdjustment() (R/results.R:298-740) on a pipeline.DESeq result `dds` (per-gene arrays over all
    N rows, NaN for all-zero rows) for the (N, m) counts it was run on and its design x.  Arguments as R's (see
    resultsSelection for name / contrast / listValues); factors: the design's level-code vectors (names, factor-level
    contrasts, betaPrior results, the two-group Cook's heuristic); lrt: a nbinomLRT result (full-length LRTStatistic /
    LRTPvalue) whose stat and p replace the Wald ones; cooks: the (N, m) Cook's distances of the first fit, needed by
    the two-group heuristic (a single factor with two levels) when a gene is flagged.  Returns {"baseMean",
    "log2FoldChange", "lfcSE", "stat", "pvalue", "padj"} over all N rows, and "metadata" (filterThreshold,
    filterTheta, filterNumRej, lo_fit, alpha, lfcThreshold, the cutoffs and the chosen index j).
    A dds with "tDegreesFreedom" (DESeq(useT=True)) is tested with t tails as R infers it (R/results.R:414): contrasts
    through getContrast(useT=True) and thresholded tests with pt at each gene's df.  useT=True itself raises, as R's
    results() has no such argument."""
    from scipy import stats as _st
    engine = engine or _default_engine
    counts = np.asarray(counts)
    N, m = counts.shape
    x = np.asarray(x, dtype=np.float64)
    p = x.shape[1]
    betaPrior = "betaPriorVar" in dds and dds.get("modelMatrix") is not None
    thresholded = results_checks(lfcThreshold, altHypothesis, lrt is not None, betaPrior, alpha, useT)
    check_filter_args(N, filter, theta, alpha, pAdjustMethod)
    sel = resultsSelection(x, name, contrast, listValues, factors, betaPrior, dds.get("modelMatrix"))
    nz = ~np.asarray(dds["allZero"], bool)
    if "weightsFail" in dds:
        nz = nz & ~np.asarray(dds["weightsFail"], bool)
    tdf = dds.get("tDegreesFreedom")
    if sel["kind"] == "coef":
        k = sel["col"]
        lfc, se = dds["betaMatrix"][:, k].copy(), dds["betaSE"][:, k].copy()
        stat, pv = dds["WaldStatistic"][:, k].copy(), dds["WaldPvalue"][:, k].copy()
        if sel["negate"]:
            lfc = -lfc
            stat = -stat
    else:
        xf = dds["modelMatrix"] if betaPrior else x
        cts = dds["replaceCounts"] if "replaceCounts" in dds else counts
        if dds.get("normalizationFactors") is not None:
            nf = np.asarray(dds["normalizationFactors"])[nz]
        else:
            nf = np.broadcast_to(dds["sizeFactors"], (int(nz.sum()), m))
        g = getContrast(cts[nz], nf, xf, dds["dispersion"][nz], dds["betaMatrix"][nz], sel["vec"],
                        betaPriorVar=dds.get("betaPriorVar"), engine=engine, minmu=minmu, weights=dds.get("weights"),
                        useT=tdf is not None, df=None if tdf is None else tdf[nz])
        lfc, se, stat, pv = (np.full(N, np.nan) for _ in range(4))
        lfc[nz], se[nz], stat[nz], pv[nz] = g["log2FoldChange"], g["lfcSE"], g["stat"], g["pvalue"]
    if sel["mask"] is not None:
        az = nz & (counts[:, sel["mask"]].sum(axis=1) == 0)
        lfc[az] = 0.0
        stat[az] = 0.0
        pv[az] = 1.0
    if lrt is not None:
        stat = np.asarray(lrt["LRTStatistic"], dtype=np.float64).copy()
        pv = np.asarray(lrt["LRTPvalue"], dtype=np.float64).copy()
    if thresholded:
        stat, pv = thresholdTest(lfc, se, lfcThreshold, altHypothesis, tdf)
    if cooksCutoff is None or cooksCutoff is True:
        cooksCutoff = float(_st.f.ppf(0.99, p, m - p))              # the dispersion design's p and m
    if cooksCutoff is not False:
        with np.errstate(invalid="ignore"):
            out = dds["maxCooks"] > float(cooksCutoff)
        if out.any() and factors is not None and len(factors) == 1 and int(np.max(factors[0])) == 1:
            if cooks is None:
                raise ValueError("the two-group Cook's heuristic needs the Cook's distances (cooks=...)")
            for ii in np.flatnonzero(out):
                row = np.asarray(cooks[ii], dtype=np.float64)
                if np.all(np.isnan(row)):
                    continue
                outCount = counts[ii, int(np.nanargmax(row))]
                if np.sum(counts[ii] > outCount) >= 3:
                    out[ii] = False
        pv[out] = np.nan
    if "replace" in dds and np.nansum(dds["replace"]) > 0:
        nowZero = np.asarray(dds["replace"], bool) & (dds["baseMean"] == 0)
        lfc[nowZero] = se[nowZero] = stat[nowZero] = 0.0
        pv[nowZero] = 1.0
    padj, meta = pvalueAdjustment(pv, dds["baseMean"], independentFiltering, filter, theta, alpha, pAdjustMethod)
    meta["lfcThreshold"] = lfcThreshold
    return {"baseMean": np.asarray(dds["baseMean"], dtype=np.float64), "log2FoldChange": lfc, "lfcSE": se,
            "stat": stat, "pvalue": pv, "padj": padj, "metadata": meta}


# ---------------------------------------------------------------- lfcShrink(type = "normal") (R/lfcShrink.R:145-327)

SHRINK_TYPES = ("normal", "apeglm", "ashr")


def lfcShrink_checks(x, coef, contrast, res_given, lfcThreshold, factors, weighted, betaPrior, type="normal"):
    """lfcShrink()'s stops (R/lfcShrink.R:145-327) and this restatement's limits, shared by lfcShrink and
    device_pipeline.lfcShrink_device.  x: the design DESeq ran on; res_given: whether a results table was passed;
    weighted: whether the DESeq run had observation weights; betaPrior: whether it ran with betaPrior=TRUE.
    Returns (expanded, k): whether the prior is on the expanded model matrix (a contrast) or on x (a coefficient),
    and the coefficient's column of x (None for a contrast)."""
    if type not in SHRINK_TYPES:
        raise ValueError(f"type must be one of {', '.join(SHRINK_TYPES)}")
    if type != "normal":
        raise ValueError(f"type={type!r} calls the {type} package, which is not part of DESeq2: only type='normal' is "
                         "implemented")
    if betaPrior:
        raise ValueError("lfcShrink() should be used downstream of DESeq() with betaPrior=FALSE (the default)")
    if coef is None and contrast is None:
        raise ValueError("type='normal' requires either 'coef' or 'contrast' be specified.")
    if coef is not None and contrast is not None:
        raise ValueError("give either 'coef' or 'contrast', not both")
    if not (np.isfinite(lfcThreshold) and lfcThreshold >= 0):
        raise ValueError("lfcThreshold must be finite and >= 0")
    x = np.asarray(x, dtype=np.float64)
    if not np.all(x[:, 0] == 1):
        raise ValueError("lfcShrink needs a design with an intercept: the first column of x must be all ones")
    if contrast is None:
        names = factorDesign(factors)[1] if factors is not None else None
        return False, _col_index(coef, names, x.shape[1])
    if not isinstance(contrast, (tuple, list)) and not res_given:
        raise ValueError("for type='normal' and numeric contrast, user must provide 'res' object (results=)")
    if factors is None:
        raise ValueError("a contrast is shrunk on the expanded model matrix, which needs the design factors "
                         "(factors=...)")
    if not np.array_equal(x, factorDesign(factors)[0]):
        raise ValueError("user-supplied design matrix supports shrinkage only with 'coef': for a contrast x must be "
                         "the standard model matrix of the factors, factorDesign(factors)[0]")
    if weighted:
        raise ValueError("observation weights are not supported with a contrast (the expanded model matrix is rank "
                         "deficient): shrink a coefficient (coef=) instead")
    return True, None


def lfcShrink(dds, counts, x, coef=None, contrast=None, res=None, lfcThreshold=0, factors=None, engine=None,
              betaTol=1e-8, maxit=100, useOptim=True, minmu=0.5, type="normal", cooks=None):
    """lfcShrink(type = "normal") (R/lfcShrink.R:145-327) on a pipeline.DESeq result dds (betaPrior=False) for the
    (N, m) counts it was run on and its design x.  coef: a column index or factorDesign name of x (the prior is
    estimateBetaPriorVar's "standard" one over x's MLE columns, the MAP fit is on x); contrast: as results() takes it
    with factors, over the expanded matrix's columns (the prior is the expanded one, the MAP fit on
    factorDesign(factors, expanded=True)[0]).  The prior is over the rows that are neither all zero, weightsFail nor
    all zero after an outlier replacement; the MAP fit (fitGLMsWithPrior with the given betaPriorVar) is on their
    ORIGINAL counts, with dds's dispersions and normalised weights.  res: the results table to modify, by default
    results(dds, name=coef) or results(dds, contrast=contrast) (with dds's LRT columns after test="LRT").  The shrunk
    table is results() of the MAP fit with lfcThreshold, minmu and defaults otherwise; its log2FoldChange and lfcSE
    replace res's, and with lfcThreshold > 0 its stat, pvalue and padj too.  Its Cook's cutoff uses the first fit's
    maxCooks without the replaceable-sample zeroing (nbinomWaldTest recomputes it, R/core.R:1452-1460), from cooks:
    the (N, m) Cook's distances of the first fit, needed then and by the two-group heuristic.  Returns res's dict
    with those columns replaced and metadata["priorInfo"] = {"type", "package", "betaPriorVar"}."""
    engine = engine or _default_engine
    counts = np.asarray(counts)
    N, m = counts.shape
    x = np.asarray(x, dtype=np.float64)
    p = x.shape[1]
    expanded, k = lfcShrink_checks(x, coef, contrast, res is not None, lfcThreshold, factors,
                                   dds.get("weights") is not None, dds.get("modelMatrix") is not None, type)
    nz = ~np.asarray(dds["allZero"], bool)
    if "weightsFail" in dds:
        nz = nz & ~np.asarray(dds["weightsFail"], bool)
    fit = nz.copy()
    replaced = "replace" in dds and np.nansum(dds["replace"]) > 0
    if replaced:                                    # all zero once replaced: allZero in R (R/core.R:2491-2492)
        fit &= ~(np.asarray(dds["replace"], bool) & (dds["baseMean"] == 0))
    betaMatrix, baseMean, dispFit = dds["betaMatrix"][fit], dds["baseMean"][fit], dds["dispFit"][fit]
    if expanded:
        _, names, fidx, _ = factorDesign(factors)
        _, mean_by_factor = estimateBetaPriorVar(betaMatrix, names, fidx, baseMean, dispFit, expandedType=True)
        betaPriorVar = np.array([1e6 if f < 0 else mean_by_factor[int(f)]
                                 for f in factorDesign(factors, expanded=True)[2]])
    else:
        names = ["Intercept"] + [f"column {j}" for j in range(1, p)]
        betaPriorVar, _ = estimateBetaPriorVar(betaMatrix, names, np.r_[-1, np.zeros(p - 1, int)], baseMean,
                                               dispFit, expandedType=False)
    if dds.get("normalizationFactors") is not None:
        nf = np.asarray(dds["normalizationFactors"])[fit]
    else:
        nf = np.broadcast_to(dds["sizeFactors"], (int(fit.sum()), m))
    w = dds.get("weights")
    if w is not None:
        w = np.asarray(w)[fit[nz]]
    gp = fitGLMsWithPrior(counts[fit], nf, factors, dds["dispersion"][fit], None, None, engine=engine,
                          betaTol=betaTol, maxit=maxit, minmu=minmu, useOptim=useOptim, betaPriorVar=betaPriorVar,
                          modelMatrix=None if expanded else x, weights=w)
    f = gp["fit"]
    with np.errstate(divide="ignore", invalid="ignore"):
        stat = f["betaMatrix"] / f["betaSE"]
    shr = dict(dds)
    shr["test"] = "Wald"
    shr.pop("tDegreesFreedom", None)                # the MAP refit's nbinomWaldTest drops it: normal tails
    for key, v in (("betaMatrix", f["betaMatrix"]), ("betaSE", f["betaSE"]), ("WaldStatistic", stat),
                   ("WaldPvalue", 2.0 * _sp.ndtr(-np.abs(stat)))):
        shr[key] = np.full((N, v.shape[1]), np.nan)
        shr[key][fit] = v
    if expanded:
        shr["betaPriorVar"], shr["modelMatrix"] = betaPriorVar, gp["modelMatrix"]
    if replaced and lfcThreshold > 0:
        if cooks is None:
            raise ValueError("after an outlier refit a thresholded shrunk table needs the first fit's Cook's "
                             "distances (cooks=...)")
        shr["maxCooks"] = np.full(N, np.nan)
        shr["maxCooks"][nz] = recordMaxCooks(x, np.asarray(cooks, dtype=np.float64)[nz])
    sel = dict(contrast=contrast) if expanded else dict(name=k)
    if res is None:
        lrt = ({"LRTStatistic": dds["LRTStatistic"], "LRTPvalue": dds["LRTPvalue"]} if dds.get("test") == "LRT"
               else None)
        res = results(dds, counts, x, factors=factors, lrt=lrt, cooks=cooks, engine=engine, **sel)
    tab = results(shr, counts, x, lfcThreshold=lfcThreshold, factors=factors, minmu=minmu, cooks=cooks,
                  engine=engine, **sel)
    out = dict(res)
    for key in ["log2FoldChange", "lfcSE"] + (["stat", "pvalue", "padj"] if lfcThreshold > 0 else []):
        out[key] = tab[key]
    out["metadata"] = dict(res.get("metadata", {}))
    out["metadata"]["priorInfo"] = {"type": "normal", "package": "DESeq2", "betaPriorVar": betaPriorVar}
    return out
