"""Device-resident DESeq() Wald path: counts go in once (gene-major, on the GPU), every per-gene step runs on the
device, only a handful of scalars ever reach the host.

Same sequence as deseq2_b200/pipeline.py (the numpy restatement of R/core.R:280-432 with test="Wald",
fitType="parametric", no outlier replacement by default; betaPrior=FALSE by default), but
  * the pre-steps (base mean/variance, rough + moments dispersion, linear-model mu, IRLS start values) are one
    CUDA kernel (b200nb_prep_dev, csrc/pipeline_kernels.cu),
  * the parametric dispersion-trend fit is one single-CTA kernel (b200nb_trend_fit_dev),
  * fitDisp / fitDispGrid / fitBeta are the engine's device entry points,
  * the elementwise rules between them (noIncrease, convergence flags, clamps, outlier rule, MAD, Wald statistic
    and p-value) are a few torch tensor ops -- plumbing, not the product.
This is SURVEY.md section 8(f) rows 2-3 (pre-steps and Wald statistics on device) layered on rows (a)-(e).
DESeq_device(betaPrior=True, factors=...) runs the reference's betaPrior=TRUE Wald path for additive factor designs
(fitGLMsWithPrior, R/fitNbinomGLMs.R:242-337): the MLE fit above, the prior variance of estimateBetaPriorVar
("weighted": one launch of b200nb_beta_prior_quantile_dev, csrc/beta_prior.cuh, for all columns and level contrasts,
then averagePriorsOverLevels in torch), and the MAP fit on the expanded model matrix.
DESeq_device(weights=...), nbinomLRT_device(weights=...) and getContrast_device(weights=...) take observation
weights (the "weights" assay): the weight checks and the weighted pre-steps are the weighted instantiation of the prep
kernel (b200nb_prep_weighted_dev), and every fit passes the normalised weights to the engine's weighted fitDisp /
fitDispGrid / fitBeta / log-likelihood / optim entry points.
DESeq_device(normalizationFactors=...) (or avgTxLength=..., estimated by normalization_factors), nbinomLRT_device and
getContrast_device take gene-specific normalization factors (the "normalizationFactors" assay): the pre-steps and
Cook's distances are the nf instantiations of their kernels (b200nb_prep_nf_dev, b200nb_cooks_nf_dev), and every fit
gets the nf rows of its genes, which the engine's fitBeta / log-likelihood / optim entry points take in place of the
size-factor vector.
DESeq_device(sfType="iterate") estimates the size factors with size_factors_iterate (estimateSizeFactorsIterate,
R/core.R:2589-2622): the dispersion chain for ~1 with fitType "mean" on the device, and scipy's L-BFGS-B over the log
size factors whose every objective call (value and central differences) is b200nb_sf_iterate_objective_dev
(csrc/sf_iterate.cuh).  DESeq_device(fitType="mean") replaces the parametric trend by the trimmed mean of the
gene-wise estimates (mean_disp).
vst_device, varianceStabilizingTransformation_device, vst_transform and normTransform_device (R/vst.R,
R/helper.R:421-435) fit the dispersion function with DESeq_device's GeneEst block and trend, and transform the n x m
matrix with one kernel (b200nb_transform_dev, csrc/transform.cuh).
rlog_device (R/rlog.R) fits the dispersion function the same way, then runs rlogData's prior variance
(b200nb_rlog_prior_var_dev) and its per-gene fit of the design [1 | I_m] (b200nb_rlog_fit_dev, csrc/rlog.cuh).
lfcShrink_device (R/lfcShrink.R, type "normal") refits a DESeq_device result with a zero-centred normal prior: the
standard (coef) or expanded (contrast) prior variance from the prior-variance kernel, the MAP fit shared with
DESeq_device(betaPrior=True) (_map_fit), and results_device on it.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib
from . import device as D
# The call helpers live in device.py.  Their names stay importable from here for callers that use or replace
# device_pipeline._p / ._stream; the bindings below call D._p and D._stream() at call time, so replacing
# device._stream is what changes the stream they use.
from .device import _p, _stream  # noqa: F401
from .pipeline import check_test_args, modelMatrixGroups

F64 = torch.float64
LN2 = float(np.log(2.0))


_WS = {}


def _ws(name, shape, dtype, dev):
    """Reusable n x ld work matrices (fitted means, hat diagonals): at 20k x 1000 a fresh 160 MB torch allocation per
    call was measured to cost tens of ms in allocator / cudaMalloc churn, far more than the kernels that fill it.
    The tensors returned by DESeq_device under "mu" / "H" are views of this workspace: valid until the next call."""
    key = (name, str(dev))
    t = _WS.get(key)
    if t is None or t.shape != tuple(shape) or t.dtype != dtype:
        t = torch.empty(shape, dtype=dtype, device=dev)
        _WS[key] = t
    return t


def size_factor_ratios(y, m, poscounts=False, divisor=None, ws="sf_ratios"):
    """One launch of b200nb_size_factors_dev (b200nb_size_factors_norm_dev with a gene-major (n, ld) divisor matrix):
    returns {"sizeFactors": (m,), "loggeomeans": (n,), "ratios": the (m, n) log ratios of the median, one sample per
    row, +Inf where an entry does not take part (a view of the workspace named `ws`: valid until the next call that
    uses it), "n_finite": the number of genes with a finite log geometric mean as a 1-element device tensor}.  Does
    not raise when it is 0."""
    L = _lib.lib()
    dev = y.device
    n, ld = y.shape
    out = {"sizeFactors": torch.empty(m, dtype=F64, device=dev), "loggeomeans": torch.empty(n, dtype=F64, device=dev),
           "n_finite": torch.zeros(1, dtype=torch.int32, device=dev)}
    gm = _ws(ws, (n, ld), F64, dev)
    cm = _ws(ws + "_cm", (n * m,), F64, dev)
    if divisor is None:
        _lib.check(L.b200nb_size_factors_dev(D._p(y), D._ytype(y), int(poscounts), n, m, ld, D._p(out["loggeomeans"]),
                                             D._p(gm), D._p(cm), D._p(out["sizeFactors"]), D._p(out["n_finite"]),
                                             D._stream()), "size_factors")
    else:
        _lib.check(L.b200nb_size_factors_norm_dev(D._p(y), D._ytype(y), D._p(divisor), int(poscounts), n, m, ld,
                                                  D._p(out["loggeomeans"]), D._p(gm), D._p(cm),
                                                  D._p(out["sizeFactors"]), D._p(out["n_finite"]), D._stream()),
                   "size_factors_norm")
    out["ratios"] = cm.view(m, n)
    return out


def _no_finite_loggeomean():
    return ValueError("every gene contains at least one zero, cannot compute log geometric means")


def size_factors(y, m, type="ratio", controlGenes=None, geoMeans=None):
    """b200nb_size_factors_dev: estimateSizeFactorsForMatrix (R/core.R:535-578, locfunc = median) on the device.
    y: gene-major (n, ld) device tensor, m samples.  Returns {"sizeFactors": (m,) device tensor, "loggeomeans": (n,)}.
    Raises like the reference when every gene contains a zero (the only host read: one int).
    controlGenes (a boolean mask with one entry per row, or 0-based row indices; pipeline.controlGeneRows) and
    geoMeans (one value per row, numpy or a device tensor) as in R, through control_ratios: the median is over the
    control rows, the stop looks at every row, and with geoMeans the factors are rescaled to geometric mean 1 (type
    "ratio" only: "poscounts" with geoMeans raises ValueError).  As without them, "poscounts" factors are returned
    unscaled."""
    if controlGenes is None and geoMeans is None:
        if type not in ("ratio", "poscounts"):
            raise ValueError("type must be 'ratio' or 'poscounts'")
        r = size_factor_ratios(y, m, poscounts=type == "poscounts")
        if int(r["n_finite"].item()) == 0:
            raise _no_finite_loggeomean()
        return {"sizeFactors": r["sizeFactors"], "loggeomeans": r["loggeomeans"]}
    r = control_ratios(y, m, type, None, controlGenes, geoMeans)
    if int(r["n_finite"].item()) == 0:
        raise _no_finite_loggeomean()
    return {"sizeFactors": control_sizes(r), "loggeomeans": r["loggeomeans"]}


def _kernel_ratios(y, m, poscounts, divisor, ws):
    """size_factor_ratios, or for no rows what the median of no rows gives: NaN factors, no ratio, n_finite 0."""
    if y.shape[0] == 0:
        dev = y.device
        return {"sizeFactors": torch.full((m,), math.nan, dtype=F64, device=dev),
                "ratios": torch.empty((m, 0), dtype=F64, device=dev),
                "loggeomeans": torch.empty(0, dtype=F64, device=dev),
                "n_finite": torch.zeros(1, dtype=torch.int32, device=dev)}
    return size_factor_ratios(y, m, poscounts=poscounts, divisor=divisor, ws=ws)


def given_geo_mean_ratios(y, m, loggeomeans, divisor=None):
    """The (m, n) log ratios of the median against given log geometric means, laid out as the size-factor kernel's
    ratio scratch: log K_ij - loggeomeans_i (log(K_ij / d_ij) with a gene-major divisor), +Inf where the entry does not
    take part (loggeomeans_i not finite, or K_ij = 0).  One elementwise pass in torch; the log is torch's."""
    k = y[:, :m].to(F64)
    if divisor is not None:
        k = k / divisor[:, :m]
    use = torch.isfinite(loggeomeans)[:, None] & (k > 0)
    return torch.where(use, torch.log(k) - loggeomeans[:, None], math.inf).t().contiguous()


def column_medians(ratios):
    """(m,) exact medians of the rows of an (m, k) ratio matrix over their entries below +Inf, as sf_median_kernel takes
    them: the lower middle element for an odd count, the mean of the two middle elements for an even one (R's median),
    NaN for none; and the (m,) counts.  One segmented sort."""
    m, k = ratios.shape
    nv = (ratios < math.inf).sum(dim=1)
    if k == 0:
        return torch.full((m,), math.nan, dtype=F64, device=ratios.device), nv
    s = torch.sort(ratios, dim=1)[0]
    lo = s.gather(1, (torch.clamp(nv - 1, min=0) // 2)[:, None]).squeeze(1)
    hi = s.gather(1, torch.clamp(nv // 2, max=k - 1)[:, None]).squeeze(1)
    med = torch.where(nv % 2 == 1, lo, 0.5 * (lo + hi))
    return torch.where(nv == 0, math.nan, med), nv


def control_ratios(y, m, type, divisor, controlGenes, geoMeans):
    """The ratios estimateSizeFactorsForMatrix takes the median of when controlGenes and / or geoMeans are given
    (R/core.R:539-572), for size_factors, normalization_factors and their gene-sharded forms.  Checks the arguments
    (ValueError) and returns {"ratios": (m, k) ratios of the k control rows (+Inf where an entry does not take part),
    "loggeomeans": (n,) of every row, "n_finite": 1-element device count of the rows whose loggeomeans is not infinite
    (R stops when it is 0), "sizeFactors": the kernel's medians of "ratios", or None with geoMeans,
    "incoming": whether geoMeans were given}.
      * controlGenes only: the size-factor kernel on all rows (loggeomeans and the stop count, exactly as without
        controlGenes), then on the gathered control rows for the ratios and their medians (its own workspace).  The
        log geometric means are per row, so the second launch's equal the first's.
      * geoMeans: loggeomeans = torch.log(geoMeans) (0 gives -Inf, a negative value or NaN gives NaN), the ratios of
        the control rows (every row without controlGenes) by given_geo_mean_ratios."""
    from .pipeline import checkGeoMeansType, controlGeneRows
    checkGeoMeansType(type, geoMeans)
    n = y.shape[0]
    dev = y.device
    rows = None
    if controlGenes is not None:
        rows = torch.as_tensor(controlGeneRows(controlGenes, n), device=dev)

    def sub(t):
        return t if rows is None or t is None else t[rows].contiguous()

    if geoMeans is None:
        full = _kernel_ratios(y, m, type == "poscounts", divisor, "sf_ratios")
        part = _kernel_ratios(sub(y), m, type == "poscounts", sub(divisor), "sf_ratios_ctl")
        return {"ratios": part["ratios"], "loggeomeans": full["loggeomeans"], "n_finite": full["n_finite"],
                "sizeFactors": part["sizeFactors"], "incoming": False}
    g = geoMeans if isinstance(geoMeans, torch.Tensor) else torch.as_tensor(np.asarray(geoMeans, dtype=np.float64))
    if g.dim() != 1 or g.shape[0] != n:
        raise ValueError("geoMeans should be as long as the number of rows of counts")
    lg = torch.log(g.to(device=dev, dtype=F64))
    return {"ratios": given_geo_mean_ratios(sub(y), m, sub(lg), sub(divisor)), "loggeomeans": lg,
            "n_finite": (~torch.isinf(lg)).sum().reshape(1), "sizeFactors": None, "incoming": True}


def rescaled_to_geo_mean_one(sf):
    """The incoming-geoMeans rescaling sf / exp(mean(log sf)) (R/core.R:573-576): one NaN factor makes all NaN."""
    return sf / torch.exp(torch.log(sf).mean())


def control_sizes(r):
    """The size factors of control_ratios' result on one device: the kernel's medians, or with geoMeans the exact
    column medians through the kernel's exp (sharded._sizes_of), rescaled to geometric mean 1."""
    if r["sizeFactors"] is not None:
        return r["sizeFactors"]
    from .sharded import _sizes_of
    med, nv = column_medians(r["ratios"])
    return rescaled_to_geo_mean_one(_sizes_of(med, nv))


def sf_iterate_objective(y, q, alpha, par, m, h=1e-3, Q=0.05, max_tile_cols=0, out=None):
    """b200nb_sf_iterate_objective_dev: estimateSizeFactorsIterate's objective at the log size factors `par` and at
    the 2m points of optim's central differences, as a (2m + 1,) device tensor in the column order of
    pipeline.iterateObjective.  y: gene-major (n, ld) counts; q: gene-major (n, ld) float64 mu / s; alpha: (n,)
    dispersions; par: (m,) float64 device tensor.  max_tile_cols bounds the objective columns per tile (0: the
    library's default).  Enqueue only."""
    L = _lib.lib()
    n, ld = y.shape
    if out is None:
        out = torch.empty(2 * m + 1, dtype=F64, device=y.device)
    _lib.check(L.b200nb_sf_iterate_objective_dev(D._p(y), D._ytype(y), D._p(q), D._p(alpha), D._p(par),
                                                 float(h), float(Q), n, m, ld, int(max_tile_cols), D._p(out),
                                                 D._stream()), "sf_iterate_objective")
    return out


def mean_disp(dge, minDisp=1e-8):
    """fitType = "mean" (R/core.R:900-905) on a device tensor: mean(dge[dge > 10 minDisp], trim = 0.001) with
    mean.default's bounds floor(n trim) + 1 .. n - floor(n trim) and .Internal(mean)'s residual correction.  Raises
    ValueError, as estimateDispersionsFit does, when no estimate exceeds 100 minDisp (one host read).  Returns a
    0-d device tensor."""
    if not bool((dge > 100 * minDisp).any()):
        raise ValueError("all gene-wise dispersion estimates are within 2 orders of magnitude from the minimum value")
    v, _ = torch.sort(dge[dge > 10 * minDisp])
    n = v.numel()
    lo = int(np.floor(n * 0.001))
    v = v[lo:n - lo]
    s = v.sum() / v.numel()
    return s + (v - s).sum() / v.numel()


def _check_positive_matrix(t, y, m, name):
    """A gene-major float64 tensor of the counts' shape on their device whose first m columns are finite and > 0
    (normalizationFactors<-, R/methods.R:345-350).  One host read."""
    if not isinstance(t, torch.Tensor) or t.dtype != F64 or t.device != y.device:
        raise ValueError(f"{name} must be a float64 tensor on the counts' device")
    if tuple(t.shape) != tuple(y.shape) or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous gene-major tensor of the counts' shape {tuple(y.shape)}, "
                         f"got {tuple(t.shape)}")
    v = t[:, :m]
    if bool((~(torch.isfinite(v) & (v > 0))).any()):
        raise ValueError(f"{name} must be finite and positive")


def normalization_factors(y, m, normMatrix=None, avgTxLength=None, type="ratio", controlGenes=None, geoMeans=None):
    """estimateSizeFactors with a normMatrix or an avgTxLength assay (R/methods.R:363-406) on the device: exactly one of
    the two, a gene-major (n, ld) float64 tensor aligned with y.  avgTxLength is first divided by its row geometric
    mean.  estimateNormFactors (R/core.R:2159-2163): the median-of-ratios size factors of K / normMatrix
    (b200nb_size_factors_norm_dev; for "poscounts" the log geometric means come from the raw counts and the factors are
    rescaled to geometric mean 1, R/core.R:573-576), then nf = normMatrix * sf divided by its row geometric mean.
    controlGenes and geoMeans as in size_factors: the median is over the control rows, given geoMeans are compared with
    K / normMatrix (and the factors rescaled), and nf is formed for every row.
    Returns {"normalizationFactors": (n, ld) device tensor (padding columns 1), "sizeFactors": (m,)}.
    Raises ValueError for a non-positive / non-finite matrix and when every gene contains a zero."""
    nm, d = norm_divisor(y, m, normMatrix, avgTxLength, type)
    if controlGenes is not None or geoMeans is not None:
        r = control_ratios(y, m, type, d, controlGenes, geoMeans)
        if int(r["n_finite"].item()) == 0:
            raise _no_finite_loggeomean()
        return norm_factors_from(nm, d, control_sizes(r), m, type)
    r = size_factor_ratios(y, m, poscounts=type == "poscounts", divisor=d)
    if int(r["n_finite"].item()) == 0:
        raise _no_finite_loggeomean()
    return norm_factors_from(nm, d, r["sizeFactors"], m, type)


def norm_divisor(y, m, normMatrix, avgTxLength, type):
    """The checks of normalization_factors and its divisor: (normMatrix, or avgTxLength over its row geometric mean, as
    an (n, m) tensor; the same in a gene-major (n, ld) matrix whose padding columns are 1)."""
    if type not in ("ratio", "poscounts"):
        raise ValueError("type must be 'ratio' or 'poscounts'")
    if (normMatrix is None) == (avgTxLength is None):
        raise ValueError("give exactly one of normMatrix and avgTxLength")
    name = "normMatrix" if normMatrix is not None else "avgTxLength"
    src = normMatrix if normMatrix is not None else avgTxLength
    _check_positive_matrix(src, y, m, name)
    n, ld = y.shape
    nm = src[:, :m]
    if avgTxLength is not None:
        nm = nm / torch.exp(torch.log(nm).mean(dim=1, keepdim=True))
    d = torch.ones((n, ld), dtype=F64, device=y.device)
    d[:, :m] = nm
    return nm, d


def norm_factors_from(nm, d, sf, m, type):
    """normalization_factors' last step from the size factors of K / normMatrix: the poscounts rescaling, nf =
    normMatrix * sf over its row geometric mean, written into d's first m columns."""
    if type == "poscounts":
        sf = sf / torch.exp(torch.log(sf).mean())
    nf = nm * sf[None, :]
    nf = nf / torch.exp(torch.log(nf).mean(dim=1, keepdim=True))
    d[:, :m] = nf
    return {"normalizationFactors": d, "sizeFactors": sf}


def nf_column_sums(nf, m):
    """The two numbers per sample that momentsDispEstimate's xim needs from a set of rows: their nf column sums (m,)
    and their count.  Summed over the ranks in rank order by the sharded driver."""
    return nf[:, :m].sum(dim=0), nf.shape[0]


def nf_xim(colsum, count):
    """xim = mean(1 / colMeans(nf)) (R/core.R:2440-2441) from nf_column_sums."""
    return float((1.0 / (colsum / count)).mean().item())


def _rows(nfd, rows):
    """The normalization factors of `rows` (a gene-major matrix), or the size-factor vector unchanged."""
    return nfd[rows].contiguous() if nfd.dim() == 2 else nfd


def _projection(x):
    """(X'X)^-1 X' (p x m) WITHOUT a BLAS / LAPACK call.  numpy hands `x.T @ x` and linalg.solve to OpenBLAS, whose
    worker threads (one per CPU the process may run on: 64-128 on the GPU hosts) then busy-wait for ~100 ms; under a
    container CPU quota (the 1-GPU lease: cpu.max = 16 CPUs) that spin exhausts the quota and the kernel throttles the
    WHOLE process for the rest of the period, leaving random holes of tens of ms in the host timeline.  The matrices
    are p x p with p <= 32: einsum's own loops and a Gauss-Jordan sweep with partial pivoting are plenty."""
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    a = np.einsum("ik,il->kl", x, x)                       # X'X (c_einsum loops, no BLAS)
    aug = np.concatenate([a, np.ascontiguousarray(x.T)], axis=1)   # [X'X | X']
    for c in range(p):
        piv = c + int(np.argmax(np.abs(aug[c:, c])))
        if aug[piv, c] == 0.0:
            raise np.linalg.LinAlgError("singular design matrix")
        if piv != c:
            aug[[c, piv]] = aug[[piv, c]]
        aug[c] /= aug[c, c]
        f = aug[:, c].copy()
        f[c] = 0.0
        aug -= f[:, None] * aug[c][None, :]
    return np.ascontiguousarray(aug[:, p:])


def prep(y, x, sizeFactors, minDisp=1e-8, minmu=0.5, want_mu=True, want_beta0=True, weights=None,
         weightThreshold=1e-2, normalizationFactors=None, xim=None):
    """b200nb_prep_dev.  y: gene-major (n, ld) int32/float64 device tensor; x: (m, p) numpy; sizeFactors: (m,) numpy.
    weights: gene-major (n, ld) float64 device tensor of raw observation weights -> b200nb_prep_weighted_dev, which
    adds "weightsNorm" (n, ld: weights / row maximum), "weightsFail" (n,) int32 and "status" (1,) int32, the number
    of rows whose weights the reference rejects (the caller raises when it is not 0).  mu_lin is not computed then.
    normalizationFactors: gene-major (n, ld) float64 device tensor of the same rows -> b200nb_prep_nf_dev
    (sizeFactors is ignored); xim defaults to mean(1 / colMeans(nf)) over these rows.  "sfd" is then this matrix."""
    L = _lib.lib()
    dev = y.device
    n, ld = y.shape
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    proj = _projection(x)                                      # (X'X)^-1 X', p x m
    xd = D.x_to_device(x, dev)
    projd = torch.as_tensor(np.ascontiguousarray(proj), device=dev)
    nf = normalizationFactors
    if nf is None:
        sfd = torch.as_tensor(np.asarray(sizeFactors, dtype=np.float64), device=dev)
        xim = float(np.mean(1.0 / np.asarray(sizeFactors)))
    else:
        if weights is not None:
            raise ValueError("observation weights together with normalization factors are not supported")
        sfd = nf
        if xim is None:
            xim = nf_xim(*nf_column_sums(nf, m))
    out = {"baseMean": torch.empty(n, dtype=F64, device=dev), "baseVar": torch.empty(n, dtype=F64, device=dev),
           "allZero": torch.empty(n, dtype=torch.int32, device=dev), "alpha0": torch.empty(n, dtype=F64, device=dev),
           "mu_lin": _ws("mu_lin", (n, ld), F64, dev) if want_mu else None,
           "beta0": torch.empty((p, n), dtype=F64, device=dev) if want_beta0 else None}
    args = (D._p(y), D._ytype(y), D._p(xd), D._p(projd), D._p(sfd), float(xim), float(minDisp),
            float(max(10, m)), float(minmu), n, m, p, ld, D._p(out["baseMean"]), D._p(out["baseVar"]),
            D._p(out["allZero"]), D._p(out["alpha0"]))
    if nf is not None:
        _lib.check(L.b200nb_prep_nf_dev(*args, D._p(out["mu_lin"]), D._p(out["beta0"]), D._stream()), "prep_nf_dev")
    elif weights is None:
        rc = L.b200nb_prep_dev(*args, D._p(out["mu_lin"]), D._p(out["beta0"]), D._stream())
        _lib.check(rc, "prep_dev")
    else:
        _check_weights_tensor(weights, y)
        out["mu_lin"] = None
        out["weightsNorm"] = torch.empty((n, ld), dtype=F64, device=dev)
        out["weightsFail"] = torch.empty(n, dtype=torch.int32, device=dev)
        out["status"] = torch.zeros(1, dtype=torch.int32, device=dev)
        rc = L.b200nb_prep_weighted_dev(*args, None, D._p(out["beta0"]), D._p(weights), float(weightThreshold),
                                        D._p(out["weightsNorm"]), D._p(out["weightsFail"]), D._p(out["status"]),
                                        D._stream())
        _lib.check(rc, "prep_weighted_dev")
    out["xd"], out["sfd"] = xd, sfd
    return out


def _check_weights_tensor(weights, y):
    if not isinstance(weights, torch.Tensor) or weights.dtype != F64 or weights.device != y.device:
        raise ValueError("weights must be a float64 tensor on the counts' device")
    if tuple(weights.shape) != tuple(y.shape) or not weights.is_contiguous():
        raise ValueError(f"weights must be a contiguous gene-major tensor of the counts' shape {tuple(y.shape)}, "
                         f"got {tuple(weights.shape)}")


def normalize_weights(weights, y, m):
    """weights / row maximum over the first m columns (the normalisation of getContrast and fitNbinomGLMs,
    R/results.R:794, R/core.R:2700-2702), padding columns 0.  Idempotent: normalised rows come back bit for bit.
    Raises ValueError, with one host read, on a negative or NaN weight or a row without a positive, finite maximum."""
    _check_weights_tensor(weights, y)
    w = weights[:, :m]
    wmax = w.max(dim=1).values if w.shape[0] else torch.zeros(0, dtype=F64, device=w.device)
    bad = (~(w >= 0)).any(dim=1) | ~(wmax > 0) | ~torch.isfinite(wmax)
    if bool(bad.any()):
        raise ValueError(f"{int(bad.sum())} row(s) of weights have a negative or NaN weight or no positive, finite "
                         "maximum")
    out = torch.zeros_like(weights)
    out[:, :m] = w / wmax[:, None]
    return out


def trend_fit(means, disps, minDisp=1e-8):
    """parametricDispersionFit on device: returns a 4-vector tensor (asymptDisp, extraPois, status, rounds)."""
    L = _lib.lib()
    out = torch.empty(4, dtype=F64, device=means.device)
    _lib.check(L.b200nb_trend_fit_dev(D._p(means), D._p(disps), means.numel(), float(minDisp), D._p(out), D._stream()),
               "trend_fit_dev")
    return out


def cooks(y, mu, hat, x, sizeFactors, want_matrix=True, normalizationFactors=None):
    """b200nb_cooks_dev: Cook's distances, their per-gene maximum and the robust moments dispersion.
    normalizationFactors: gene-major (n, ld) of the same rows -> b200nb_cooks_nf_dev (sizeFactors is ignored)."""
    from .pipeline import designCells
    L = _lib.lib()
    dev = y.device
    n, ld = y.shape
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    cells, sizes = designCells(x)
    order = np.argsort(cells, kind="stable").astype(np.int32)
    ptr = np.r_[0, np.cumsum(sizes)].astype(np.int32)
    ptrd = torch.as_tensor(ptr, device=dev)
    ordd = torch.as_tensor(order, device=dev)
    nf = normalizationFactors
    sfd = nf if nf is not None else torch.as_tensor(np.asarray(sizeFactors, dtype=np.float64), device=dev)
    out = {"cooks": torch.empty((n, ld), dtype=F64, device=dev) if want_matrix else None,
           "maxCooks": torch.empty(n, dtype=F64, device=dev), "robustDisp": torch.empty(n, dtype=F64, device=dev)}
    entry = L.b200nb_cooks_nf_dev if nf is not None else L.b200nb_cooks_dev
    rc = entry(D._p(y), D._ytype(y), D._p(mu), D._p(hat), D._p(sfd), D._p(ptrd), D._p(ordd),
               len(sizes), n, m, p, ld, D._p(out["cooks"]), D._p(out["maxCooks"]), D._p(out["robustDisp"]), D._stream())
    _lib.check(rc, "cooks_dev")
    return out


def beta_prior_quantile(beta, baseMean, dispFit, col_a, col_b, prob):
    """b200nb_beta_prior_quantile_dev: Hmisc.wtd.quantile(|x_c|, 1/(1/baseMean + dispFit), prob, normwt=TRUE) over the
    entries with |x_c| < 10, for every column x_c = beta[a] - (b < 0 ? 0 : beta[b]).  beta: (p, n) contiguous device
    tensor (log2 scale); col_a / col_b: integer sequences of equal length k.  Returns (k,) with NaN where no entry
    is kept."""
    L = _lib.lib()
    dev = beta.device
    p, n = beta.shape
    ca = torch.as_tensor(np.asarray(col_a, dtype=np.int32), device=dev)
    cb = torch.as_tensor(np.asarray(col_b, dtype=np.int32), device=dev)
    out = torch.empty(ca.numel(), dtype=F64, device=dev)
    _lib.check(L.b200nb_beta_prior_quantile_dev(D._p(beta), n, p, D._p(baseMean), D._p(dispFit), D._p(ca), D._p(cb),
                                                ca.numel(), float(prob), D._p(out), D._stream()),
               "beta_prior_quantile_dev")
    return out


def beta_prior_columns(fidx):
    """The columns estimateBetaPriorVar takes quantiles of, for a standard factor design whose column c belongs to
    factor fidx[c] (-1 = intercept): every non-intercept column, then addAllContrasts' differences of each factor's
    level columns in R's is/js order (R/expanded.R:76-98).  Returns (col_a, col_b, factor of each column)."""
    fidx = np.asarray(fidx)
    a = [c for c in range(len(fidx)) if fidx[c] >= 0]
    b = [-1] * len(a)
    owner = [int(fidx[c]) for c in a]
    for f in sorted({int(v) for v in fidx if v >= 0}):
        cols = np.flatnonzero(fidx == f)
        for j in range(len(cols) - 1):
            for i in range(j + 1, len(cols)):
                a.append(int(cols[i]))
                b.append(int(cols[j]))
                owner.append(f)
    return np.asarray(a, np.int32), np.asarray(b, np.int32), np.asarray(owner)


def estimate_beta_prior_var(betaMatrix, factors, baseMean, dispFit, upperQuantile=0.05, expandedType=True):
    """estimateBetaPriorVar (R/core.R:1601-1689, betaPriorMethod "weighted") on the device.
    betaMatrix: (n, p) MLE log2 fold changes (DESeq_device's "betaMatrix"); baseMean / dispFit: (n,) device tensors.
    expandedType=True (modelMatrixType "expanded", DESeq(betaPrior=TRUE) and lfcShrink(contrast=)): betaMatrix is on
    the standard matrix factorDesign(factors)[0]; the quantiles of all columns and addAllContrasts' level differences
    are one kernel launch, averagePriorsOverLevels (R/expanded.R:20-73) a few torch ops, and the result holds the
    prior variances of the EXPANDED matrix's columns.  expandedType=False (modelMatrixType "standard",
    lfcShrink(coef=)): betaMatrix is on any design whose column 0 is the intercept (factors is not used); one quantile
    per other column, in one launch, and the result holds the prior variances of those p columns.  Either way the
    intercept gets 1e6, a column with no |beta| < 10 gets 1e6, and a single gene gets beta^2 (R/core.R:1648-1666).
    Returns a device tensor.  Raises ValueError like R when one of them is NA or not positive (one host read)."""
    from scipy import stats as _st
    from .pipeline import factorDesign
    bt = betaMatrix.T.contiguous()                                      # (p, n): a view's base when it is one
    dev = bt.device
    if expandedType:
        _, _, fidx, _ = factorDesign(factors, expanded=False)
        _, enames, efidx, _ = factorDesign(factors, expanded=True)
        col_a, col_b, owner = beta_prior_columns(fidx)
    else:
        p = bt.shape[0]
        col_a, col_b = np.arange(1, p, dtype=np.int32), np.full(p - 1, -1, np.int32)
        enames = ["Intercept"] + [f"column {k}" for k in range(1, p)]
    if bt.shape[1] > 1:
        q = beta_prior_quantile(bt, baseMean, dispFit, col_a, col_b, 1.0 - upperQuantile)
        z = float(_st.norm.ppf(1.0 - upperQuantile / 2.0))
        pv = torch.where(torch.isnan(q), torch.full_like(q, 1e6), (q / z) ** 2)   # no kept entry: wide prior
    else:                                                               # one gene: betaMatrix^2, no quantile
        a = torch.as_tensor(col_a.astype(np.int64), device=dev)
        b = torch.as_tensor(col_b.astype(np.int64), device=dev)
        x = bt[a, 0] - torch.where(b >= 0, bt[b.clamp(min=0), 0], torch.zeros_like(bt[a, 0]))
        pv = x ** 2
    if expandedType:
        out = torch.full((len(efidx),), 1e6, dtype=F64, device=dev)
        owner_d = torch.as_tensor(owner, device=dev)
        for f in sorted({int(v) for v in efidx if v >= 0}):
            out[torch.as_tensor(efidx == f, device=dev)] = pv[owner_d == f].mean()
    else:
        out = torch.cat([torch.full((1,), 1e6, dtype=F64, device=dev), pv])
    bad = (torch.isnan(out) | (out <= 0)).cpu().numpy()
    if bad.any():
        raise ValueError("beta prior for " + ",".join(np.asarray(enames)[bad]) + " is NA or not greater than 0")
    return out


def _median(v):
    """R's median (mean of the two middle order statistics for even length)."""
    s, _ = torch.sort(v)
    k = s.numel()
    return s[k // 2] if k % 2 else 0.5 * (s[k // 2 - 1] + s[k // 2])


def _grid_refit(y, xd, mu, sel, m, prior_mean, prior_sigmasq, usePrior, weights=None, weightThreshold=1e-2):
    """fitDispGridWrapper (R/wrappers.R:63-83) on the genes flagged in boolean `sel`; returns (idx, alpha)."""
    idx = torch.nonzero(sel).squeeze(1)
    if idx.numel() == 0:
        return idx, None
    grid = np.linspace(np.log(1e-8), np.log(max(10, m)), 20)
    pm = prior_mean[idx] if prior_mean is not None else torch.zeros(idx.numel(), dtype=F64, device=y.device)
    w = None if weights is None else weights[idx].contiguous()
    la = D.fit_disp_grid(y[idx].contiguous(), xd, mu[idx].contiguous(), grid, pm, prior_sigmasq, usePrior, weights=w,
                         weightThreshold=weightThreshold)["log_alpha"]
    return idx, torch.exp(la)


def getContrast_device(ynz, x, sizeFactors, dispersion, betaMatrix, contrast, betaPriorVar=None, minmu=0.5,
                       weights=None, normalizationFactors=None, useT=False, df=None):
    """getContrast (R/results.R:760-827) on device tensors: fitBeta's maxit = 0 mode (covariance at the given betas).
    ynz: gene-major counts the model was fitted to; betaMatrix: (n, p) log2-scale coefficients (DESeq_device's
    "betaMatrix").  weights: gene-major (n, ld) float64 observation weights of the same rows (raw, or DESeq_device's
    normalised "weights"), normalised by the row maximum and passed to fitBeta without the rank tests, as in the
    reference.  normalizationFactors: gene-major (n, ld) float64 factors of the same rows, in place of sizeFactors
    (None then).  useT: the p-value is 2 pt(|stat|, df, lower.tail = FALSE) (t_wald_pvalue, R/results.R:812-816) with
    df the rows' t degrees of freedom (a DESeq_device(useT=True) result's "tDegreesFreedom"); useT without df raises
    ValueError, as R's stopifnot.  Returns log2FoldChange, lfcSE, stat, pvalue as device tensors."""
    if useT and df is None:
        raise ValueError("useT=True needs the t degrees of freedom (tDegreesFreedom) of the rows")
    dev = ynz.device
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    sfd = _size_or_norm_factors(ynz, m, sizeFactors, normalizationFactors, weights)
    contrast = np.asarray(contrast, dtype=np.float64)
    if contrast.shape != (p,):
        raise ValueError("numeric contrast vector should have one element for every element of 'resultsNames(object)'")
    pv = np.full(p, 1e6) if betaPriorVar is None else np.asarray(betaPriorVar, dtype=np.float64)
    lam = torch.as_tensor(1.0 / (LN2 ** 2 * pv), device=dev)
    beta_nat = (betaMatrix.T * LN2).contiguous()                       # (p, n) = column-major n x p, natural log scale
    wn = None if weights is None else normalize_weights(weights, ynz, m)
    r = D.fit_beta(ynz, D.x_to_device(x, dev), sfd, dispersion, torch.as_tensor(contrast, device=dev), beta_nat, lam,
                   1e-8, 0, useQR=False, minmu=minmu, weights=wn, want_hat=False, want_mu=False)
    est, se = r["contrast_num"] / LN2, r["contrast_denom"] / LN2
    stat = est / se
    return {"log2FoldChange": est, "lfcSE": se, "stat": stat,
            "pvalue": t_wald_pvalue(stat, df) if useT else wald_pvalue(stat)}


def wald_pvalue(stat):
    """R's two-sided normal p-value 2 * pnorm(abs(stat), lower.tail = FALSE) (R/core.R:1507, R/results.R:822) as
    erfc(|stat| / sqrt 2): relative accuracy of a few ulps plus stat^2 ulps (the rounding of the argument) down to
    DBL_MIN, subnormal beyond |stat| = 37.5, 1 at 0, 0 at +-inf, NaN at NaN.  torch's ndtr is (1 + erf(x / sqrt 2)) / 2,
    which cancels: its p-values are multiples of about 1.1e-16 and reach 0 from |stat| = 8.3 on."""
    return torch.erfc(stat.abs() * 0.7071067811865476)


# lgamma(z) - ((z - 1/2) log z - z + log(2 pi) / 2) = sum_k B_2k / (2k (2k - 1) z^(2k - 1)): the first eight terms,
# whose truncation error is below 1e-17 for z >= 10
_STIRLING = (1.0 / 12.0, -1.0 / 360.0, 1.0 / 1260.0, -1.0 / 1680.0, 1.0 / 1188.0, -691.0 / 360360.0, 1.0 / 156.0,
             -3617.0 / 122400.0)
_SQRT_PI = 1.7724538509055160
_T_CHUNK = 8            # continued-fraction steps between two checks of which genes are still iterating
_T_MAXIT = 20000


def _stirling_delta(z):
    r = 1.0 / z
    r2 = r * r
    s = torch.full_like(z, _STIRLING[-1])
    for c in _STIRLING[-2::-1]:
        s = s * r2 + c
    return s * r


def _gamma_ratio_half(a):
    """Gamma(a + 1/2) / Gamma(a) for a > 0 to a few ulps, without lgamma (whose absolute error, relative to the ratio,
    is ~lgamma(a) ulps): for b = a + k >= 10 it is sqrt(b) exp(b log1p(1 / (2b)) - 1/2 + delta(b + 1/2) - delta(b))
    (Stirling's series; the exponent is O(1/b), so its rounding costs nothing), and below 10 the recurrence
    Gamma(a + 1/2) / Gamma(a) = Gamma(b + 1/2) / Gamma(b) prod_{j < k} (a + j) / (a + j + 1/2)."""
    k = torch.clamp(torch.ceil(10.0 - a), min=0.0)
    b = a + k
    r = torch.sqrt(b) * torch.exp(b * torch.log1p(0.5 / b) - 0.5 + _stirling_delta(b + 0.5) - _stirling_delta(b))
    for j in range(10):
        r = torch.where(k > j, r * ((a + j) / (a + j + 0.5)), r)
    return r


def _beta_cf(a, b, x):
    """The continued fraction of I_x(a, b) (modified Lentz, as in Numerical Recipes' betacf), elementwise over 1-D
    tensors, each element iterating until its step changes the value by at most an ulp.  The coefficients are formed
    as products of ratios, so that no intermediate overflows for any finite a.  Steps run _T_CHUNK at a time on the
    elements still iterating; each chunk costs one host read (how many are left)."""
    tiny = 1e-300
    h = torch.empty_like(x)
    ix = torch.arange(x.numel(), device=x.device)
    qab, qap, qam = a + b, a + 1.0, a - 1.0
    d = 1.0 - (qab / qap) * x
    d = 1.0 / torch.where(d.abs() < tiny, tiny, d)
    c, hh = torch.ones_like(x), d
    m = 1
    while ix.numel() and m <= _T_MAXIT:
        done = torch.zeros_like(x, dtype=torch.bool)
        for _ in range(_T_CHUNK):
            m2 = 2.0 * m
            for coef in ((m / (qam + m2)) * ((b - m) / (a + m2)) * x,
                         -((a + m) / (a + m2)) * ((qab + m) / (qap + m2)) * x):
                d = 1.0 + coef * d
                d = 1.0 / torch.where(d.abs() < tiny, tiny, d)
                c = 1.0 + coef / c
                c = torch.where(c.abs() < tiny, tiny, c)
                step = d * c
                hh = torch.where(done, hh, hh * step)
            done = done | ((step - 1.0).abs() <= 2.3e-16)
            m += 1
        fin = torch.nonzero(done).squeeze(1)
        h[ix[fin]] = hh[fin]
        left = torch.nonzero(~done).squeeze(1)
        ix, a, b, x, qab, qap, qam, c, d, hh = (t[left] for t in (ix, a, b, x, qab, qap, qam, c, d, hh))
    h[ix] = hh
    return h


def _expansion_coefs(b=0.5, n=30):
    """The constants d_n of the large-a expansion of I_x(a, b) (Didonato and Morris 1992, ACM TOMS 708, section 9):
    c_n = c_(n-1) / (2n (2n + 1)), c_0 = 1, d_n = (b - 1) c_n + (1 / n) sum_(i < n) (i b - n) c_i d_(n - i)."""
    c, d, cn = [], [], 1.0
    for k in range(1, n + 1):
        cn /= (2.0 * k) * (2.0 * k + 1.0)
        c.append(cn)
        d.append((b - 1.0) * cn + sum((i * b - k) * c[i - 1] * d[k - 1 - i] for i in range(1, k)) / k)
    return d


_EXPANSION_D = _expansion_coefs()


def _t_two_sided_expansion(q, df):
    """I_x(a, 1/2), a = df / 2, x = df / (df + q^2), by the asymptotic expansion for large a and b <= 1 of
    Didonato and Morris (TOMS 708, section 9) with b = 1/2, where the incomplete gamma function it rests on is
    Q(1/2, z) = erfc(sqrt z): I = erfc(sqrt z) Gamma(a + 1/2) / (Gamma(a) sqrt(T)) (1 + sum_n d_n J_n / J_0),
    T = a - 1/4, z = -T log x, J_0 = sqrt(pi) erfcx(sqrt z) / sqrt z and
    J_n = ((2n - 3/2)(2n - 1/2) J_(n-1) + (z + 2n - 1/2) (log(x) / 2)^(2n - 2)) / (4 T^2).  Every input is a
    function of log x = -log1p(q^2 / df), never of a rounded x, so large df loses nothing to the rounding of x (the
    continued fraction in x would lose about df / 2 ulps); the relative error stays within an ulp or two of the tail's
    condition number.  Used for df >= 20 where log1p(q^2 / df) <= 1, where the series converges within 30 terms."""
    a = 0.5 * df
    T = a - 0.25
    lnx = -torch.log1p(q * q / df)
    z = -T * lnx
    sz = torch.sqrt(z)
    inv_j0 = sz / (torch.special.erfcx(sz) * _SQRT_PI)
    v = 0.25 / (T * T)
    t2 = 0.25 * lnx * lnx
    k, t, s = torch.ones_like(q), torch.ones_like(q), torch.ones_like(q)
    for n, dn in enumerate(_EXPANSION_D):
        bp = 0.5 + 2.0 * n
        k = (bp * (bp + 1.0) * k + (z + bp + 1.0) * t * inv_j0) * v
        t = t * t2
        term = dn * k
        s = s + term
        if n % 6 == 5 and not bool(((term.abs() > 1e-17 * s.abs()) & torch.isfinite(s)).any()):
            break
    return torch.erfc(sz) * (_gamma_ratio_half(a) / torch.sqrt(T)) * s


def _t_two_sided_cf(q, df):
    """I_x(a, 1/2), a = df / 2, x = df / (df + q^2), by continued fractions, for the df < 20 and the far tails the
    expansion does not take.  Where x < (a + 1) / (a + 5/2) the continued fraction of I_x(a, 1/2) gives the tail
    itself; beyond, 1 - I_y(1/2, a) with y = 1 - x (Numerical Recipes' rule).  The factor x^a is
    exp(-a log1p(q^2 / df)) while log1p(q^2 / df) <= 2 (its error is then a log1p(...) ulps, the tail's own
    condition); beyond, r^df (1 + r^2)^-a with r = sqrt(df) / q, whose error is about df ulps, which is the tail's
    condition there, where the exp of a large logarithm would lose its size in ulps.  sqrt(y) = 1 / sqrt(1 + r^2), so
    neither q^2 overflowing nor q = inf yields NaN."""
    a = 0.5 * df
    q2 = q * q
    r = torch.sqrt(df) / q
    L = torch.log1p(q2 / df)
    xa = torch.where(L <= 2.0, torch.exp(-a * L), torch.pow(r, df) * torch.exp(-a * torch.log1p(r * r)))
    sy = torch.rsqrt(1.0 + r * r)
    ratio = _gamma_ratio_half(a)
    x = 1.0 / (1.0 + q2 / df)
    y = 1.0 / (1.0 + r * r)
    direct = x < (a + 1.0) / (a + 2.5)
    half = torch.full_like(q, 0.5)
    h = _beta_cf(torch.where(direct, a, half), torch.where(direct, half, a), torch.where(direct, x, y))
    tail = xa * sy * (ratio / (a * _SQRT_PI)) * h                   # I_x(a, 1/2) = x^a y^(1/2) / (a B(a, 1/2)) cf
    body = 1.0 - xa * sy * (2.0 * ratio / _SQRT_PI) * h             # 1 - y^(1/2) x^a / (B(1/2, a) / 2) cf
    return torch.where(direct, tail, body)


def _t_two_sided_finite(q, df):
    """2 pt(q, df, lower.tail = FALSE) = I_x(df / 2, 1/2) for 1-D tensors q > 0 (not NaN) and finite df > 0: the
    expansion where df >= 20 and log1p(q^2 / df) <= 1, the continued fractions elsewhere."""
    out = torch.empty_like(q)
    exp_rows = (df >= 20.0) & (torch.log1p(q * q / df) <= 1.0)
    for rows, fn in ((torch.nonzero(exp_rows).squeeze(1), _t_two_sided_expansion),
                     (torch.nonzero(~exp_rows).squeeze(1), _t_two_sided_cf)):
        if rows.numel():
            out[rows] = fn(q[rows], df[rows])
    return out


def _t_two_sided(q, df):
    """2 pt(|q|, df, lower.tail = FALSE) on broadcast tensors, and the masks of infinite and of invalid df.  Only the
    elements with a finite df > 0 and a non-NaN q reach the continued fraction."""
    q, df = torch.broadcast_tensors(q.to(F64), torch.as_tensor(df, dtype=F64, device=q.device))
    q, df = q.abs().reshape(-1), df.reshape(-1)
    inf_df = torch.isinf(df) & (df > 0)
    bad = ~(df > 0)
    out = torch.full_like(q, math.nan)
    out = torch.where(q == 0, 1.0, out)
    run = torch.nonzero(~inf_df & ~bad & (q > 0)).squeeze(1)
    if run.numel():
        out[run] = _t_two_sided_finite(q[run], df[run])
    return out, inf_df, bad


def t_upper(q, df):
    """R's pt(q, df, lower.tail = FALSE) on device tensors for any real df > 0 (q and df broadcast; df a per-gene
    vector, a tensor or a float): for q >= 0 half of the two-sided tail _t_two_sided_finite computes, for q < 0 one
    minus that.  df = Inf gives the normal tail erfc(q / sqrt 2) / 2; df NaN or <= 0 gives NaN, as R gives NA.  The
    relative error is a few ulps plus the tail's condition number |q f(q) / (1 - F(q))| in ulps down to DBL_MIN
    (DESIGN.md, p-value accuracy).  R switches to a normal approximation above df = 4e5; this stays exact there.
    The work is a masked continued fraction in torch, a few dozen steps for most elements, with one host read per
    _T_CHUNK steps."""
    shape = torch.broadcast_shapes(q.shape, torch.as_tensor(df).shape)
    qf = q.to(F64).expand(shape).reshape(-1)
    two, inf_df, bad = _t_two_sided(q, df)
    up = torch.where(qf >= 0, 0.5 * two, 1.0 - 0.5 * two)
    up = torch.where(inf_df, 0.5 * torch.erfc(qf * 0.7071067811865476), up)
    return torch.where(bad, math.nan, up).reshape(shape)


def t_wald_pvalue(stat, df):
    """nbinomWaldTest's and getContrast's useT p-value 2 pt(|stat|, df, lower.tail = FALSE) (R/core.R:1505,
    R/results.R:815) on device tensors: the two-sided tail of t_upper without the halving; rows with df = Inf get
    wald_pvalue's bits, df NaN or <= 0 gives NaN.  stat: (n,) or (p, n) with df (n,) broadcast along the last axis."""
    two, inf_df, bad = _t_two_sided(stat, df)
    shape = torch.broadcast_shapes(stat.shape, torch.as_tensor(df).shape)
    norm = wald_pvalue(stat.to(F64).expand(shape).reshape(-1))
    return torch.where(bad, math.nan, torch.where(inf_df, norm, two)).reshape(shape)


def _size_or_norm_factors(y, m, sizeFactors, normalizationFactors, weights):
    """getSizeOrNormFactors (R/core.R:2221-2228) for the fits: the checked nf matrix, or the size factors as a device
    vector.  Raises ValueError when both or neither are given, or nf together with weights."""
    if normalizationFactors is None:
        if sizeFactors is None:
            raise ValueError("give sizeFactors or normalizationFactors")
        return torch.as_tensor(np.asarray(sizeFactors, dtype=np.float64), device=y.device)
    if sizeFactors is not None:
        raise ValueError("give sizeFactors or normalizationFactors, not both")
    if weights is not None:
        raise ValueError("observation weights together with normalization factors are not supported")
    _check_positive_matrix(normalizationFactors, y, m, "normalizationFactors")
    return normalizationFactors


def _optim_fallback(ysrc, xd, sfd, dispersion, fb, beta0, lam, contrast, maxit, minmu, ll, useOptim=True,
                    weights=None):
    """R/fitNbinomGLMs.R:186-227 on device results: rows with NA coefficients or non-positive variances -- and, with
    useOptim (the reference's default), rows whose IRLS did not converge -- are refitted by b200nb_beta_optim_dev
    (fitNbinomGLMsOptim, :340-407); their coefficients, standard errors (sandwich at the clamped mean, :386-396),
    fitted means and log-likelihoods are overwritten in `fb` / `ll` in place.  The hat diagonals keep the IRLS values,
    as in the reference (:234).  With weights the objective, the sandwich and the log-likelihood are weighted
    (:343-400).  Returns betaConv (n,) bool.  Costs one host sync (the number of such rows)."""
    beta = fb["beta_mat"]                                             # (p, n), natural-log scale
    betaConv = fb["iter"] < maxit
    rowStable = ~torch.isnan(beta).any(dim=0)
    rowVarPositive = ~(fb["beta_var_mat"] <= 0).any(dim=0)
    need = (~rowStable) | (~rowVarPositive)
    if useOptim:
        need = need | (~betaConv)
    rows = torch.nonzero(need).squeeze(1)
    if rows.numel() == 0:
        return betaConv, 0
    usable = rowStable[rows] & ((beta[:, rows] / LN2).abs() < 30.0).all(dim=0)
    start = torch.where(usable[None, :], beta[:, rows], beta0[:, rows]).contiguous()
    start = torch.nan_to_num(start, nan=0.0)
    ysub = ysrc[rows].contiguous()
    sfd = _rows(sfd, rows)
    asub = dispersion[rows].contiguous()
    wsub = None if weights is None else weights[rows].contiguous()
    o = D.beta_optim(ysub, xd, sfd, asub, lam, start, weights=wsub)
    cov = D.fit_beta(ysub, xd, sfd, asub, contrast, o["beta_mat"], lam, 1e-8, 0, minmu=minmu, weights=wsub,
                     want_hat=False, want_mu=False)
    l2 = D.nb_loglik(ysub, xd, sfd, asub, o["beta_mat"], weights=wsub, want_mu=ll.get("mu") is not None,
                     minmu=minmu)
    fb["beta_mat"][:, rows] = o["beta_mat"]
    fb["beta_var_mat"][:, rows] = cov["beta_var_mat"]
    fb["contrast_num"][rows] = cov["contrast_num"]
    fb["contrast_denom"][rows] = cov["contrast_denom"]
    ll["logLike"][rows] = l2["logLike"]
    if ll.get("mu") is not None:
        ll["mu"][rows] = l2["mu"]
    betaConv = betaConv.clone()
    betaConv[rows] = betaConv[rows] | (o["converged"] != 0)
    return betaConv, int(rows.numel())


def nbinomLRT_device(ynz, x_full, x_reduced, sizeFactors, dispersion, betaTol=1e-8, maxit=100, minmu=0.5,
                     useOptim=True, weights=None, normalizationFactors=None):
    """nbinomLRT (R/core.R:1787-2012) on device tensors: two IRLS fits, LRT statistic 2 (logLike_full - logLike_reduced)
    (R/core.R:1877) and its chi-square p-value.  The log-likelihoods are evaluated at the UNCLAMPED fitted means
    nf * exp(x beta) as the reference does (R/fitNbinomGLMs.R:180-182) by b200nb_nb_loglik_dev -- NOT taken from the IRLS
    kernel's deviance, which is at the minmu-clamped mean and differs by several units when a design cell is all zeros.
    weights: gene-major (n, ld) float64 observation weights of the rows (raw or normalised): both fits, their
    log-likelihoods and the optim fallback are weighted, and an intercept-only reduced model takes the reference's
    weighted closed form (R/fitNbinomGLMs.R:99-137) instead of an IRLS fit.
    normalizationFactors: gene-major (n, ld) float64 factors of the rows, in place of sizeFactors (None then); both
    fits, their start values and log-likelihoods use them, and the intercept-only reduced model is an IRLS fit as on
    the size-factor path."""
    sfd = _size_or_norm_factors(ynz, np.asarray(x_full).shape[0], sizeFactors, normalizationFactors, weights)
    wn = None if weights is None else normalize_weights(weights, ynz, np.asarray(x_full).shape[0])
    res = {}
    for name, x in (("full", x_full), ("reduced", x_reduced)):
        res[name] = _lrt_model_fit(ynz, x, sizeFactors, sfd, dispersion, wn, closed_form=wn is not None,
                                   betaTol=betaTol, maxit=maxit, minmu=minmu, useOptim=useOptim,
                                   normalizationFactors=normalizationFactors, full=(name == "full"))
    df = x_full.shape[1] - x_reduced.shape[1]
    stat, pval = _lrt_stats(res["full"]["logLike"], res["reduced"]["logLike"], df)
    return {"LRTStatistic": stat, "LRTPvalue": pval, "deviance": -2.0 * res["full"]["logLike"], "df": df,
            "betaMatrix": (res["full"]["beta_mat"] / LN2).T,
            "betaSE": (torch.sqrt(torch.clamp(res["full"]["beta_var_mat"], min=0.0)) / LN2).T,
            "fullBetaConv": res["full"]["conv"], "reducedBetaConv": res["reduced"]["conv"],
            "mu": res["full"]["mu"], "H": res["full"]["hat_diagonals"]}


def _is_intercept_only(x):
    """fitNbinomGLMs' justIntercept for a model matrix (R/fitNbinomGLMs.R:99-103): one column, every entry 1."""
    return x.shape[1] == 1 and bool(np.all(x == 1))


def _lrt_model_fit(ynz, x, sizeFactors, sfd, dispersion, wn, closed_form, betaTol=1e-8, maxit=100, minmu=0.5,
                   useOptim=True, normalizationFactors=None, full=False):
    """One of nbinomLRT's two fitNbinomGLMs calls (R/core.R:1850-1873) on the rows of ynz: an intercept-only model by
    R's closed form when closed_form is set (_intercept_only), else the pre-step kernel's start values and _glm_fit,
    with the hat diagonals and the fitted mean only for the full model.  Returns the fitBeta result (the closed form:
    "beta_mat" only) with "conv", "logLike" and "mu" added.  The start values need no xim: it is passed as 1 so that
    the nf path makes no host read."""
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    if closed_form and _is_intercept_only(x):
        return _intercept_only(ynz, sfd, dispersion, wn, m)
    pr = prep(ynz, x, sizeFactors, minmu=minmu, want_mu=False, normalizationFactors=normalizationFactors, xim=1.0)
    contrast, lam = _mle_penalty(p, ynz.device)
    fit, ll, conv, _ = _glm_fit(ynz, pr["xd"], sfd, dispersion, contrast, pr["beta0"], lam, betaTol=betaTol,
                                maxit=maxit, minmu=minmu, useOptim=useOptim, weights=wn, want_hat=full, want_mu=full)
    fit["conv"], fit["logLike"], fit["mu"] = conv, ll["logLike"], ll["mu"]
    return fit


def _lrt_stats(ll_full, ll_reduced, df):
    """nbinomLRT's LRTStatistic = 2 (logLike_full - logLike_reduced) (R/core.R:1877) and its chi-square upper tail with
    df degrees of freedom, pchisq(stat, df, lower.tail = FALSE) (:1878): 1 for a statistic <= 0."""
    stat = 2.0 * (ll_full - ll_reduced)
    return stat, chisq_upper(stat, df)


def chisq_upper(stat, df):
    """pchisq(stat, df, lower.tail = FALSE) for an integer df >= 1 as Q(df / 2, x), x = max(stat, 0) / 2, by its
    finite sums of positive terms: Q(k, x) = e^-x sum_{j < k} x^j / j! for even df, and Q(k + 1/2, x) = erfc(sqrt x)
    + sum_{j = 1..k} e^-x x^(j - 1/2) / Gamma(j + 1/2) for odd df, each term as exp(j log x - x - lgamma).  Nothing
    cancels, so the relative error is a few ulps plus the rounding of the exponent, about x ulps.  torch's igammac
    forms Q as 1 - P for small x and loses up to 30 ulps there (DESIGN.md, p-value accuracy).  1 at stat <= 0, 0 at
    +inf, NaN at NaN."""
    x = torch.clamp(stat, min=0.0) / 2.0
    lx = torch.log(x)
    odd = df % 2 == 1
    p = torch.erfc(torch.sqrt(x)) if odd else torch.exp(-x)
    for j in range(1, (df + 1) // 2):
        a = j - 0.5 if odd else float(j)
        term = torch.exp(a * lx - x - math.lgamma(a + 1.0))
        p = p + torch.where(torch.isinf(x), 0.0, term)               # e^-x x^a at x = inf: inf - inf
    return p


def _intercept_only(ynz, sfd, dispersion, wn, m):
    """R/fitNbinomGLMs.R:99-137, no IRLS: beta = log(mean of K/nf), or log(sum(w K/nf) / sum(w)) with the normalised
    weights wn, and the log-likelihood (weighted with wn) at mu = nf e^beta by b200nb_nb_loglik_dev.  sfd: the
    size-factor vector or the gene-major nf rows of ynz."""
    dev = ynz.device
    norm = ynz[:, :m].to(F64) / (sfd[:, :m] if sfd.dim() == 2 else sfd[None, :])
    if wn is None:
        beta = torch.log(norm.mean(dim=1))
    else:
        w = wn[:, :m]
        beta = torch.log((w * norm).sum(dim=1) / w.sum(dim=1))
    beta = beta[None, :].contiguous()                                                # (1, n), natural-log scale
    ones = torch.ones((1, m), dtype=F64, device=dev)
    ll = D.nb_loglik(ynz, ones, sfd, dispersion, beta, weights=wn, want_mu=False)
    return {"beta_mat": beta, "logLike": ll["logLike"], "mu": None,
            "conv": torch.ones(ynz.shape[0], dtype=torch.bool, device=dev)}


def _dispersions_intercept_mean(ynz, m, sf, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6, maxit=100, minmu=0.5,
                                outlierSD=2.0):
    """estimateDispersions(design ~1, fitType = "mean") as estimateSizeFactorsIterate runs it (R/core.R:2594-2597):
    the pre-step kernel's clamped linear mu, then DESeq_device's stages for x = 1: _gene_est, the trimmed-mean trend,
    _disp_prior_var and _disp_map.  Returns (q = mu / sf as a fresh gene-major tensor, final dispersions, dispGeneEst,
    meanDisp, dispPriorVar)."""
    pr = prep(ynz, np.ones((m, 1)), sf, minDisp=minDisp, minmu=minmu, want_mu=True, want_beta0=False)
    xd, bm, mu = pr["xd"], pr["baseMean"], pr["mu_lin"]
    _, _, dge, _ = _gene_est(ynz, xd, pr["sfd"], pr["alpha0"], None, mu, m, minDisp=minDisp, kappa_0=kappa_0,
                             dispTol=dispTol, maxit=maxit, minmu=minmu)
    tr = _dispersion_trend(bm, dge, "mean", minDisp)
    dispFit = tr[0] + tr[1] / bm
    varLogDispEsts, dispPriorVar = _disp_prior_var(dge, dispFit, m, 1, minDisp)
    _, dispersion, _, _, _ = _disp_map(ynz, xd, mu, dge, dispFit, varLogDispEsts, dispPriorVar, m, minDisp=minDisp,
                                       kappa_0=kappa_0, dispTol=dispTol, maxit=maxit, outlierSD=outlierSD)
    q = torch.ones_like(mu)
    q[:, :m] = mu[:, :m] / pr["sfd"][None, :]
    return q, dispersion, dge, tr[0], dispPriorVar


def size_factors_iterate(y, m, niter=10, Q=0.05, minDisp=1e-8, minmu=0.5, kappa_0=1.0, dispTol=1e-6, maxit=100,
                         outlierSD=2.0, h=1e-3, max_tile_cols=0):
    """estimateSizeFactorsIterate (R/core.R:2589-2622) on the device: the rows of y (gene-major (N, ld) counts) with
    a positive sum, s = 1 to start; each outer iteration runs the dispersion chain for design ~1 with fitType "mean"
    (_dispersions_intercept_mean) and maximises the trimmed total log-likelihood over the log size factors with
    pipeline.optimizeLogSizeFactors (scipy's L-BFGS-B with optim's settings, the host mirror's driver): every
    objective call is one b200nb_sf_iterate_objective_dev launch sequence and one D2H copy of 2m + 1 doubles.  R's
    stops raise ValueError (see pipeline.iterateSizeFactors; niter = 1 always stops, as in R).
    Returns {"sizeFactors": (m,) numpy, "iterations", "evaluations": objective calls per iteration, "dispersion",
    "dispGeneEst", "meanDisp", "dispPriorVar" of the last iteration (device tensors / floats), "idx": kept rows}."""
    from .pipeline import iterateSizeFactors
    dev = y.device
    idx = torch.nonzero(y[:, :m].sum(dim=1) > 0).squeeze(1)
    ynz = y if idx.numel() == y.shape[0] else y[idx].contiguous()
    out = torch.empty(2 * m + 1, dtype=F64, device=dev)

    def step(sf):
        q, disp, dge, meanDisp, dpv = _dispersions_intercept_mean(ynz, m, sf, minDisp=minDisp, kappa_0=kappa_0,
                                                                  dispTol=dispTol, maxit=maxit, minmu=minmu,
                                                                  outlierSD=outlierSD)

        def evaluate(par):
            pd = torch.as_tensor(np.asarray(par, dtype=np.float64), device=dev)
            return sf_iterate_objective(ynz, q, disp, pd, m, h=h, Q=Q, max_tile_cols=max_tile_cols,
                                        out=out).cpu().numpy()

        return evaluate, {"dispersion": disp, "dispGeneEst": dge, "meanDisp": float(meanDisp.item()),
                          "dispPriorVar": dpv, "q": q}

    r = iterateSizeFactors(m, step, niter=niter, h=h)
    res = {"sizeFactors": r["sizeFactors"], "iterations": r["iterations"], "evaluations": r["evaluations"],
           "idx": idx}
    res.update(r["last"])
    return res


def _mle_penalty(p, dev):
    """fitNbinomGLMs' maximum-likelihood fit (R/fitNbinomGLMs.R:29-236): the contrast e1 and lambda = 1e-6 on the
    log2 scale, as (contrast, lam) device tensors."""
    contrast = torch.zeros(p, dtype=F64, device=dev)
    contrast[0] = 1.0
    return contrast, torch.full((p,), 1e-6 / LN2 ** 2, dtype=F64, device=dev)


def _gene_est(ynz, xd, sfd, alpha0, beta0, mu_lin, m, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6, maxit=100,
              betaTol=1e-8, minmu=0.5, wn=None, wdisp=None, weightThreshold=1e-2, mu_out=None, penalty=None,
              mark=lambda name: None):
    """estimateDispersionsGeneEst (R/core.R:657-860) after the pre-steps: the gene-wise mean (mu_lin, the prep
    kernel's linear mu, when it is given; else a GLM fit, weighted with R's defaults when the normalised weights wn
    are given), the fitDisp MLE, the noIncrease rule, the grid refit of the unconverged genes and the clamps.  sfd:
    the size-factor vector or the nf rows of ynz; alpha0 / beta0: the prep kernel's start values; wdisp:
    pmax(wn, 1e-6).  The GLM mean is written to mu_out, an (n, ld) buffer, or to a fresh tensor; penalty: the
    (contrast, lam) of that fit, _mle_penalty's when not given.  Returns (mu, the fitDisp result, dispGeneEst, number
    of grid refits)."""
    maxDisp = float(max(10, m))
    if mu_lin is not None:
        mu = mu_lin
    else:
        contrast, lam = penalty if penalty is not None else _mle_penalty(beta0.shape[0], ynz.device)
        if wn is not None:
            # fitNbinomGLMs with the normalised weights, its defaults minmu = 0.5 and useOptim = TRUE (R/core.R:752-755
            # passes neither), its unclamped mean nf exp(x beta) (R/fitNbinomGLMs.R:180; the optim rows' own, :383)
            # bounded at minmu (:764)
            _, ll0, _, _ = _glm_fit(ynz, xd, sfd, alpha0, contrast, beta0, lam, betaTol=betaTol, maxit=maxit, minmu=0.5,
                                    weights=wn, want_hat=False, out_mu=mu_out)
            mu = ll0["mu"].clamp_(min=minmu)
        else:
            mu = D.fit_beta(ynz, xd, sfd, alpha0, contrast, beta0, lam, betaTol, maxit, minmu=minmu, want_hat=False,
                            out_mu=mu_out)["mu"]
    la0 = torch.log(alpha0)
    mark("mu")
    r = D.fit_disp(ynz, xd, mu, la0, la0, 1.0, float(np.log(minDisp / 10)), kappa_0, dispTol, maxit, False,
                   weights=wdisp, weightThreshold=weightThreshold)
    mark("fit_disp_mle")
    dge = torch.clamp(torch.exp(r["log_alpha"]), max=maxDisp)
    noIncrease = r["last_lp"] < r["initial_lp"] + r["initial_lp"].abs() / 1e6
    dge = torch.where(noIncrease, alpha0, dge)
    conv = (r["iter"] < maxit) & (r["iter"] != 1)
    gi, ga = _grid_refit(ynz, xd, mu, (~conv) & (dge > minDisp * 10), m, None, 1.0, False, wdisp, weightThreshold)
    if ga is not None:
        dge[gi] = ga
    dge = torch.clamp(dge, minDisp, maxDisp)
    return mu, r, dge, int(gi.numel())


def _dispersion_trend(baseMean, dge, fitType, minDisp=1e-8):
    """estimateDispersionsFit's fit (R/core.R:864-940) as a 4-vector (a, b, status, rounds) with dispFit = a + b /
    baseMean: parametricDispersionFit on the device (trend_fit), or for fitType "mean" (mean_disp, 0, 0, 0), so that
    every a + b / baseMean downstream (the MAP prior, the outlier refit) equals meanDisp.  A failed parametric fit
    raises FloatingPointError (one host read; R would fall back to the local fit)."""
    if fitType == "mean":
        tr = torch.zeros(4, dtype=F64, device=dge.device)
        tr[0] = mean_disp(dge, minDisp)
        return tr
    tr = trend_fit(baseMean, dge, minDisp)
    status = tr[2].item()
    if status != 0:
        raise FloatingPointError(f"parametric dispersion fit failed on device (status {int(status)})")
    return tr


def _disp_prior_var(dge_all, dispFit_all, m, p, minDisp=1e-8):
    """varLogDispEsts as dispersionFunction<- computes it (R/methods.R:142-190: the squared MAD of the log residuals of
    the estimates >= 100 minDisp) and estimateDispersionsPriorVar (R/core.R:1135-1208), over all genes.  Returns
    (varLogDispEsts as a 0-d device tensor, dispPriorVar as a float)."""
    above = dge_all >= minDisp * 100
    resid = (torch.log(dge_all) - torch.log(dispFit_all))[above]
    med = _median(resid)
    varLogDispEsts = (1.4826 * _median((resid - med).abs())) ** 2
    if m - p <= 3 and m > p:
        # 2-vs-2 / 3-vs-2 experiments: the reference's Monte-Carlo KL match (R/core.R:1157-1193) is host glue (numpy);
        # it needs the log-dispersion residuals of all genes: one D2H of two doubles per gene
        from .pipeline import estimateDispersionsPriorVar
        dispPriorVar = estimateDispersionsPriorVar(float(varLogDispEsts.item()), m, p, dge_all.cpu().numpy(),
                                                   dispFit_all.cpu().numpy(), minDisp)
    elif m > p:
        expVar = torch.special.polygamma(1, torch.tensor((m - p) / 2.0, dtype=F64, device=dge_all.device))
        dispPriorVar = float(torch.clamp(varLogDispEsts - expVar, min=0.25).item())
    else:
        dispPriorVar = float(varLogDispEsts.item())
    return varLogDispEsts, dispPriorVar


def _disp_map(ynz, xd, mu, dge, dispFit, varLogDispEsts, dispPriorVar, m, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6,
              maxit=100, outlierSD=2.0, wn=None, weightThreshold=1e-2, mark=lambda name: None):
    """estimateDispersionsMAP (R/core.R:943-1131): dispInit, the fitDisp MAP with the log trend as prior mean, the
    grid refit of the genes at maxit, the clamps and the dispersion-outlier rule.  wn: the normalised weights.
    Returns (dispMAP, dispersion, dispOutlier, dispIter, number of grid refits)."""
    maxDisp = float(max(10, m))
    dispInit = torch.where(dge > 0.1 * dispFit, dge, dispFit)
    logFit = torch.log(dispFit)
    rm = D.fit_disp(ynz, xd, mu, torch.log(dispInit), logFit, dispPriorVar, float(np.log(minDisp / 10)), kappa_0,
                    dispTol, maxit, True, weights=wn, weightThreshold=weightThreshold)
    mark("fit_disp_map")
    dispMAP = torch.exp(rm["log_alpha"])
    gi, ga = _grid_refit(ynz, xd, mu, rm["iter"] >= maxit, m, logFit, dispPriorVar, True, wn, weightThreshold)
    if ga is not None:
        dispMAP[gi] = ga
    dispMAP = torch.clamp(dispMAP, minDisp, maxDisp)
    dispOutlier = torch.log(dge) > logFit + outlierSD * torch.sqrt(varLogDispEsts)
    dispersion = torch.where(dispOutlier, dge, dispMAP)
    return dispMAP, dispersion, dispOutlier, rm["iter"], int(gi.numel())


def _glm_fit(y, xd, sfd, dispersion, contrast, beta0, lam, betaTol=1e-8, maxit=100, minmu=0.5, useOptim=True,
             weights=None, out=None, want_hat=True, out_mu=None, want_mu=True, mark=lambda name: None):
    """fitNbinomGLMs (R/fitNbinomGLMs.R:29-236): the IRLS fit (out / want_hat: its buffers or its hat diagonals), the
    log-likelihood at the UNCLAMPED fitted mean nf * exp(x beta) that R recomputes right after the native call
    (:180-182; out_mu / want_mu: that mean's buffer or whether it is wanted), then the optim fallback (:186-227).
    Returns (the fitBeta result, the log-likelihood result, betaConv, number of optim rows)."""
    fb = D.fit_beta(y, xd, sfd, dispersion, contrast, beta0, lam, betaTol, maxit, minmu=minmu, weights=weights,
                    want_hat=want_hat, want_mu=False, out=out)
    mark("fit_beta")
    ll = D.nb_loglik(y, xd, sfd, dispersion, fb["beta_mat"], weights=weights, want_mu=want_mu, out_mu=out_mu)
    betaConv, n_optim = _optim_fallback(y, xd, sfd, dispersion, fb, beta0, lam, contrast, maxit, minmu, ll,
                                        useOptim=useOptim, weights=weights)
    return fb, ll, betaConv, n_optim


def _wald_stats(fit):
    """nbinomWaldTest's betaMatrix, betaSE, WaldStatistic and WaldPvalue (n, p) on the log2 scale from a fitBeta
    result."""
    betaMatrix = fit["beta_mat"] / LN2                     # (p, n)
    betaSE = torch.sqrt(torch.clamp(fit["beta_var_mat"], min=0.0)) / LN2
    stat = betaMatrix / betaSE
    return {"betaMatrix": betaMatrix.T, "betaSE": betaSE.T, "WaldStatistic": stat.T,
            "WaldPvalue": wald_pvalue(stat).T}


def DESeq_device(y, x, sizeFactors=None, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6, maxit=100, betaTol=1e-8, minmu=0.5,
                 outlierSD=2.0, minReplicatesForReplace=np.inf, allgather=None, useOptim=True, betaPrior=False,
                 factors=None, weights=None, weightThreshold=1e-2, normalizationFactors=None, avgTxLength=None,
                 nfXim=None, sfType="ratio", fitType="parametric", test="Wald", reduced=None, useT=False, df=None):
    """y: gene-major (N, ld) device tensor of counts (int32 or float64).  Returns a dict of device tensors over the
    rows with a non-zero sum (`idx` maps them back to the N input rows) plus the trend / prior scalars.
    sizeFactors: (m,) numpy or a device tensor (read to the host once); None estimates them on the device first
    (median of ratios, R/core.R:535-578; returned under "sizeFactors").  minReplicatesForReplace: the reference's default is 7 (replace count outliers by the trimmed mean
    and refit those genes, R/core.R:419-426, 2069-2115, 2484-2565); the default here is Inf = off (what bench.py's
    full_pipeline times).  With a finite value the per-gene results of the refitted rows are overwritten in place
    and "replace" / "replaceable" / "n_replaced" are added.
    allgather: for the gene-sharded multi-GPU run (deseq2_b200/sharded.py::sharded_DESeq_device): a callable that
    concatenates each of a LIST of per-gene 1-D device tensors over the ranks, in rank order (one collective).  It is used at the one point where the
    reference needs every gene (R/parallel.R:25-28): the dispersion trend and the prior variance are then fitted,
    identically on every rank, to all genes' baseMean / dispGeneEst instead of the shard's.  With betaPrior it is
    called once more, for the MLE coefficients the prior variance is estimated from (R/parallel.R:39-40).
    betaPrior=True: nbinomWaldTest with a zero-centred normal prior on the coefficients (fitGLMsWithPrior,
    R/fitNbinomGLMs.R:242-337) for an additive factor design: `factors` are the level-code vectors of
    pipeline.factorDesign and x must be factorDesign(factors)[0].  The dispersions and the MLE fit (whose mu / H give
    Cook's distances) are on x; the prior variance comes from the MLE log2 fold changes (estimate_beta_prior_var) and
    the reported coefficients, standard errors, Wald statistics and deviance from the MAP fit on the expanded matrix
    factorDesign(factors, expanded=True)[0] with lambda = 1 / betaPriorVar.  Adds "mleBetaMatrix", "betaPriorVar" and
    "modelMatrix" (the expanded matrix).
    weights: observation weights (the "weights" assay) as a gene-major (N, ld) float64 device tensor aligned with y.
    getAndCheckWeights (R/core.R:2697-2752) runs in the weighted prep kernel: rows with a negative, NaN or infinite
    weight or no positive weight raise ValueError, and rows whose weights leave the design rank deficient
    ("weightsFail", over the N input rows; a warning as in R) are dropped with the all-zero rows.  baseMean / baseVar
    use the raw weights; mu comes from a weighted GLM fit (no linear mu); the gene-wise fitDisp / fitDispGrid get
    max(w, 1e-6), every other fit the normalised weights, returned under "weights" for the rows in idx.  Weights are
    not supported with betaPrior=True or outlier replacement (ValueError).
    normalizationFactors: gene-specific normalization factors (the "normalizationFactors" assay) as a gene-major
    (N, ld) float64 device tensor aligned with y, finite and > 0 in the first m columns; they take the place of the size
    factors everywhere (getSizeOrNormFactors): baseMean / baseVar, rough dispersion, linear mu and start values of
    K/nf, xim = mean(1 / colMeans(nf)) over the non-all-zero rows, and the nf rows of idx in every fit, Cook's
    distances and outlier replacement.  avgTxLength (same layout, instead of normalizationFactors): the factors are
    estimated first by normalization_factors, as DESeq() -> estimateSizeFactors does for a tximport dataset.  Returned
    under "normalizationFactors" (rows in idx).  Not with sizeFactors or weights (ValueError).  nfXim: xim computed
    by the caller (the sharded driver, over every rank's rows).
    sfType: the estimator used when none of sizeFactors, normalizationFactors and avgTxLength is given: "ratio" (the
    default), "poscounts", or "iterate" (size_factors_iterate with its defaults, whatever minmu / minDisp this call
    uses, as DESeq() -> estimateSizeFactors does; its iteration and objective-call counts are returned under
    "sfIterate").  "iterate" with weights, normalizationFactors or avgTxLength raises ValueError.
    fitType: "parametric" (the default; "trendCoefs") or "mean": dispFit is the trimmed mean of the gathered
    gene-wise estimates (mean_disp, no extra collective), reported under "meanDisp" instead of "trendCoefs".  Both
    are reported under "fitType".
    test="LRT", reduced=<(m, p_r) numpy model matrix nested in x>: DESeq(test = "LRT") with matrices (R/core.R:318-341,
    nbinomLRT :1787-2012).  The dispersions and the fit on x are the Wald path's: that fit is nbinomLRT's full fit (the
    same fitNbinomGLMs call), so its mu / H give the Cook's distances and the Wald columns stay, as R's
    results(test = "Wald") derives them from an LRT object (makeWaldTest, R/results.R:1101-1116).  One more fit on the
    same rows, dispersions, minmu, useOptim and weights is added: R's closed form when reduced is ~1
    (R/fitNbinomGLMs.R:99-137, no IRLS), else the pre-step kernel's start values and an IRLS fit with the optim
    fallback.  Adds "LRTStatistic" = 2 (logLike_full - logLike_reduced), "LRTPvalue" (chi-square upper tail, df = p -
    p_r), "df", "fullBetaConv" (= betaConv), "reducedBetaConv" and "reducedModelMatrix".  With outlier replacement the
    refitted rows get the reduced fit too and their LRT columns are overwritten (R/core.R:2530-2531).  R's stops
    raise ValueError: no reduced, betaPrior=True, p_r >= p, a model matrix that is not full rank, and reduced with
    test="Wald".  "test" reports the test ("Wald" or "LRT") for results_device.
    useT=True (test="Wald"; ignored by the LRT, as in R): nbinomWaldTest's Student t p-values (R/core.R:1478-1508):
    every WaldPvalue column is 2 pt(|stat|, df, lower.tail = FALSE) (t_wald_pvalue) and "tDegreesFreedom" (rows in
    idx) is added, which results_device / getContrast_device then use.  df: a scalar or one value per input row (the
    rows of y), subset to idx; by default m - p (p = ncol(x), the standard design's count also with betaPrior), with
    weights the row sums of the normalised weights minus p.  df <= 0 or NaN gives NaN (R's NA).  The rows an outlier
    refit replaces get normal p-values and keep the first fit's df, as refitWithoutOutliers does (it does not pass
    useT on); rows whose replaced counts are all zero get NaN."""
    dev = y.device
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    if isinstance(sizeFactors, torch.Tensor):       # e.g. size_factors' or sharded_size_factors_device's device tensor
        sizeFactors = sizeFactors.cpu().numpy()
    reduced = check_test_args(x, test, reduced, betaPrior)
    if sfType not in ("ratio", "poscounts", "iterate"):
        raise ValueError("sfType must be 'ratio', 'poscounts' or 'iterate'")
    if fitType not in ("parametric", "mean"):
        raise ValueError("fitType must be 'parametric' or 'mean'")
    if sfType == "iterate" and sizeFactors is None and (weights is not None or normalizationFactors is not None
                                                        or avgTxLength is not None):
        raise ValueError("sfType='iterate' is not supported with observation weights, normalizationFactors or "
                         "avgTxLength")
    sfIterate = None
    if avgTxLength is not None:
        if normalizationFactors is not None:
            raise ValueError("give normalizationFactors or avgTxLength, not both")
        if sizeFactors is not None:
            raise ValueError("avgTxLength estimates normalization factors: sizeFactors must be None")
        normalizationFactors = normalization_factors(y, m, avgTxLength=avgTxLength)["normalizationFactors"]
    nf = normalizationFactors
    if nf is not None:
        _size_or_norm_factors(y, m, sizeFactors, nf, weights)
    if weights is not None:
        _check_weights_tensor(weights, y)
        if betaPrior:
            raise ValueError("observation weights are not supported with betaPrior=True")
        if np.isfinite(minReplicatesForReplace):
            raise ValueError("observation weights are not supported with outlier replacement "
                             "(finite minReplicatesForReplace)")
    if betaPrior:
        from .pipeline import factorDesign
        if factors is None:
            raise ValueError("betaPrior=True needs the design factors (factors=...)")
        if not np.array_equal(x, factorDesign(factors)[0]):
            raise ValueError("betaPrior=True: x must be the standard model matrix of the factors, factorDesign(factors)[0]")
        if np.isfinite(minReplicatesForReplace):
            raise ValueError("outlier replacement (finite minReplicatesForReplace) is not supported with betaPrior=True")
    estimated = sizeFactors is None and nf is None
    if estimated:
        if sfType == "iterate":
            # DESeq() passes none of its dispersion / fit arguments to estimateSizeFactors: the iterate estimator's
            # estimateDispersions call runs with its own defaults (minmu = 0.5, R/core.R:388, 2596, 662)
            sfIterate = size_factors_iterate(y, m)
            sizeFactors = sfIterate["sizeFactors"]
        elif sfType == "poscounts":
            sf = size_factors(y, m, type="poscounts")["sizeFactors"]
            sizeFactors = (sf / torch.exp(torch.log(sf).mean())).cpu().numpy()   # incoming geoMeans (R/core.R:573-576)
        else:
            sizeFactors = size_factors(y, m)["sizeFactors"].cpu().numpy()
    import os
    import time
    stage_ms = {}
    _t = [time.perf_counter()]
    debug = bool(os.environ.get("B200NB_PIPE_DEBUG"))

    def mark(name):
        if debug:
            torch.cuda.synchronize()
            now = time.perf_counter()
            stage_ms[name] = round((now - _t[0]) * 1e3, 3)
            _t[0] = now

    linearMu = modelMatrixGroups(x) == p and weights is None
    wn = wdisp = weightsFail = None
    if weights is None:
        # rows with a zero sum are dropped before anything else (R/core.R:706), so every later array is aligned
        idx = torch.nonzero(y[:, :m].sum(dim=1) != 0).squeeze(1)
        ynz = y if idx.numel() == y.shape[0] else y[idx].contiguous()
        nfz = None if nf is None else (nf if idx.numel() == y.shape[0] else nf[idx].contiguous())
        pr = prep(ynz, x, sizeFactors, minDisp=minDisp, minmu=minmu, want_mu=linearMu, normalizationFactors=nfz,
                  xim=nfXim)
        bm = pr["baseMean"]
        alpha0 = pr["alpha0"]
        beta0 = pr["beta0"]
    else:
        # the weighted prep runs on all rows: getAndCheckWeights checks every row and its weightsFail rows join the
        # all-zero rows (R/core.R:2733-2736) before the same drop
        pr = prep(y, x, sizeFactors, minDisp=minDisp, minmu=minmu, want_mu=False, weights=weights,
                  weightThreshold=weightThreshold)
        weightsFail = pr["weightsFail"] != 0
        keep = (pr["allZero"] == 0) & ~weightsFail
        n_bad, n_fail = (int(v) for v in torch.stack([pr["status"][0].to(torch.int64),
                                                       weightsFail.sum()]).cpu().tolist())
        if n_bad:
            raise ValueError(f"{n_bad} row(s) of weights have a negative, NaN or infinite weight or no positive weight")
        if n_fail:
            import warnings
            warnings.warn(f"for {n_fail} row(s), the weights as supplied won't allow parameter estimation, producing "
                          "a degenerate design matrix. These rows have been flagged in weightsFail and treated as if "
                          "the row contained all zeros.")
        idx = torch.nonzero(keep).squeeze(1)
        if idx.numel() == y.shape[0]:
            ynz, bm, alpha0, beta0, wn = y, pr["baseMean"], pr["alpha0"], pr["beta0"], pr["weightsNorm"]
        else:
            ynz, bm, alpha0 = y[idx].contiguous(), pr["baseMean"][idx], pr["alpha0"][idx]
            beta0, wn = pr["beta0"][:, idx].contiguous(), pr["weightsNorm"][idx].contiguous()
        wdisp = torch.clamp(wn, min=1e-6)                   # pmax(weights, 1e-6) for the gene-wise estimate (:702)
    xd, sfd = pr["xd"], pr["sfd"]
    contrast, lam = _mle_penalty(p, dev)

    # ---- estimateDispersionsGeneEst (R/core.R:657-860)
    mu_glm = None if linearMu else _ws("mu_glm", tuple(ynz.shape), F64, dev)
    mu, r, dge, n_refit_geneest = _gene_est(ynz, xd, sfd, alpha0, beta0, pr["mu_lin"], m, minDisp=minDisp,
                                            kappa_0=kappa_0, dispTol=dispTol, maxit=maxit, betaTol=betaTol,
                                            minmu=minmu, wn=wn, wdisp=wdisp, weightThreshold=weightThreshold,
                                            mu_out=mu_glm, penalty=(contrast, lam), mark=mark)
    mark("rules+grid_mle")

    # ---- estimateDispersionsFit + dispersionFunction<- + PriorVar (R/core.R:864-940, R/methods.R:142-190, R/core.R:1135-1208)
    # ONE packed collective for the two vectors the global step needs (sharded.PackedGather accepts a list)
    bm_all, dge_all = allgather([bm, dge]) if allgather is not None else (bm, dge)
    tr = _dispersion_trend(bm_all, dge_all, fitType, minDisp)
    dispFit, dispFit_all = tr[0] + tr[1] / bm, tr[0] + tr[1] / bm_all
    varLogDispEsts, dispPriorVar = _disp_prior_var(dge_all, dispFit_all, m, p, minDisp)
    mark("trend+priorvar")

    # ---- estimateDispersionsMAP (R/core.R:943-1131)
    dispMAP, dispersion, dispOutlier, dispIter, n_refit_map = _disp_map(
        ynz, xd, mu, dge, dispFit, varLogDispEsts, dispPriorVar, m, minDisp=minDisp, kappa_0=kappa_0, dispTol=dispTol,
        maxit=maxit, outlierSD=outlierSD, wn=wn, weightThreshold=weightThreshold, mark=mark)
    mark("rules+grid_map")

    # ---- nbinomWaldTest (R/core.R:1332-1565) via fitNbinomGLMs (R/fitNbinomGLMs.R:29-236)
    nn, ldd = ynz.shape
    outb = {"beta_mat": torch.empty((p, nn), dtype=F64, device=dev), "beta_var_mat": torch.empty((p, nn), dtype=F64, device=dev),
            "iter": torch.empty(nn, dtype=F64, device=dev), "contrast_num": torch.empty(nn, dtype=F64, device=dev),
            "contrast_denom": torch.empty(nn, dtype=F64, device=dev), "deviance": torch.empty(nn, dtype=F64, device=dev),
            "hat_diagonals": _ws("H", (nn, ldd), F64, dev), "mu": None}
    # Cook's distances and the reported deviance use the UNCLAMPED fitted mean nf * exp(x beta) and the log-likelihood
    # at it (one small kernel, b200nb_nb_loglik_dev); the IRLS kernel's fused mean / deviance are at the minmu clamp.
    # Rows the IRLS could not fit go to the box-constrained maximiser (R/fitNbinomGLMs.R:203-227, useOptim = TRUE).
    fb, ll, betaConv, n_optim = _glm_fit(ynz, xd, sfd, dispersion, contrast, beta0, lam, betaTol=betaTol, maxit=maxit,
                                         minmu=minmu, useOptim=useOptim, weights=wn, out=outb,
                                         out_mu=_ws("mu_cooks", (nn, ldd), F64, dev), mark=mark)
    mark("loglik+optim")
    fit, fit_ll, prior = fb, ll, {}
    if betaPrior:
        fit, fit_ll, betaConv, prior = _fit_with_prior(ynz, factors, sfd, dispersion, fb, bm, bm_all, dispFit_all,
                                                       allgather, betaTol, maxit, minmu, useOptim)
        mark("beta_prior_var+fit_beta_map")
    from .pipeline import nOrMoreInCell
    do_replace = bool(np.isfinite(minReplicatesForReplace)) and bool(nOrMoreInCell(x, minReplicatesForReplace).any())
    mu_cooks = ll["mu"]
    ck = cooks(ynz, mu_cooks, fb["hat_diagonals"], x, sizeFactors, want_matrix=do_replace,   # R/core.R:1457-1460
               normalizationFactors=sfd if nf is not None else None)
    mark("wald_stats+cooks")
    lrt = {}
    if test == "LRT":
        # nbinomLRT (R/core.R:1850-1877): the fit above is its full fit; only the reduced model is fitted here
        red = _lrt_model_fit(ynz, reduced, sizeFactors, sfd, dispersion, wn, closed_form=True, betaTol=betaTol,
                             maxit=maxit, minmu=minmu, useOptim=useOptim, normalizationFactors=sfd if nf is not None
                             else None)
        df = p - reduced.shape[1]
        stat, pval = _lrt_stats(fit_ll["logLike"], red["logLike"], df)
        lrt = {"LRTStatistic": stat, "LRTPvalue": pval, "df": df, "reducedBetaConv": red["conv"],
               "reducedModelMatrix": reduced}
        mark("lrt_reduced_fit")
    res = {"stage_ms": stage_ms, "maxCooks": ck["maxCooks"], "idx": idx, "baseMean": bm, "dispGeneEst": dge, "dispFit": dispFit, "dispMAP": dispMAP,
            "dispersion": dispersion, "dispOutlier": dispOutlier, "dispGeneIter": r["iter"], "dispIter": dispIter,
            **_wald_stats(fit),
            "betaIter": fit["iter"], "betaConv": betaConv, "n_optim": n_optim, "deviance": -2.0 * fit_ll["logLike"], "mu": mu_cooks,
            "H": fb["hat_diagonals"], "varLogDispEsts": varLogDispEsts,
            "dispPriorVar": dispPriorVar, "n_refit_geneest": n_refit_geneest, "n_refit_map": n_refit_map,
            "n_input_rows": y.shape[0],
            "sizeFactors": None if nf is not None else np.asarray(sizeFactors, dtype=np.float64), "fitType": fitType,
            "test": test, **lrt}
    if fitType == "mean":
        res["meanDisp"] = float(tr[0].item())
    else:
        res["trendCoefs"] = tr[:2]
    if sfIterate is not None:
        res["sfIterate"] = {"iterations": sfIterate["iterations"], "evaluations": sfIterate["evaluations"]}
    res.update(prior)
    if weights is not None:
        res["weightsFail"], res["weights"] = weightsFail, wn
    if nf is not None:
        res["normalizationFactors"] = sfd
    if useT and test == "Wald":
        res["tDegreesFreedom"] = t_degrees_freedom(df, y.shape[0], idx, m, p, wn)
        res["WaldPvalue"] = t_wald_pvalue(res["WaldStatistic"], res["tDegreesFreedom"][:, None])
    if do_replace and m > p:
        _replace_and_refit(res, ynz, ck["cooks"], x, sizeFactors, sfd, tr, minReplicatesForReplace, minDisp=minDisp,
                           kappa_0=kappa_0, dispTol=dispTol, maxit=maxit, betaTol=betaTol, minmu=minmu,
                           outlierSD=outlierSD, useOptim=useOptim, reduced=reduced if test == "LRT" else None)
    if test == "LRT":
        res["fullBetaConv"] = res["betaConv"]
    return res


def t_degrees_freedom(df, N, idx, m, p, wn=None):
    """nbinomWaldTest's t degrees of freedom (R/core.R:1478-1504) for the rows idx of N input rows, as an (n,)
    device tensor: a given df (a scalar, or one value per input row, subset to idx), else m - p, or with the
    normalised weights wn of the rows rowSums(wn) - p; NaN where it is not > 0 (ifelse(df > 0, df, NA))."""
    dev = idx.device
    n = idx.numel()
    if df is None:
        tdf = (wn[:, :m].sum(dim=1) if wn is not None else torch.full((n,), float(m), dtype=F64, device=dev)) - p
    else:
        d = torch.as_tensor(df, dtype=F64).to(dev).reshape(-1)
        if d.numel() == 1:
            tdf = d.expand(n).clone()
        elif d.numel() == N:
            tdf = d[idx]
        else:
            raise ValueError(f"df must be a scalar or have one value per row of the counts ({N}), got {d.numel()}")
    return torch.where(tdf > 0, tdf, math.nan)


def _fit_with_prior(ynz, factors, sfd, dispersion, mle, bm, bm_all, dispFit_all, allgather, betaTol, maxit, minmu,
                    useOptim):
    """The betaPrior half of fitGLMsWithPrior (R/fitNbinomGLMs.R:242-337) after the MLE fit `mle`: prior variance
    over all genes, then the MAP fit on the expanded matrix, its log-likelihood and the optim fallback with the same
    lambda.  Returns (fit, loglik, betaConv, extra result entries)."""
    from .pipeline import factorDesign
    p = mle["beta_mat"].shape[0]
    mleBeta = mle["beta_mat"] / LN2                                     # (p, n), log2 scale
    if allgather is not None:
        # ONE packed collective: the p - 1 non-intercept MLE columns of every gene; the intercept's prior is fixed
        g = allgather([mleBeta[k] for k in range(1, p)])
        beta_all = torch.stack([torch.zeros_like(g[0])] + list(g))
    else:
        beta_all = mleBeta
    pv = estimate_beta_prior_var(beta_all.T, factors, bm_all, dispFit_all)
    x_exp = factorDesign(factors, expanded=True)[0]
    fit, ll, betaConv, n_optim = _map_fit(ynz, x_exp, sfd, dispersion, pv, _expanded_start(bm, x_exp.shape[1]),
                                          betaTol, maxit, minmu, useOptim)
    return fit, ll, betaConv, {"mleBetaMatrix": mleBeta.T, "betaPriorVar": pv.cpu().numpy(), "modelMatrix": x_exp,
                               "n_optim_map": n_optim}


def _expanded_start(bm, pe):
    """The start values of a fit on the rank-deficient expanded matrix: (log baseMean, 0, ..., 0) per gene
    (R/fitNbinomGLMs.R:146-151), as a (pe, n) device tensor."""
    beta0 = torch.zeros((pe, bm.numel()), dtype=F64, device=bm.device)
    beta0[0] = torch.log(bm)
    return beta0


def _map_fit(ynz, x, sfd, dispersion, betaPriorVar, beta0, betaTol, maxit, minmu, useOptim, weights=None):
    """fitGLMsWithPrior's refit (R/fitNbinomGLMs.R:311-330): fitNbinomGLMs on the model matrix x (numpy) with
    lambda = 1 / betaPriorVar ((p,) device tensor, log2 scale) from the start values beta0 ((p, n), natural log): the
    IRLS fit, the log-likelihood at the unclamped mean and the optim fallback with the same lambda.  weights: the
    normalised observation weights of the rows.  Returns _glm_fit's (fit, loglik, betaConv, number of optim rows)."""
    p = x.shape[1]
    lam = 1.0 / (LN2 ** 2 * betaPriorVar)
    contrast = torch.zeros(p, dtype=F64, device=ynz.device)
    contrast[0] = 1.0
    return _glm_fit(ynz, D.x_to_device(x, ynz.device), sfd, dispersion, contrast, beta0, lam, betaTol=betaTol,
                    maxit=maxit, minmu=minmu, useOptim=useOptim, weights=weights, want_hat=False, want_mu=False)


def _replacement_counts(ys, nfm, over, replaceable, m, trim=0.2):
    """replaceOutliers' new counts (R/core.R:2069-2115) of the rows ys ((k, m) float64 counts, nfm their factors):
    the outlying entries (`over`) of replaceable samples become as.integer(trimmed mean of K / nf * nf)."""
    srt, _ = torch.sort(ys / nfm, dim=1)
    lo = int(np.floor(m * trim))
    tbm = srt[:, lo:m - lo].mean(dim=1)
    replacement = torch.trunc(tbm[:, None] * nfm)
    return torch.where(over & replaceable[None, :], replacement, ys)


def _replace_and_refit(res, ynz, cooksm, x, sizeFactors, sfd, tr, minReplicates, minDisp=1e-8, kappa_0=1.0,
                       dispTol=1e-6, maxit=100, betaTol=1e-8, minmu=0.5, outlierSD=2.0, useOptim=True, trim=0.2,
                       reduced=None):
    """replaceOutliers + refitWithoutOutliers (R/core.R:2069-2115, 2484-2565) on the device results `res` (in place).
    Only the flagged rows move: their counts are gathered, the outlying entries of replaceable samples become
    as.integer(trimmed mean of the normalised counts * size factor), and the rows go through DESeq_device's stages
    (GeneEst -> MAP -> Wald) with the trend `tr` and res's prior variance, as refitWithoutOutliers does with
    objectSub.  `sfd` is the size-factor vector or the nf matrix of ynz's rows: with nf the trimmed mean is of K/nf
    and the replacement count trunc(trimmed mean * nf_ij) (R/core.R:2089-2096).  reduced (test="LRT"): the rows also
    get the reduced fit and their LRT columns are overwritten, as nbinomLRT(objectSub) does (R/core.R:2530-2531).
    Every fit here takes DESeq_device's minmu, where R's refit passes none (0.5)."""
    from scipy import stats as _st
    from .pipeline import nOrMoreInCell
    dev = ynz.device
    m, p = x.shape
    cutoff = float(_st.f.ppf(0.99, p, m - p))
    replaceable = torch.as_tensor(nOrMoreInCell(x, minReplicates), device=dev)
    over = cooksm[:, :m] > cutoff                                   # NaN compares false, like NA in which()/any()
    replace = over.any(dim=1)
    rows = torch.nonzero(replace).squeeze(1)
    res["replace"], res["replaceable"], res["n_replaced"] = replace, replaceable, int(rows.numel())
    if rows.numel() == 0:
        return
    ys = ynz[rows][:, :m].to(F64)
    nfm = sfd[rows][:, :m] if sfd.dim() == 2 else sfd[None, :]
    new = _replacement_counts(ys, nfm, over[rows], replaceable, m, trim)
    res["baseMean"] = res["baseMean"].clone()
    res["baseMean"][rows] = (new / nfm).mean(dim=1)                 # getBaseMeansAndVariances on the new counts
    newAllZero = new.sum(dim=1) == 0
    keep = ~newAllZero
    rr = rows[keep]
    if rr.numel() > 0:
        ysub = torch.zeros((rr.numel(), ynz.shape[1]), dtype=F64, device=dev)
        ysub[:, :m] = new[keep]
        # no mu_out: a GLM mean of the subset goes to a fresh tensor, not into the full-size "mu_glm" workspace; with
        # nf, xim is over the subset's rows, as estimateDispersionsGeneEst(objectSub) computes it (R/core.R:2503-2510)
        pr = prep(ysub, x, sizeFactors, minDisp=minDisp, minmu=minmu, want_mu=modelMatrixGroups(x) == p,
                  normalizationFactors=sfd[rr].contiguous() if sfd.dim() == 2 else None)
        xd, sfs, beta0 = pr["xd"], pr["sfd"], pr["beta0"]
        contrast, lam = _mle_penalty(p, dev)
        mu, r, dge, _ = _gene_est(ysub, xd, sfs, pr["alpha0"], beta0, pr["mu_lin"], m, minDisp=minDisp,
                                  kappa_0=kappa_0, dispTol=dispTol, maxit=maxit, betaTol=betaTol, minmu=minmu,
                                  penalty=(contrast, lam))
        dispFit = tr[0] + tr[1] / pr["baseMean"]
        dispMAP, dispersion, dispOutlier, dispIter, _ = _disp_map(
            ysub, xd, mu, dge, dispFit, res["varLogDispEsts"], res["dispPriorVar"], m, minDisp=minDisp,
            kappa_0=kappa_0, dispTol=dispTol, maxit=maxit, outlierSD=outlierSD)
        fb, ll, betaConv, _ = _glm_fit(ysub, xd, sfs, dispersion, contrast, beta0, lam, betaTol=betaTol, maxit=maxit,
                                       minmu=minmu, useOptim=useOptim, want_hat=False, want_mu=False)
        sub = {"dispGeneEst": dge, "dispFit": dispFit, "dispMAP": dispMAP, "dispersion": dispersion,
               "dispOutlier": dispOutlier, "dispGeneIter": r["iter"], "dispIter": dispIter, **_wald_stats(fb),
               "betaIter": fb["iter"], "betaConv": betaConv, "deviance": -2.0 * ll["logLike"]}
        results_cols = ["betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "deviance"]
        if reduced is not None:
            red = _lrt_model_fit(ysub, reduced, sizeFactors, sfs, dispersion, None, closed_form=True, betaTol=betaTol,
                                 maxit=maxit, minmu=minmu, useOptim=useOptim,
                                 normalizationFactors=sfs if sfd.dim() == 2 else None)
            sub["LRTStatistic"], sub["LRTPvalue"] = _lrt_stats(ll["logLike"], red["logLike"], res["df"])
            sub["reducedBetaConv"] = red["conv"]
            results_cols += ["LRTStatistic", "LRTPvalue"]
        if "tDegreesFreedom" in res:                    # a "results" column, kept for the refitted rows (:2524-2534)
            results_cols.append("tDegreesFreedom")
        for k, v in sub.items():
            res[k] = res[k].clone()
            res[k][rr] = v.to(res[k].dtype)
        for k in results_cols:
            res[k][rows[newAllZero]] = float("nan")
        if bool(replaceable.all()):
            res["maxCooks"] = torch.full_like(res["maxCooks"], float("nan"))
        else:                                   # replaceCooks[, replaceable] <- 0, then recordMaxCooks (:2537-2543)
            from .pipeline import designCells
            cells, sizes = designCells(x)
            forCooks = torch.as_tensor(sizes[cells] >= 3, device=dev)
            rc = cooksm[:, :m].clone()
            rc[:, replaceable] = 0.0
            res["maxCooks"] = (rc[:, forCooks].max(dim=1).values if bool(forCooks.any())
                               else torch.full_like(res["maxCooks"], float("nan")))


# ---------------------------------------------------------------- transforms: vst(), varianceStabilizingTransformation(),
# normTransform() (R/vst.R, R/helper.R:421-435)

_TRANSFORM_MODE = {"parametric": 0, "mean": 1, "log2": 2}     # B200NB_TRANSFORM_* of include/b200nb.h


def transform(y, m, mode, c0, c1, sfd):
    """b200nb_transform_dev: a fresh contiguous (N, m) float64 device tensor of the transformed normalized counts
    K / s_j (sfd: the (m,) size-factor device vector) or K / nf_ij (sfd: the gene-major (N, ld) nf matrix) of all N
    rows of y.  mode "parametric" (c0 = asymptDisp, c1 = extraPois), "mean" (c0 = the mean dispersion) or "log2"
    (c0 = the pseudocount).  Enqueue only."""
    if y.dim() != 2 or y.dtype not in (torch.int32, F64) or not y.is_contiguous():
        raise ValueError("y must be a contiguous gene-major int32 or float64 tensor")
    L = _lib.lib()
    n, ld = y.shape
    out = torch.empty((n, m), dtype=F64, device=y.device)
    sf, nf = D._split_factors(sfd)
    _lib.check(L.b200nb_transform_dev(D._p(y), D._ytype(y), D._p(sf), D._p(nf), n, m, ld,
                                      _TRANSFORM_MODE[mode], float(c0), float(c1), D._p(out), m, D._stream()),
               "transform_dev")
    return out


def _vst_constants(dispersionFunction):
    """(mode, c0, c1) of b200nb_transform_dev for a dispersion function given as DESeq_device returns it."""
    fitType = dispersionFunction.get("fitType")
    if fitType == "parametric":
        a = dispersionFunction["trendCoefs"]
        a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64)
        return "parametric", float(a[0]), float(a[1])
    if fitType == "mean":
        return "mean", float(dispersionFunction["meanDisp"]), 0.0
    raise ValueError(f"fitType {fitType!r}: only 'parametric' and 'mean' dispersion functions have a variance "
                     "stabilizing transformation here (there is no 'local' trend fit)")


def _check_vst_fit_type(fitType):
    if fitType not in ("parametric", "mean"):
        raise ValueError(f"fitType must be 'parametric' or 'mean' (there is no 'local' trend fit), got {fitType!r}")


def _factors(y, m, sizeFactors, normalizationFactors, avgTxLength=None):
    """The normalization of R's transforms: normalizationFactors, or those estimated from avgTxLength (as DESeq_device
    does), or sizeFactors (numpy or a device tensor), or, when none is given, the median-of-ratios size factors
    (estimateSizeFactors).  Returns (size factors as numpy or None, nf matrix or None, the factors as sfd for
    transform / the fits)."""
    if avgTxLength is not None:
        if normalizationFactors is not None:
            raise ValueError("give normalizationFactors or avgTxLength, not both")
        if sizeFactors is not None:
            raise ValueError("avgTxLength estimates normalization factors: sizeFactors must be None")
        normalizationFactors = normalization_factors(y, m, avgTxLength=avgTxLength)["normalizationFactors"]
    if sizeFactors is None and normalizationFactors is None:
        sizeFactors = size_factors(y, m)["sizeFactors"]
    if sizeFactors is not None:
        sizeFactors = (sizeFactors.cpu().numpy() if isinstance(sizeFactors, torch.Tensor)
                       else np.asarray(sizeFactors, dtype=np.float64))
        if sizeFactors.shape != (m,):
            raise ValueError(f"sizeFactors must have one value per sample ({m}), got shape {sizeFactors.shape}")
    sfd = _size_or_norm_factors(y, m, sizeFactors, normalizationFactors, None)
    return sizeFactors, normalizationFactors, sfd


def _vst_design(x, m, blind):
    """~1 when blind, else the given design (m rows)."""
    if blind:
        return np.ones((m, 1))
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 2 or x.shape[0] != m:
        raise ValueError(f"x must be a design matrix with one row per sample ({m}), got shape {x.shape}")
    return x


def gene_wise_dispersions(ynz, x, sizeFactors, nfz, xim=None, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6, maxit=100,
                          betaTol=1e-8, minmu=0.5):
    """estimateDispersionsGeneEst with its defaults on the rows of ynz (none of them all-zero; nfz: their nf rows, xim
    over them unless given): the pre-step kernel and _gene_est, as in DESeq_device.  Returns (baseMean, dispGeneEst)."""
    m, p = x.shape
    linearMu = modelMatrixGroups(x) == p
    pr = prep(ynz, x, sizeFactors, minDisp=minDisp, minmu=minmu, want_mu=linearMu, normalizationFactors=nfz, xim=xim)
    mu_glm = None if linearMu else _ws("mu_glm", tuple(ynz.shape), F64, ynz.device)
    _, _, dge, _ = _gene_est(ynz, pr["xd"], pr["sfd"], pr["alpha0"], pr["beta0"], pr["mu_lin"], m, minDisp=minDisp,
                             kappa_0=kappa_0, dispTol=dispTol, maxit=maxit, betaTol=betaTol, minmu=minmu,
                             mu_out=mu_glm)
    return pr["baseMean"], dge


def dispersion_function_of(baseMean, dge, fitType, minDisp=1e-8):
    """estimateDispersionsFit (_dispersion_trend) as a dispersion function: {"fitType", "trendCoefs" (device (2,)) or
    "meanDisp" (float)}.  A failed parametric fit raises FloatingPointError (R would fall back to the local fit)."""
    tr = _dispersion_trend(baseMean, dge, fitType, minDisp)
    if fitType == "mean":
        return {"fitType": "mean", "meanDisp": float(tr[0].item())}
    return {"fitType": "parametric", "trendCoefs": tr[:2].clone()}


def _dispersion_function(ynz, x, sizeFactors, nfz, fitType, minDisp=1e-8, kappa_0=1.0, dispTol=1e-6, maxit=100,
                         betaTol=1e-8, minmu=0.5):
    """estimateDispersionsGeneEst + estimateDispersionsFit with their defaults on the rows of ynz (none of them
    all-zero; nfz: their nf rows, xim is taken over them): gene_wise_dispersions and dispersion_function_of."""
    bm, dge = gene_wise_dispersions(ynz, x, sizeFactors, nfz, minDisp=minDisp, kappa_0=kappa_0, dispTol=dispTol,
                                    maxit=maxit, betaTol=betaTol, minmu=minmu)
    return dispersion_function_of(bm, dge, fitType, minDisp)


def _vst_result(y, m, fn, sizeFactors, nf, sfd):
    mode, c0, c1 = _vst_constants(fn)
    res = {"vst": transform(y, m, mode, c0, c1, sfd), "fitType": fn["fitType"]}
    res.update({k: fn[k] for k in ("trendCoefs", "meanDisp") if k in fn})
    if nf is not None:
        res["normalizationFactors"] = nf
    else:
        res["sizeFactors"] = sizeFactors
    return res


def vst_transform(y, m, dispersionFunction, sizeFactors=None, normalizationFactors=None):
    """getVarianceStabilizedData (R/vst.R:145-196) on the device: the VST of the normalized counts of all N rows of y
    (gene-major (N, ld), int32 or float64) as a fresh contiguous (N, m) float64 device tensor; all-zero rows too.
    dispersionFunction: a dict as DESeq_device or the VST functions return it, {"fitType": "parametric",
    "trendCoefs": (asymptDisp, extraPois)} or {"fitType": "mean", "meanDisp": alpha}.  Applying the function of one
    analysis to other samples (any m) is R's frozen VST (R/vst.R:69-76).  Exactly one of sizeFactors ((m,) numpy or
    device tensor) and normalizationFactors (gene-major (N, ld) float64 device tensor) is needed.  Any other fitType
    ("local") raises ValueError."""
    mode, c0, c1 = _vst_constants(dispersionFunction)
    if isinstance(sizeFactors, torch.Tensor):
        sizeFactors = sizeFactors.cpu().numpy()
    sfd = _size_or_norm_factors(y, m, sizeFactors, normalizationFactors, None)
    return transform(y, m, mode, c0, c1, sfd)


def varianceStabilizingTransformation_device(y, m, x=None, blind=True, fitType="parametric", sizeFactors=None,
                                             normalizationFactors=None, avgTxLength=None, dispersionFunction=None):
    """varianceStabilizingTransformation (R/vst.R:112-142) on the device, for y gene-major (N, ld) counts of m samples.
    The size factors are estimated (median of ratios) when none of sizeFactors / normalizationFactors / avgTxLength is
    given; avgTxLength estimates the nf as DESeq_device does.  With blind=True (the design is ~1) or without a
    dispersionFunction, estimateDispersionsGeneEst + estimateDispersionsFit (fitType "parametric" or "mean") run on
    the rows with a non-zero sum, with design x when blind=False; otherwise dispersionFunction is used as it is and
    fitType is ignored, as in R.  Returns {"vst": (N, m) device tensor, "fitType", "trendCoefs" or "meanDisp",
    "sizeFactors" or "normalizationFactors"}; the dispersion keys can be passed back as a frozen dispersionFunction.
    blind=False without x or dispersionFunction raises ValueError; a failed parametric fit raises FloatingPointError."""
    refit = blind or dispersionFunction is None
    if refit:
        if not blind and x is None:
            raise ValueError("blind=False needs the design x or a dispersionFunction")
        _check_vst_fit_type(fitType)
        x = _vst_design(x, m, blind)
    sizeFactors, nf, sfd = _factors(y, m, sizeFactors, normalizationFactors, avgTxLength)
    if refit:
        idx = torch.nonzero(y[:, :m].sum(dim=1) != 0).squeeze(1)
        whole = idx.numel() == y.shape[0]
        ynz = y if whole else y[idx].contiguous()
        nfz = None if nf is None else (nf if whole else nf[idx].contiguous())
        dispersionFunction = _dispersion_function(ynz, x, sizeFactors, nfz, fitType)
    return _vst_result(y, m, dispersionFunction, sizeFactors, nf, sfd)


def vst_device(y, m, x=None, blind=True, nsub=1000, fitType="parametric", sizeFactors=None,
               normalizationFactors=None, avgTxLength=None):
    """vst (R/vst.R:219-267) on the device: the dispersion function is fitted on nsub genes only, then the VST runs
    over all N rows of y (gene-major (N, ld) counts of m samples).  Factors as in
    varianceStabilizingTransformation_device.  The genes: baseMean (the pre-step kernel's row mean of the normalized
    counts) > 5, in the order of a stable sort of baseMean, at the positions pipeline.vstSubsetPositions(L, nsub);
    estimateDispersionsGeneEst + estimateDispersionsFit run on them in that order, with design ~1 when blind and x
    otherwise (xim over the subset's nf rows).  R's two stops raise ValueError.  Returns the dict of
    varianceStabilizingTransformation_device plus "subset": the nsub row indices into y, in fit order."""
    from .pipeline import vstSubsetPositions
    if y.shape[0] < nsub:
        raise ValueError("less than 'nsub' rows, it is recommended to use varianceStabilizingTransformation directly")
    if not blind and x is None:
        raise ValueError("blind=False needs the design x")
    _check_vst_fit_type(fitType)
    x = _vst_design(x, m, blind)
    sizeFactors, nf, sfd = _factors(y, m, sizeFactors, normalizationFactors, avgTxLength)
    # rowMeans(counts(normalized = TRUE)) over all rows: the pre-step kernel's baseMean for x = 1 (xim is not used)
    bm = prep(y, np.ones((m, 1)), sizeFactors, want_mu=False, want_beta0=False, normalizationFactors=nf,
              xim=1.0)["baseMean"]
    cand = torch.nonzero(bm > 5).squeeze(1)
    L = cand.numel()
    if L < nsub:
        raise ValueError("less than 'nsub' rows with mean normalized count > 5, it is recommended to use "
                         "varianceStabilizingTransformation directly")
    _, o = torch.sort(bm[cand], stable=True)
    subset = cand[o[torch.as_tensor(vstSubsetPositions(L, nsub), device=y.device)]]
    ysub = y[subset].contiguous()
    nfsub = None if nf is None else nf[subset].contiguous()
    res = _vst_result(y, m, _dispersion_function(ysub, x, sizeFactors, nfsub, fitType), sizeFactors, nf, sfd)
    res["subset"] = subset
    return res


def normTransform_device(y, m, sizeFactors=None, normalizationFactors=None, pc=1.0):
    """normTransform(f = log2) (R/helper.R:421-435) on the device: log2(normalized counts + pc) of all N rows of y as a
    fresh (N, m) float64 device tensor; the size factors are estimated (median of ratios) when neither sizeFactors
    nor normalizationFactors is given."""
    _, _, sfd = _factors(y, m, sizeFactors, normalizationFactors)
    return transform(y, m, "log2", pc, 0.0, sfd)


# ---------------------------------------------------------------- rlog() (R/rlog.R)

def rlog_prior_var(y, m, sfd, baseMean, dispFit):
    """b200nb_rlog_prior_var_dev: rlogData's betaPriorVar (R/rlog.R:233-240) over every entry of the N rows of y
    (gene-major (N, ld) int32 or float64): the weighted 95 % quantile of |log2(K / s + 0.5) - log2(baseMean + 0.5)| with
    weights 1 / (1 / baseMean + dispFit), matched to a normal.  sfd: the (m,) size-factor device vector or a gene-major
    (N, ld) nf matrix; baseMean, dispFit: (N,) device tensors.  Rows whose weight is NaN or 0 (all-zero rows) do not
    take part.  Returns a 0-d device tensor (NaN when no entry takes part).  Enqueue only."""
    L = _lib.lib()
    n, ld = y.shape
    out = torch.empty(1, dtype=F64, device=y.device)
    sf, nf = D._split_factors(sfd)
    _lib.check(L.b200nb_rlog_prior_var_dev(D._p(y), D._ytype(y), D._p(sf), D._p(nf), D._p(baseMean),
                                           D._p(dispFit), n, m, ld, D._p(out), D._stream()), "rlog_prior_var_dev")
    return out[0]


def rlog_fit(y, m, sfd, dispFit, betaPriorVar, intercept=None, betaTol=1e-4, maxit=100, minmu=0.5):
    """b200nb_rlog_fit_dev: rlogData's fitNbinomGLMs call (R/rlog.R:249-253) for all N rows of y (gene-major (N, ld)
    int32 or float64): the design [1 | I_m], or I_m on nf 2^intercept when `intercept` ((N,) float64 device tensor of
    log2 intercepts) is given.  sfd as for rlog_prior_var; dispFit: (N,) device tensor.  Returns {"rlog": fresh (N, m)
    device tensor on the log2 scale, "intercept": (N,) fitted log2 intercepts (-Inf for all-zero rows; None with a
    frozen intercept), "betaIter": (N,)}.  Rows R leaves out (all-zero; a non-finite frozen intercept) are 0 with
    betaIter 0.  Enqueue only."""
    if y.dim() != 2 or y.dtype not in (torch.int32, F64) or not y.is_contiguous():
        raise ValueError("y must be a contiguous gene-major int32 or float64 tensor")
    L = _lib.lib()
    n, ld = y.shape
    dev = y.device
    out = torch.empty((n, m), dtype=F64, device=dev)
    icpt = None if intercept is not None else torch.empty(n, dtype=F64, device=dev)
    it = torch.empty(n, dtype=F64, device=dev)
    sf, nf = D._split_factors(sfd)
    _lib.check(L.b200nb_rlog_fit_dev(D._p(y), D._ytype(y), D._p(sf), D._p(nf), D._p(intercept), D._p(dispFit),
                                     n, m, ld, float(betaPriorVar), float(betaTol), int(maxit), float(minmu), D._p(out),
                                     m, D._p(icpt), D._p(it), D._stream()), "rlog_fit_dev")
    return {"rlog": out, "intercept": icpt, "betaIter": it}


def _sparse_test(q, rs, p=0.9, t1=100, t2=0.1):
    """sparseTest (R/rlog.R:274-287) on the normalized counts q (N, m) with row sums rs: warns when, among the rows
    whose sum exceeds t1, more than a fraction t2 have one sample holding more than p of the row sum."""
    import warnings
    rmx = q.amax(dim=1)
    sel = rs > t1
    if not bool(sel.any()):
        return
    total = float(((rmx[sel] / rs[sel]) > p).to(F64).mean().item())
    if total > t2:
        warnings.warn("the rlog assumes that data is close to a negative binomial distribution, an assumption which is "
                      "sometimes not compatible with datasets where many genes have many zero counts despite a few "
                      f"very large counts.  In this data, for {round(total, 3) * 100}% of genes with a sum of "
                      f"normalized counts above {t1}, it was the case that a single sample's normalized count made up "
                      f"more than {p * 100}% of the sum over all samples.  The threshold for this warning is "
                      f"{t2 * 100}% of genes.  We recommend instead using the varianceStabilizingTransformation or "
                      "shifted log.", stacklevel=3)


def _row_vector(v, n, dev, name):
    """An (n,) float64 device tensor from a numpy array or tensor; ValueError for another length."""
    t = torch.as_tensor(v, dtype=F64, device=dev).reshape(-1)
    if t.numel() != n:
        raise ValueError(f"{name} should be as long as the number of rows of object ({n}), got {t.numel()}")
    return t.contiguous()


def rlog_device(y, m, x=None, blind=True, intercept=None, betaPriorVar=None, fitType="parametric", sizeFactors=None,
                normalizationFactors=None, avgTxLength=None, dispFit=None):
    """rlog / rlogData (R/rlog.R:108-272) on the device for y gene-major (N, ld) counts of m samples, in R's order:
    the factors (_factors: estimated size factors, sizeFactors, normalizationFactors or avgTxLength); sparseTest as a
    warning when no intercept is given; with blind=True or without dispFit, estimateDispersionsGeneEst +
    estimateDispersionsFit (fitType "parametric" or "mean") on the non-zero rows with design ~1 when blind and x
    otherwise, and dispFit = the trend at baseMean; else dispFit ((N,) device tensor aligned with y's rows, R's
    mcols(object)$dispFit) as given.  betaPriorVar, when not given, by rlog_prior_var; then one rlog_fit.
    With intercept ((N,) log2, R's rlogIntercept of an earlier call), the frozen rlog: design I_m on nf 2^intercept,
    rows with a non-finite intercept left out (0) and the intercept added back.
    Returns {"rlog": (N, m) device tensor, "betaPriorVar": float, "intercept": (N,) device tensor (None when frozen),
    "dispFit", "fitType" and "trendCoefs" / "meanDisp" (when estimated), "sizeFactors" / "normalizationFactors",
    "betaIter", "n_nonfinite"}.  Rows whose fit is not finite (R's rowStable would send them to optim) are counted in
    n_nonfinite with a warning, not refitted.  R's stops raise ValueError (intercept length, dispFit missing or not
    finite and positive on a fitted row); a failed parametric trend raises FloatingPointError."""
    import warnings
    dev = y.device
    n = y.shape[0]
    if intercept is not None:
        intercept = _row_vector(intercept, n, dev, "intercept")
    refit = blind or dispFit is None
    if refit:
        if not blind and x is None:
            raise ValueError("blind=False needs the design x or dispFit")
        _check_vst_fit_type(fitType)
        x = _vst_design(x, m, blind)
    sizeFactors, nf, sfd = _factors(y, m, sizeFactors, normalizationFactors, avgTxLength)
    # the normalized counts of sparseTest and getBaseMeansAndVariances' baseMean = rowMeans (any m, also 1)
    q = y[:, :m].to(F64) / (sfd[:, :m] if sfd.dim() == 2 else sfd)
    rs = q.sum(dim=1)
    if intercept is None:
        _sparse_test(q, rs)
    del q
    bm = rs / m
    res = {}
    if refit:
        idx = torch.nonzero(bm > 0).squeeze(1)
        whole = idx.numel() == n
        ynz = y if whole else y[idx].contiguous()
        nfz = None if nf is None else (nf if whole else nf[idx].contiguous())
        fn = _dispersion_function(ynz, x, sizeFactors, nfz, fitType)
        res.update(fn)
        if fitType == "mean":
            dispFit = torch.full((n,), fn["meanDisp"], dtype=F64, device=dev)
        else:
            dispFit = fn["trendCoefs"][0] + fn["trendCoefs"][1] / bm
    else:
        dispFit = _row_vector(dispFit, n, dev, "dispFit")
    fit_rows = torch.isfinite(intercept) if intercept is not None else bm > 0
    d = dispFit[fit_rows]
    if not bool(torch.all(torch.isfinite(d) & (d > 0))):
        raise ValueError("dispFit must be finite and positive on every row the rlog fits")
    if betaPriorVar is None:
        if intercept is None:
            bpv = rlog_prior_var(y, m, sfd, bm, dispFit)
        else:
            # the entries of the rows with a finite intercept, normalized by nf 2^intercept (R/rlog.R:219, :234)
            keep = torch.nonzero(fit_rows).squeeze(1)
            ysub = y[keep].contiguous()
            base = sfd[keep][:, :m] if sfd.dim() == 2 else sfd[None, :]
            nfp = torch.ones(ysub.shape, dtype=F64, device=dev)
            nfp[:, :m] = base * torch.pow(2.0, intercept[keep])[:, None]
            bpv = rlog_prior_var(ysub, m, nfp, bm[keep].contiguous(), dispFit[keep].contiguous())
        betaPriorVar = float(bpv.item())
        if not (np.isfinite(betaPriorVar) and betaPriorVar > 0):
            raise ValueError(f"the estimated betaPriorVar ({betaPriorVar}) is not finite and positive")
    fit = rlog_fit(y, m, sfd, dispFit, betaPriorVar, intercept=intercept)
    bad = int((~torch.isfinite(fit["rlog"])).any(dim=1).sum().item())
    if bad:
        warnings.warn(f"{bad} rows of the rlog fit are not finite (R would refit them with optim); they are returned "
                      "as they are", stacklevel=2)
    res.update({"rlog": fit["rlog"], "betaPriorVar": betaPriorVar, "intercept": fit["intercept"], "dispFit": dispFit,
                "betaIter": fit["betaIter"], "n_nonfinite": bad})
    if nf is not None:
        res["normalizationFactors"] = nf
    else:
        res["sizeFactors"] = sizeFactors
    return res


# ---------------------------------------------------------------- results() and pvalueAdjustment() (R/results.R)

_ALT_CODE = {"greaterAbs": 1, "greaterAbs2014": 2, "lessAbs": 3, "greater": 4, "less": 5}     # B200NB_ALT_*
_PADJ_CODE = {"BH": 0, "fdr": 0, "BY": 1, "holm": 2, "hochberg": 3, "bonferroni": 4, "none": 5}   # B200NB_PADJ_*


def filter_cutoffs(filter, theta):
    """b200nb_filter_cutoffs_dev: quantile(filter, theta, type = 7) of a (N,) float64 device tensor at the (T,) device
    probabilities, one CTA per probability.  Enqueue only."""
    L = _lib.lib()
    out = torch.empty(theta.numel(), dtype=F64, device=filter.device)
    _lib.check(L.b200nb_filter_cutoffs_dev(D._p(filter), filter.numel(), D._p(theta), theta.numel(), D._p(out),
                                           D._stream()), "filter_cutoffs_dev")
    return out


def filter_numrej(p_sorted, filter_sorted, cutoffs, method, alpha):
    """b200nb_filter_numrej_dev: numRej of pvalueAdjustment for every cutoff, from the p-values sorted ascending (NaN
    last) and their filter values.  Returns a (T,) int32 device tensor.  Enqueue only."""
    L = _lib.lib()
    out = torch.empty(cutoffs.numel(), dtype=torch.int32, device=p_sorted.device)
    _lib.check(L.b200nb_filter_numrej_dev(D._p(p_sorted), D._p(filter_sorted), p_sorted.numel(), D._p(cutoffs),
                                          cutoffs.numel(), _PADJ_CODE[method], float(alpha), D._p(out), D._stream()),
               "filter_numrej_dev")
    return out


def padj_column(p_sorted, filter_sorted, order, method, cutoffs=None, j=0):
    """b200nb_padj_dev: p.adjust(method) over the genes with filter >= cutoffs[j] (cutoffs None: every gene with a
    p-value), as a (N,) device tensor in gene order with NaN for the others.  Enqueue only."""
    L = _lib.lib()
    out = torch.empty(p_sorted.numel(), dtype=F64, device=p_sorted.device)
    _lib.check(L.b200nb_padj_dev(D._p(p_sorted), D._p(filter_sorted), D._p(order), p_sorted.numel(), D._p(cutoffs),
                                 int(j), _PADJ_CODE[method], D._p(out), D._stream()), "padj_dev")
    return out


def p_value_adjustment(pvalue, filter, independentFiltering=True, theta=None, alpha=0.1, pAdjustMethod="BH"):
    """pvalueAdjustment (R/results.R:638-718) on (N,) float64 device tensors: the p-values sorted once (torch.sort,
    plumbing), then the cutoff, rejection-count and adjusted-column kernels.  theta: numpy probabilities, or None for
    seq(mean(filter == 0), .95 or 1, length = 50) formed on the device.  The one host read is numRej (with theta and the
    cutoffs), which lowess needs.  Returns (padj (N,) device tensor, metadata)."""
    from .pipeline import filter_choose, lowess
    dev = pvalue.device
    meta = {"alpha": alpha}
    ps, order = torch.sort(pvalue)                          # NaN last
    fs = filter[order].contiguous()
    if not independentFiltering:
        return padj_column(ps, fs, order, pAdjustMethod), meta
    if theta is None:
        # divisors as device tensors: a division by a Python scalar becomes a multiplication by its reciprocal on the
        # GPU, which is not R's rounding
        cst = lambda v: torch.tensor(v, dtype=F64, device=dev)
        lo = (filter == 0).to(F64).sum() / cst(float(filter.numel()))
        hi = torch.where(lo < 0.95, cst(0.95), cst(1.0))
        th = lo + torch.arange(50, dtype=F64, device=dev) * ((hi - lo) / cst(49.0))
        th[49] = hi
    else:
        th = torch.as_tensor(theta, dtype=F64, device=dev)
    cutoffs = filter_cutoffs(filter, th)
    numRej = filter_numrej(ps, fs, cutoffs, pAdjustMethod, alpha)
    host = torch.stack([numRej.to(F64), th, cutoffs]).cpu().numpy()
    nr, theta, cut = host[0].astype(np.int64), host[1], host[2]
    lo_fit = lowess(theta, nr, f=1.0 / 5.0)
    j = filter_choose(nr, lo_fit["y"])
    meta.update(filterThreshold=float(cut[j]), filterTheta=float(theta[j]),
                filterNumRej={"theta": theta, "numRej": nr}, lo_fit=lo_fit, j=j, cutoffs=cut)
    return padj_column(ps, fs, order, pAdjustMethod, cutoffs, j), meta


def results_gene(ynz, m, lfc, se, stat, pvalue, negate=False, zero_mask=None, lrt=False, alt=0, lfcThreshold=0.0,
                 maxCooks=None, cooksCutoff=0.0, keep=None, replace=None, baseMean=None):
    """b200nb_results_gene_dev: results()' per-gene steps for the n rows of ynz (gene-major counts, read for
    zero_mask only): swapped reference, contrastAllZero, threshold test, Cook's cutoff, now-all-zero rows.  Returns
    (log2FoldChange, lfcSE, stat, pvalue) as fresh (n,) device tensors.  Enqueue only."""
    L = _lib.lib()
    n, ld = ynz.shape
    out = [torch.empty(n, dtype=F64, device=ynz.device) for _ in range(4)]
    _lib.check(L.b200nb_results_gene_dev(D._p(ynz), D._ytype(ynz), n, m, ld, D._p(lfc), D._p(se), D._p(stat),
                                         D._p(pvalue), int(negate), D._p(zero_mask), int(lrt), int(alt),
                                         float(lfcThreshold), D._p(maxCooks), float(cooksCutoff), D._p(keep),
                                         D._p(replace), D._p(baseMean), *(D._p(t) for t in out), D._stream()),
               "results_gene_dev")
    return out


def results_heuristic(ynz, m, rows, cooks_rows, keep):
    """b200nb_results_heuristic_dev: keep[rows[r]] = (at least 3 counts of the gene are above the count at which.max of
    its Cook's row cooks_rows[r]).  Enqueue only."""
    L = _lib.lib()
    n, ld = ynz.shape
    _lib.check(L.b200nb_results_heuristic_dev(D._p(ynz), D._ytype(ynz), D._p(rows), rows.numel(), m, ld,
                                              D._p(cooks_rows), cooks_rows.shape[1], D._p(keep), D._stream()),
               "results_heuristic_dev")


def _check_first_fit_views(res, ynz):
    """Raises ValueError when res["mu"] / res["H"], views of DESeq_device's workspace, have been replaced by a later
    DESeq_device call."""
    mu_ws, h_ws = _WS.get(("mu_cooks", str(ynz.device))), _WS.get(("H", str(ynz.device)))
    if (mu_ws is None or h_ws is None or res["mu"].data_ptr() != mu_ws.data_ptr()
            or res["H"].data_ptr() != h_ws.data_ptr() or tuple(res["mu"].shape) != tuple(ynz.shape)):
        raise ValueError("res['mu'] / res['H'] are views of DESeq_device's workspace and a later DESeq_device call has "
                         "replaced it: run results_device before the next DESeq_device call")


def _first_fit_cooks(res, ynz, rows, x, sfd):
    """The Cook's rows of `rows` from the first fit's mu / H (res["mu"] / res["H"], DESeq_device's workspace views: R
    restores the first fit's Cook's distances after a refit, R/core.R:2556).  Raises ValueError when a later
    DESeq_device call has since replaced the workspace."""
    _check_first_fit_views(res, ynz)
    nf = sfd[rows].contiguous() if sfd.dim() == 2 else None
    return cooks(ynz[rows].contiguous(), res["mu"][rows].contiguous(), res["H"][rows].contiguous(), x,
                 res.get("sizeFactors"), normalizationFactors=nf)["cooks"]


def results_device(res, y, x, name=None, contrast=None, listValues=(1, -1), lfcThreshold=0, altHypothesis="greaterAbs",
                   cooksCutoff=None, independentFiltering=True, alpha=0.1, filter=None, theta=None,
                   pAdjustMethod="BH", factors=None, lrt=None, minmu=0.5, weights=None, allgather=None, test=None):
    """results() + pvalueAdjustment() (R/results.R:298-740) on a DESeq_device result `res` for the gene-major (N, ld)
    counts y it was run on and its design x.  Arguments as pipeline.results (the host mirror): name / contrast /
    listValues select the column (pipeline.resultsSelection; list and numeric contrasts, factor-level contrasts that
    involve no reference level and every betaPrior contrast go through getContrast_device, on the replaced counts
    after an outlier refit); factors: the design's level-code vectors; lrt: an nbinomLRT_device result for the same
    rows and full design.  The per-gene steps are one kernel (results_gene), the adjustment p_value_adjustment.
    res["mu"] / res["H"] are DESeq_device's workspace views, valid until the next DESeq_device call: the two-group
    heuristic and the replaced counts of a contrast after an outlier refit recompute Cook's rows from them.
    weights: the raw observation weights DESeq_device was given (gene-major (N, ld)); a weights result needs them for
    the baseMean of its weightsFail rows (mean of w K / s, as getBaseMeansAndVariances), which count in the filter.
    Host reads: at most two small ones -- the number of genes the Cook's cutoff flags (only for a single two-level
    factor) and numRej with theta and the cutoffs (only with independent filtering).  A `filter` given as a device
    tensor is read once to check it for NaN; getContrast_device reads once to check weights.
    Returns {"baseMean", "log2FoldChange", "lfcSE", "stat", "pvalue", "padj"}: (N,) device tensors over all input
    rows (all-zero rows: baseMean 0; all-zero and weightsFail rows: NaN in the other columns; both count in the
    filter), and "metadata".
    allgather (sharded_results_device): concatenates a list of per-gene vectors over the ranks in rank order (one
    collective); [filter, pvalue] of this rank's rows travel in it, the cutoffs, counts and adjusted column are
    computed on all genes, and this rank keeps the padj of its own rows (sharded.shard_bounds).
    test: as R's results(test =), by default the test DESeq_device ran (res["test"]).  An LRT result
    (DESeq_device(test="LRT")) gives its LRTStatistic / LRTPvalue with the selected column's log2FoldChange / lfcSE;
    test="Wald" on it gives the Wald columns (makeWaldTest).  test="LRT" on a Wald result, and lrt= with an LRT result,
    raise ValueError.
    A result with "tDegreesFreedom" (DESeq_device(useT=True)) is tested with t tails, as R infers useT from that column
    (R/results.R:414): a stored Wald column keeps its p-values, a contrast goes through getContrast_device(useT=True),
    and a thresholded test (R/results.R:477-518) takes pt at each gene's df (threshold_t_pvalue) from the kernel's
    log2FoldChange / lfcSE, keeping the kernel's NaN (Cook's cutoff) and 1 (rows all zero once replaced)."""
    from scipy import stats as _st
    from .pipeline import check_filter_args, results_checks, resultsSelection
    dev = y.device
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    N = y.shape[0]
    ran = res.get("test", "Wald")
    test = ran if test is None else test
    if test not in ("Wald", "LRT"):
        raise ValueError("test must be 'Wald' or 'LRT'")
    if test == "LRT" and ran == "Wald":
        raise ValueError("the LRT requires the user run nbinomLRT or DESeq(dds,test='LRT')")
    if ran == "LRT":
        if lrt is not None:
            raise ValueError("this DESeq_device result holds its own LRT: lrt= is for a Wald result")
        if test == "LRT":
            lrt = {"LRTStatistic": res["LRTStatistic"], "LRTPvalue": res["LRTPvalue"]}
    idx = res["idx"]
    betaPrior = res.get("modelMatrix") is not None
    thresholded = results_checks(lfcThreshold, altHypothesis, lrt is not None, betaPrior, alpha)
    filter, theta = check_filter_args(N, filter, theta, alpha, pAdjustMethod)
    sel = resultsSelection(x, name, contrast, listValues, factors, betaPrior, res.get("modelMatrix"))
    wf = res.get("weightsFail")
    if wf is not None and weights is None:
        raise ValueError("a DESeq_device result with observation weights needs weights= (the raw weights it was given) "
                         "for the baseMean of its weightsFail rows")
    whole = idx.numel() == N
    ynz = y if whole else y[idx].contiguous()
    nf = res.get("normalizationFactors")
    sfd = nf if nf is not None else torch.as_tensor(res["sizeFactors"], device=dev)
    replace = res.get("replace") if res.get("n_replaced", 0) > 0 else None
    tdf = res.get("tDegreesFreedom")
    # ---- the selected column (cleanContrast / getCoef)
    if sel["kind"] == "coef":
        k = sel["col"]
        cols = [res[key][:, k].contiguous() for key in ("betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue")]
    else:
        xf = res["modelMatrix"] if betaPrior else x
        ycnt = ynz
        if replace is not None:                            # getContrast reads replaceCounts (R/results.R:776-780)
            rows = torch.nonzero_static(replace, size=res["n_replaced"]).squeeze(1)   # the count is known: no read
            cutoff = float(_st.f.ppf(0.99, p, m - p))
            ck = _first_fit_cooks(res, ynz, rows, x, sfd)
            ys = ynz[rows][:, :m].to(F64)
            nfm = sfd[rows][:, :m] if sfd.dim() == 2 else sfd[None, :]
            ycnt = ynz.to(F64).clone()
            ycnt[rows, :m] = _replacement_counts(ys, nfm, ck[:, :m] > cutoff, res["replaceable"], m)
        g = getContrast_device(ycnt, xf, None if nf is not None else res["sizeFactors"], res["dispersion"],
                               res["betaMatrix"], sel["vec"], betaPriorVar=res.get("betaPriorVar"), minmu=minmu,
                               weights=res.get("weights"), normalizationFactors=nf, useT=tdf is not None, df=tdf)
        cols = [g[key].contiguous() for key in ("log2FoldChange", "lfcSE", "stat", "pvalue")]
    if lrt is not None:
        cols[2], cols[3] = lrt["LRTStatistic"].contiguous(), lrt["LRTPvalue"].contiguous()
    mask = None if sel["mask"] is None else torch.as_tensor(sel["mask"].astype(np.int32), device=dev)
    # ---- Cook's cutoff and the two-group heuristic
    maxCooks, keep, cutoff = None, None, 0.0
    if cooksCutoff is not False:
        cutoff = float(_st.f.ppf(0.99, p, m - p)) if cooksCutoff is None or cooksCutoff is True else float(cooksCutoff)
        maxCooks = res["maxCooks"].contiguous()
        if factors is not None and len(factors) == 1 and int(np.max(factors[0])) == 1:
            rows = torch.nonzero(maxCooks > cutoff).squeeze(1)
            if rows.numel() > 0:
                keep = torch.zeros(ynz.shape[0], dtype=torch.int32, device=dev)
                results_heuristic(ynz, m, rows, _first_fit_cooks(res, ynz, rows, x, sfd), keep)
    alt = _ALT_CODE[altHypothesis] if thresholded else 0
    lfc, se, stat, pv = results_gene(ynz, m, *cols, negate=sel.get("negate", False), zero_mask=mask,
                                     lrt=lrt is not None, alt=alt, lfcThreshold=lfcThreshold, maxCooks=maxCooks,
                                     cooksCutoff=cutoff, keep=keep,
                                     replace=None if replace is None else replace.to(torch.int32),
                                     baseMean=res["baseMean"])
    if thresholded and tdf is not None:
        tp = threshold_t_pvalue(lfc, se, float(lfcThreshold), altHypothesis, tdf)
        keep_kernel = torch.isnan(pv) | torch.isinf(tdf)     # Cook's NaN; df = Inf: the kernel's normal tail
        if replace is not None:
            keep_kernel = keep_kernel | (replace & (res["baseMean"] == 0))
        pv = torch.where(keep_kernel, pv, tp)
    # ---- all N rows (buildDataFrameWithNARows), then pvalueAdjustment
    out = {"baseMean": torch.zeros(N, dtype=F64, device=dev)}
    out["baseMean"][idx] = res["baseMean"]
    if wf is not None:                                  # the weightsFail rows keep their weighted baseMean
        sf = torch.as_tensor(res["sizeFactors"], device=dev)
        wbm = (weights[:, :m] * (y[:, :m].to(F64) / sf)).mean(dim=1)
        out["baseMean"] = torch.where(wf, wbm, out["baseMean"])
    for key, v in (("log2FoldChange", lfc), ("lfcSE", se), ("stat", stat), ("pvalue", pv)):
        out[key] = torch.full((N,), float("nan"), dtype=F64, device=dev)
        out[key][idx] = v
    filt = out["baseMean"] if filter is None else torch.as_tensor(filter, device=dev)
    if allgather is None:
        out["padj"], meta = p_value_adjustment(out["pvalue"], filt, independentFiltering, theta, alpha,
                                               pAdjustMethod)
    else:
        import torch.distributed as dist
        from .sharded import shard_bounds
        fa, pa = allgather([filt, out["pvalue"]])
        lo, hi = shard_bounds(pa.numel(), dist.get_world_size(), dist.get_rank())
        if hi - lo != N:
            raise ValueError(f"this rank holds {N} rows where shard_bounds gives it {hi - lo}: split the rows as "
                             "sharded.shard_bounds does")
        padj, meta = p_value_adjustment(pa, fa, independentFiltering, theta, alpha, pAdjustMethod)
        out["padj"] = padj[lo:hi]
    meta["lfcThreshold"] = lfcThreshold
    out["metadata"] = meta
    return out


def threshold_t_pvalue(lfc, se, T, altHypothesis, df):
    """results()' lfcThreshold p-values with useT (R/results.R:477-518) on device tensors: pt at each gene's df in
    place of pnorm, for the five altHypothesis forms; greaterAbs is pt((T - |lfc|) / se) + pt((-|lfc| - T) / se),
    lower tails, taken as t_upper of the negated quantiles.  (R evaluates that form through mapply over the genes with
    the whole df vector, which yields an n x n matrix; its diagonal, each gene at its own df, is what this returns.)"""
    up = lambda q: t_upper(q, df)
    if altHypothesis == "greaterAbs":
        return up((lfc.abs() - T) / se) + up((lfc.abs() + T) / se)
    if altHypothesis == "greaterAbs2014":
        return torch.clamp(2.0 * up((lfc.abs() - T) / se), max=1.0)
    if altHypothesis == "lessAbs":
        return torch.maximum(up((T - lfc) / se), up((lfc + T) / se))
    if altHypothesis == "greater":
        return up((lfc - T) / se)
    return up((-T - lfc) / se)


# ---------------------------------------------------------------- lfcShrink(type = "normal") (R/lfcShrink.R:145-327)

def _scatter_rows(v, rows, n):
    """v's rows at `rows` of a fresh (n, ...) tensor, NaN (False for bool) elsewhere."""
    fill = False if v.dtype == torch.bool else float("nan")
    out = torch.full((n,) + tuple(v.shape[1:]), fill, dtype=v.dtype, device=v.device)
    out[rows] = v
    return out


def lfcShrink_device(res, y, x, coef=None, contrast=None, results=None, lfcThreshold=0, factors=None, weights=None,
                     allgather=None, betaTol=1e-8, maxit=100, useOptim=True, minmu=0.5, type="normal"):
    """lfcShrink(type = "normal") (R/lfcShrink.R:145-327) on a DESeq_device result `res` (betaPrior=False, any
    test) for the gene-major (N, ld) counts y it was run on and its design x.  Only type "normal" exists in DESeq2;
    "apeglm" and "ashr" call other packages and raise ValueError, as do R's other stops (pipeline.lfcShrink_checks).
    coef (a column index or factorDesign name of x; x may be any full-rank design whose first column is the
    intercept, numeric covariates included -- R's user-supplied-matrix path): estimateBetaPriorVar with
    modelMatrixType "standard" (R/core.R:1601-1689: one weighted quantile per non-intercept MLE column, one launch of
    b200nb_beta_prior_quantile_dev), then fitNbinomGLMs(lambda = 1 / betaPriorVar) on x from the pre-step kernel's
    linear-model start values (R/fitNbinomGLMs.R:242-337; the MLE is skipped because mu and H exist).
    contrast (as results_device takes it with factors, over the expanded matrix's columns; x must be
    factorDesign(factors)[0]): the expanded prior (estimate_beta_prior_var) and the MAP fit on
    factorDesign(factors, expanded=True)[0] from (log baseMean, 0, ..., 0) -- what DESeq_device(betaPrior=True)
    computes.  Both fits are _map_fit: the IRLS kernel, the log-likelihood at the unclamped mean and the optim
    fallback with the same lambda, with nbinomWaldTest's betaTol / maxit / useOptim / minmu (R's lfcShrink passes
    none of DESeq's on).  The prior's weights are 1 / (1 / baseMean + dispFit) of res's rows (the weighted baseMean
    for a weights result, whose normalised weights also go to the MAP fit; weights: the raw weights, as for
    results_device, coef only).
    Outlier-refit results (R/core.R:2484-2564): the MAP fit runs on the ORIGINAL counts with the refitted
    dispersions, and the prior uses the replaced baseMean / dispFit and the refitted MLE betas; rows whose replaced
    counts are all zero are allZero in R and are neither in the prior nor fitted (the shrunk table's nowZero rule
    gives them log2FoldChange and lfcSE 0).  For a contrast the shrunk table's getContrast reads the replaced counts
    (R/results.R:779-781), rebuilt by results_device from res's "replace" / "replaceable" / "n_replaced"; with
    lfcThreshold > 0 its Cook's cutoff uses the first fit's maxCooks, recomputed from res["mu"] / res["H"] on the
    original counts without the replaceable-sample zeroing, as nbinomWaldTest recomputes it (R/core.R:1452-1460).
    res["mu"] / res["H"] are DESeq_device's workspace views: where they are read, a stale result raises ValueError
    as in results_device.
    results: the table to modify (a results_device dict over the N rows); by default results_device(res, y, x,
    name=coef) or (..., contrast=contrast) with its defaults.  The shrunk table is results_device on the MAP fit with
    the same selection, lfcThreshold and minmu; its log2FoldChange and lfcSE replace the table's, and with
    lfcThreshold > 0 its stat, pvalue and padj too (the other columns stay the table's tensors).
    allgather (sharded.sharded_lfcShrink_device): ONE packed collective carries baseMean, dispFit and the non-intercept
    MLE columns of every rank's rows for the prior; the default table and the thresholded table take one each.
    Returns the table's dict with those columns replaced, metadata["priorInfo"] = {"type": "normal", "package":
    "DESeq2", "betaPriorVar": numpy}, and "shrinkFit": the MAP fit over res's rows ("betaMatrix", "betaSE",
    "betaConv", "betaIter", "modelMatrix", "n_optim")."""
    from .pipeline import factorDesign, lfcShrink_checks
    x = np.asarray(x, dtype=np.float64)
    m, p = x.shape
    expanded, k = lfcShrink_checks(x, coef, contrast, results is not None, lfcThreshold, factors,
                                   res.get("weightsFail") is not None or weights is not None,
                                   res.get("modelMatrix") is not None, type)
    sel = dict(contrast=contrast) if expanded else dict(name=k)
    if results is None:
        results = results_device(res, y, x, factors=factors, weights=weights, allgather=allgather, **sel)
    dev = y.device
    idx = res["idx"]
    n = idx.numel()
    ynz = y if n == y.shape[0] else y[idx].contiguous()
    nf = res.get("normalizationFactors")
    sfd = nf if nf is not None else torch.as_tensor(res["sizeFactors"], device=dev)
    n_rep = res.get("n_replaced", 0)
    bm = res["baseMean"]
    rows = None                                       # the rows fitted: all of res's, or those not all zero once replaced
    if n_rep > 0:
        rows = torch.nonzero(~(res["replace"] & (bm == 0))).squeeze(1)
        if rows.numel() == n:
            rows = None
    sub = (lambda v: v) if rows is None else (lambda v: v[rows].contiguous())
    # ---- the prior over every fitted row of every rank
    B = sub(res["betaMatrix"])
    bmp, dfp = sub(bm), sub(res["dispFit"])
    if allgather is not None:
        g = allgather([bmp, dfp] + [B[:, j] for j in range(1, p)])
        bmp, dfp = g[0], g[1]
        B = torch.stack([torch.zeros_like(g[0])] + list(g[2:]), dim=1)   # the intercept's column is not read
    pv = estimate_beta_prior_var(B, factors, bmp, dfp, expandedType=expanded)
    # ---- the MAP fit on the original counts
    fy = sub(ynz)
    fsfd = sfd if rows is None else _rows(sfd, rows)
    if expanded:
        xf = factorDesign(factors, expanded=True)[0]
        bm0 = bm
        if n_rep > 0:           # the start is the mean of the ORIGINAL normalised counts; baseMean is the replaced one
            rr = torch.nonzero_static(res["replace"], size=n_rep).squeeze(1)
            nfm = sfd[rr][:, :m] if sfd.dim() == 2 else sfd[None, :]
            bm0 = bm.clone()
            bm0[rr] = (ynz[rr][:, :m].to(F64) / nfm).mean(dim=1)
        beta0 = _expanded_start(sub(bm0), xf.shape[1])
    else:
        xf = x
        beta0 = prep(fy, x, None if nf is not None else res["sizeFactors"], minmu=minmu, want_mu=False,
                     normalizationFactors=fsfd if nf is not None else None, xim=1.0)["beta0"]
    wn = res.get("weights")
    fit, _, betaConv, n_optim = _map_fit(fy, xf, fsfd, sub(res["dispersion"]), pv, beta0, betaTol, maxit, minmu,
                                         useOptim, weights=None if wn is None else sub(wn))
    st = _wald_stats(fit)
    st["betaConv"], st["betaIter"] = betaConv, fit["iter"]
    if rows is not None:
        st = {key: _scatter_rows(v, rows, n) for key, v in st.items()}
    # ---- the shrunk table: results() of the MAP fit
    shr = {key: res.get(key) for key in ("idx", "baseMean", "dispersion", "sizeFactors", "mu", "H", "maxCooks")}
    shr.update(st, test="Wald")
    for key in ("normalizationFactors", "weights", "weightsFail", "replace", "replaceable", "n_replaced"):
        if key in res:
            shr[key] = res[key]
    if expanded:
        shr["modelMatrix"], shr["betaPriorVar"] = xf, pv.cpu().numpy()
    if lfcThreshold > 0 and n_rep > 0:
        _check_first_fit_views(res, ynz)
        shr["maxCooks"] = cooks(ynz, res["mu"], res["H"], x, res.get("sizeFactors"), want_matrix=False,
                                normalizationFactors=nf)["maxCooks"]
    tab = results_device(shr, y, x, factors=factors, lfcThreshold=lfcThreshold, minmu=minmu, weights=weights,
                         allgather=allgather if lfcThreshold > 0 else None, **sel)
    out = dict(results)
    for key in ["log2FoldChange", "lfcSE"] + (["stat", "pvalue", "padj"] if lfcThreshold > 0 else []):
        out[key] = tab[key]
    out["metadata"] = dict(results.get("metadata", {}))
    out["metadata"]["priorInfo"] = {"type": "normal", "package": "DESeq2", "betaPriorVar": pv.cpu().numpy()}
    out["shrinkFit"] = {"betaMatrix": st["betaMatrix"], "betaSE": st["betaSE"], "betaConv": st["betaConv"],
                        "betaIter": st["betaIter"], "modelMatrix": xf, "n_optim": n_optim}
    return out
