"""Every p-value the device pipeline reports against 50-digit tails.

The last step of an analysis turns a statistic into a p-value and then into an adjusted p-value.  Each p-value here is
compared with a plain 50-digit (mpmath) evaluation of the same tail AT THE STATISTIC THE ENGINE RETURNED, so that
differences in the fit cannot enter and only the tail computation is tested:

  * wald_p(z) = 2 Phi(-|z|), R's 2 * pnorm(abs(stat), lower.tail = FALSE) (R/core.R:1507, R/results.R:822);
  * chisq_upper(s, df) = Q(df / 2, s / 2), R's pchisq(stat, df, lower.tail = FALSE) (R/core.R:1878);
  * R's lfcThreshold formulas (R/results.R:464-518) with their arguments q = (|LFC| - T) / SE etc. formed in float64
    exactly as R forms them (and checked bit for bit against the engine's stat), the tails exact at those q;
  * R's p.adjust (BH, BY, holm, hochberg, bonferroni, none) in exact arithmetic on the engine's own float64 p-values,
    over the subset results_device reports.

Tolerances follow from the conditioning of each tail, not from observed errors:

  * Normal tails, t(q) = Phi(-q) or Phi(q) evaluated as erfc(q / sqrt 2) / 2 at a float64 q: the product q * 2^-1/2
    is rounded once (relative 2^-53), and d log erfc(x) / d log x ~ -2 x^2 turns that into q^2 2^-53 relative; erfc
    itself, the rounding of the constant and the final product add a few ulps.  So |t - t*| <= (8 + q^2) 2^-52 t*
    wherever t* >= DBL_MIN.  Below DBL_MIN the result may be 0 or a subnormal: 0 <= t <= DBL_MIN (R returns 0 past
    |z| = 37.5193, erfc returns subnormals up to about 38.5; both are accepted).  Sums (greaterAbs), max (lessAbs)
    and 2 t (greaterAbs2014) add, take the max of, or double the allowances of their terms.
  * Chi-square: Q(a, x) is evaluated through x^a e^-x / Gamma(a) and a series or continued fraction; the exponent
    a log x - x has absolute rounding of order x 2^-53 = s 2^-54, which the exponential turns into relative error.
    So |p - p*| <= (16 + s) 2^-52 p* wherever p* >= DBL_MIN, and the same rule as above below it.
  * Special values: z = 0 gives exactly 1 and z = +-inf exactly 0; a chi-square statistic <= 0 (a fit can make it
    slightly negative by rounding) gives exactly 1, as pchisq(., lower.tail = FALSE) does; +inf gives 0; NaN stays NaN.
  * p.adjust: BH's term (n / r) p is two roundings, holm / hochberg / bonferroni one, and a cummin / cummax of terms
    each within e relative is within e relative: 4 ulps.  BY's q = sum(1 / (1:n)) is summed by the kernel in a fixed
    tree (ceil(n / 512) terms per thread, then 9 levels), each step rounding once: (ceil(n / 512) + 16) ulps.

The function sweep runs device_pipeline's _wald_stats / _lrt_stats directly (CPU tensors on every run, cuda under
-m gpu).  Against torch's gammaincc, which _lrt_stats used before, the dense small-s part of the sweep failed on the
CPU at df 1 and 3: Q is formed there as 1 - P.  The results kernel and the end-to-end cases run
on the SIMT-emulated engine on every CPU run (the product's CUDA sources compiled by g++, tests/simt_emu/) and on the
GPU under -m gpu, the end-to-end one at C2 size (50 000 genes x 100 samples) there.  Every check prints the largest
error it saw as a fraction of its bound (pytest -s).  The CPU half takes about 25 seconds on one core once the
emulated engine is built."""
import ctypes as C
import math

import mpmath
import numpy as np
import pytest
import torch

from helpers import gm
from test_sample_counts import _emu_lib
from deseq2_b200 import pipeline, synth

DPS = 50
EPS = 2.0 ** -52
DBL_MIN = float(np.finfo(np.float64).tiny)
SUBNORMAL_MIN = 2.0 ** -1074
LN2 = math.log(2.0)
NAN = float("nan")
ALTS = ("greaterAbs", "greaterAbs2014", "lessAbs", "greater", "less")


# ---------------------------------------------------------------- backends

@pytest.fixture(params=["cpu", pytest.param("cuda", marks=pytest.mark.gpu)])
def tdev(request):
    """The torch device of the function sweep (no engine involved)."""
    return torch.device(request.param)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def backend(request):
    """(device_pipeline, torch device, is the GPU).  The emulated engine is bound for the one test only."""
    from deseq2_b200 import _lib, device as D, device_pipeline as DP
    if request.param == "gpu":
        request.getfixturevalue("engine")
        yield DP, torch.device("cuda"), True
        return
    lib = _emu_lib()
    saved, saved_stream, saved_dp = _lib._lib, D._stream, DP._stream
    _lib._lib, D._stream = lib, (lambda: C.c_void_p(0))
    DP._stream = D._stream
    try:
        yield DP, torch.device("cpu"), False
    finally:
        _lib._lib, D._stream, DP._stream = saved, saved_stream, saved_dp


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


# ---------------------------------------------------------------- the 50-digit reference
# A reference is a pair (value, allowance) per entry: value an mpf (or NaN), allowance the float bound on |p - p*|.

_CACHE = {}


def _cached(key, f):
    if key not in _CACHE:
        with mpmath.workdps(DPS):
            _CACHE[key] = f()
    return _CACHE[key]


def _normal_allow(q, t):
    """The allowance of one normal tail t* at the float64 argument q (module docstring)."""
    return float((8 + q * q) * EPS * t) if t >= DBL_MIN else DBL_MIN


def _upper(q):
    """(Phi(-q) = pnorm(q, lower.tail = FALSE), allowance) at the exact value of the float64 q."""
    def f():
        if math.isinf(q):
            return (mpmath.mpf(0) if q > 0 else mpmath.mpf(1)), 0.0
        t = mpmath.erfc(mpmath.mpf(q) / mpmath.sqrt(2)) / 2
        return t, _normal_allow(q, t)
    return _cached(("upper", q), f)


def _lower(q):
    """(Phi(q) = pnorm(q), allowance)."""
    return _upper(-q)


def wald_p(z):
    """(2 Phi(-|z|), allowance): exactly 1 at z = 0, exactly 0 at +-inf, NaN at NaN."""
    if math.isnan(z):
        return NAN, 0.0
    if z == 0:
        return mpmath.mpf(1), 0.0
    if math.isinf(z):
        return mpmath.mpf(0), 0.0
    t = 2 * _upper(abs(z))[0]
    return t, _normal_allow(z, t)


def chisq_upper(s, df):
    """(Q(df / 2, s / 2) = pchisq(s, df, lower.tail = FALSE), allowance).  df = 1 and 2 by the exact identities
    erfc(sqrt(s / 2)) and exp(-s / 2) (test_reference_identities checks them against gammainc), the rest by mpmath's
    regularized upper incomplete gamma."""
    if math.isnan(s):
        return NAN, 0.0
    if s <= 0:
        return mpmath.mpf(1), 0.0
    if math.isinf(s):
        return mpmath.mpf(0), 0.0

    def f():
        x = mpmath.mpf(s) / 2
        if df == 1:
            t = mpmath.erfc(mpmath.sqrt(x))
        elif df == 2:
            t = mpmath.exp(-x)
        else:
            t = mpmath.gammainc(mpmath.mpf(df) / 2, x, mpmath.inf, regularized=True)
        return t, (float((16 + s) * EPS * t) if t >= DBL_MIN else DBL_MIN)
    return _cached(("chisq", s, df), f)


def threshold_ref(alt, lfc, se, T):
    """R's results() with lfcThreshold T (R/results.R:484-513) on float64 LFC / SE: (stat as R's float64 expressions
    give it, [(p*, allowance)]).  pnorm(x, sd = se) is pnorm(x / se)."""
    lfc, se = np.asarray(lfc, np.float64), np.asarray(se, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        if alt == "greaterAbs":
            stat = lfc / se
            q1, q2 = (-np.abs(lfc) + T) / se, (-np.abs(lfc) - T) / se
            refs = []
            for a, b in zip(q1, q2):
                if math.isnan(a) or math.isnan(b):
                    refs.append((NAN, 0.0))
                    continue
                (t1, e1), (t2, e2) = _lower(float(a)), _lower(float(b))
                refs.append((t1 + t2, e1 + e2))
        elif alt == "greaterAbs2014":
            q = (np.abs(lfc) - T) / se
            stat = np.sign(lfc) * np.where(np.isnan(q), NAN, np.maximum(q, 0.0))
            refs = []
            for a in q:
                if math.isnan(a):
                    refs.append((NAN, 0.0))
                    continue
                t, e = _upper(float(a))
                refs.append((min(mpmath.mpf(1), 2 * t), 2 * e))
        elif alt == "lessAbs":
            qa, qb = (T - lfc) / se, (lfc + T) / se
            stat = np.minimum(np.maximum(qa, 0.0), np.maximum(qb, 0.0))
            refs = []
            for a, b in zip(qa, qb):
                if math.isnan(a) or math.isnan(b):
                    refs.append((NAN, 0.0))
                    continue
                (t1, e1), (t2, e2) = _upper(float(a)), _upper(float(b))
                refs.append((max(t1, t2), max(e1, e2)))
        elif alt == "greater":
            q = (lfc - T) / se
            stat = np.maximum(q, 0.0)
            refs = [(NAN, 0.0) if math.isnan(a) else _upper(float(a)) for a in q]
        else:
            stat = np.minimum((lfc + T) / se, 0.0)
            q = (-T - lfc) / se
            refs = [(NAN, 0.0) if math.isnan(a) else _upper(float(a)) for a in q]
    return stat, refs


def p_adjust_exact(p, method):
    """R's p.adjust(p, method) (stats/R/p.adjust.R) in exact arithmetic on the float64 p: n is the number of non-NA
    p-values; NA stays NA.  Returns (list of mpf / NaN, relative allowance of the engine's float64 result)."""
    p = np.asarray(p, np.float64)
    out = [NAN] * len(p)
    keep = np.flatnonzero(~np.isnan(p))
    n = len(keep)
    if n == 0:
        return out, 0.0
    with mpmath.workdps(DPS):
        pm = [mpmath.mpf(float(v)) for v in p[keep]]
        if n <= 1 or method == "none":
            adj = pm
        elif method == "bonferroni":
            adj = [min(mpmath.mpf(1), n * v) for v in pm]
        else:
            o = np.argsort(p[keep], kind="stable")
            adj = [None] * n
            if method == "holm":
                run = mpmath.mpf(0)
                for i, k in enumerate(o, start=1):               # cummax((n - i + 1) p_(i)) in increasing order
                    run = max(run, (n - i + 1) * pm[k])
                    adj[k] = min(mpmath.mpf(1), run)
            else:
                q = mpmath.fsum(mpmath.mpf(1) / k for k in range(1, n + 1)) if method == "BY" else None
                run = mpmath.inf
                for i in range(n, 0, -1):                        # cummin over decreasing p: i = rank in increasing order
                    k = o[i - 1]
                    if method == "hochberg":
                        term = (n + 1 - i) * pm[k]
                    elif method == "BY":
                        term = q * n / i * pm[k]
                    else:
                        term = mpmath.mpf(n) / i * pm[k]
                    run = min(run, term)
                    adj[k] = min(mpmath.mpf(1), run)
    for k, v in zip(keep, adj):
        out[k] = v
    rel = (math.ceil(n / 512) + 16) * EPS if method == "BY" else 4 * EPS
    return out, rel


# ---------------------------------------------------------------- the checks

def check_tails(p, refs, what, stat=None, na=False):
    """Every entry of p against its (p*, allowance): NaN exactly where p* is NaN, p >= 0, |p - p*| <= allowance, and
    p <= DBL_MIN where p* underflows.  na: results() may set a p-value to NA (Cook's cutoff), so an NA p-value is
    accepted wherever p* is not NA (if most are not), and every other one is checked.  Returns the largest
    |p - p*| / allowance (0 where the allowance is 0 and p is exact)."""
    p = np.asarray(p, np.float64).ravel()
    assert len(p) == len(refs)
    ref_nan = np.array([isinstance(r, float) and math.isnan(r) for r, _ in refs])
    if na:
        assert np.isnan(p[~ref_nan]).mean() < 0.2, (what, "most p-values are NA")
        ref_nan |= np.isnan(p)
    bad = np.flatnonzero(np.isnan(p) != ref_nan)
    assert len(bad) == 0, (what, "NaN mismatch", bad[:5], p[bad[:5]])
    worst, fails = 0.0, []
    with mpmath.workdps(DPS):
        for i in np.flatnonzero(~ref_nan):
            r, a = refs[i]
            e = float(abs(mpmath.mpf(float(p[i])) - r))
            ok = p[i] >= 0 and e <= a and (r >= DBL_MIN or p[i] <= DBL_MIN)
            if not ok:
                fails.append((i, None if stat is None else float(np.ravel(stat)[i]), float(p[i]),
                               mpmath.nstr(r, 6), e / a if a else math.inf))
            elif a > 0:
                worst = max(worst, e / a)
    assert not fails, (what, f"{len(fails)} of {len(p)} outside the bound; (index, stat, p, p*, error / bound):",
                       fails[:6])
    print(f"{what}: largest error / bound {worst:.3g} over {int((~ref_nan).sum())} p-values")
    return worst


def check_wald(p, stat, what, na=False):
    p, stat = _np(p).ravel(), _np(stat).ravel()
    return check_tails(p, [wald_p(float(z)) for z in stat], what, stat, na)


def check_chisq(p, stat, df, what, na=False):
    p, stat = _np(p).ravel(), _np(stat).ravel()
    return check_tails(p, [chisq_upper(float(s), df) for s in stat], what, stat, na)


def check_padj(out, filt, method="BH", independentFiltering=True):
    """results_device's padj against the exact p.adjust of its own pvalue over the genes it reports: those with a
    p-value and (with independent filtering) a filter statistic >= metadata's filterThreshold."""
    p, padj, filt = _np(out["pvalue"]), _np(out["padj"]), _np(filt)
    member = ~np.isnan(p)
    if independentFiltering:
        member &= filt >= out["metadata"]["filterThreshold"]
    assert np.array_equal(~np.isnan(padj), member), "padj is reported on another subset"
    ref, rel = p_adjust_exact(np.where(member, p, NAN), method)
    # plus two roundings at the subnormal scale, where relative bounds do not hold
    refs = [(NAN, 0.0) if not member[i] else (ref[i], float(rel * ref[i]) + 2 * SUBNORMAL_MIN)
            for i in range(len(p))]
    return check_tails(padj, refs, f"padj {method}")


# ---------------------------------------------------------------- the reference itself

def test_reference_identities():
    """chisq_upper's closed forms for df = 1, 2 against mpmath's gammainc; the tails against known values (R:
    2 * pnorm(-9) = 2.257177e-19, 2 * pnorm(-20) = 5.507248e-89, pchisq(100, 1, lower = FALSE) = 1.523971e-23)."""
    with mpmath.workdps(DPS):
        for s in (1e-300, 1e-8, 0.3, 1.0, 17.0, 400.0, 1450.0):
            for df in (1, 2):
                g = mpmath.gammainc(mpmath.mpf(df) / 2, mpmath.mpf(s) / 2, mpmath.inf, regularized=True)
                assert abs(chisq_upper(s, df)[0] / g - 1) < mpmath.mpf(10) ** -45
        assert abs(wald_p(9.0)[0] / mpmath.mpf("2.257176811907681e-19") - 1) < 1e-14
        assert abs(wald_p(-20.0)[0] / mpmath.mpf("5.507248237212467e-89") - 1) < 1e-14
        assert abs(chisq_upper(100.0, 1)[0] / mpmath.mpf("1.523970604832105e-23") - 1) < 1e-14
    assert wald_p(0.0)[0] == 1 and wald_p(math.inf)[0] == 0 and chisq_upper(-1e-13, 3)[0] == 1
    # the exact p.adjust on a hand-worked vector (test_results_device.test_p_adjust_hand_worked's values)
    p = np.array([0.01, NAN, 0.04, 0.03, 0.03, 0.5])
    for method, want in (("holm", [0.05, NAN, 0.12, 0.12, 0.12, 0.5]), ("hochberg", [0.05, NAN, 0.08, 0.08, 0.08, 0.5]),
                         ("BH", [0.05, NAN, 0.05, 0.05, 0.05, 0.5]), ("bonferroni", [0.05, NAN, 0.2, 0.15, 0.15, 1.0])):
        got = [float(v) for v in p_adjust_exact(p, method)[0]]
        assert np.allclose(got, want, rtol=1e-15, equal_nan=True), method
    by = [float(v) for v in p_adjust_exact(p, "BY")[0]]
    assert np.allclose(by, pipeline.p_adjust(p, "BY"), rtol=1e-14, equal_nan=True)


# ---------------------------------------------------------------- 1. function sweep

Z_SWEEP = np.r_[np.linspace(0.0, 40.0, 801), 8.29, 8.30, 37.5193, 38.5, 1e-300, 5e-324, 1e-8]
DFS = (1, 2, 3, 4, 5, 9, 10, 31)
S_SWEEP = np.r_[np.linspace(0.0, 1450.0, 291)[1:], np.linspace(0.0, 10.0, 201)[1:], 1e-300, 1e-12, 1e-3, 0.1, 0.5, 1.0, 2.0, 3.84, 6.63, 10.83]


def test_wald_stats_sweep(tdev):
    """_wald_stats (DESeq_device, its betaPrior / weights / nf paths, the sharded pipeline, lfcShrink_device) on a
    synthetic fit: the dense z grid over [0, 40] with both signs, the switch points of ndtr and erfc, +-inf (SE 0) and
    NaN (0 / 0 and a NaN coefficient)."""
    from deseq2_b200 import device_pipeline as DP
    z = np.r_[Z_SWEEP, -Z_SWEEP]
    beta = np.r_[z * LN2, 1.0, -1.0, 0.0, NAN]
    var = np.r_[np.full(len(z), LN2 ** 2), 0.0, 0.0, 0.0, LN2 ** 2]
    fit = {"beta_mat": torch.tensor(np.stack([beta, -beta]), device=tdev),
           "beta_var_mat": torch.tensor(np.stack([var, var]), device=tdev)}
    st = DP._wald_stats(fit)
    stat, p = _np(st["WaldStatistic"]), _np(st["WaldPvalue"])
    assert stat.shape == (len(beta), 2)
    assert np.array_equal(np.isinf(stat[:, 0]), np.r_[np.zeros(len(z), bool), True, True, False, False])
    assert np.all(p[stat == 0] == 1.0) and np.all(p[np.isinf(stat)] == 0.0)
    assert np.array_equal(np.isnan(p), np.isnan(stat)) and np.isnan(stat[-2:]).all()
    check_wald(p, stat, f"_wald_stats on {tdev.type}")


def test_lrt_stats_sweep(tdev):
    """_lrt_stats at df 1-31 for s up to 1450 (stat = 2 (s / 2 - 0) = s exactly), rounding-negative statistics,
    +inf and NaN."""
    from deseq2_b200 import device_pipeline as DP
    s = np.r_[S_SWEEP, -1e-13, -1e-300, -2.0, 0.0, math.inf, NAN]
    llf = torch.tensor(np.r_[s[:-2] / 2, math.inf, NAN], device=tdev)
    llr = torch.zeros(len(s), dtype=torch.float64, device=tdev)
    worst = {}
    for df in DFS:
        stat, p = DP._lrt_stats(llf, llr, df)
        stat, p = _np(stat), _np(p)
        assert np.array_equal(stat, s, equal_nan=True)
        assert np.all(p[s <= 0] == 1.0) and p[np.isinf(s)][0] == 0.0 and np.isnan(p[-1])
        worst[df] = check_chisq(p, stat, df, f"_lrt_stats df {df} on {tdev.type}")
    print(f"chi-square sweep on {tdev.type}, largest error / bound per df: {worst}")


# ---------------------------------------------------------------- 2. the results kernel

def _results_inputs(dev, T):
    """A synthetic DESeq_device result (x = ~condition, m = 4) whose condition column has LFC / SE chosen so that every
    threshold argument q sweeps [-45, 45] (q near 0, 8-10, 30-38, beyond) at SE = T / 20, T / 3 and 2 T: one term of
    greaterAbs underflows wherever T / SE is large.  Rows of LFC T + q SE, -(T + q SE) and q SE."""
    from deseq2_b200 import device_pipeline as DP
    q = np.r_[np.linspace(-45.0, 45.0, 181), 8.29, 8.3, 9.0, 37.5193, 38.5, -8.3, -37.5193, 1e-300]
    lfc, se = [], []
    for s in (T / 20, T / 3, 2 * T):
        for v in (T + q * s, -(T + q * s), q * s):
            lfc.append(v)
            se.append(np.full(len(q), s))
    lfc, se = np.concatenate(lfc), np.concatenate(se)
    lfc[:3], se[:3] = (0.0, 1.0, NAN), (0.0, 0.0, 1.0)            # 0 / 0, 1 / 0 and a NaN coefficient
    n, m = len(lfc), 4
    beta = np.stack([np.full(n, 5.0), lfc]) * LN2
    var = np.stack([np.full(n, 0.01), se ** 2]) * LN2 ** 2
    res = DP._wald_stats({"beta_mat": torch.tensor(beta, device=dev), "beta_var_mat": torch.tensor(var, device=dev)})
    res.update(idx=torch.arange(n, device=dev), test="Wald", sizeFactors=np.ones(m),
               baseMean=torch.tensor(np.linspace(1.0, 500.0, n)[np.random.default_rng(3).permutation(n)], device=dev))
    y = gm(np.ones((n, m), np.int32), dev)
    return res, y, synth.design_condition(m)


@pytest.mark.parametrize("T", [0.5, 2.0])
def test_results_kernel_tails(backend, T):
    """results_device on the coefficient column with each altHypothesis at threshold T, and without a threshold (the
    WaldPvalue column passed through): stat equal to R's float64 expressions bit for bit, pvalue within the tail
    bounds, padj the exact p.adjust of pvalue."""
    DP, dev, _ = backend
    res, y, x = _results_inputs(dev, T)
    out = DP.results_device(res, y, x, name=1, cooksCutoff=False)
    assert np.array_equal(_np(out["stat"]), _np(res["WaldStatistic"][:, 1]), equal_nan=True)
    check_wald(out["pvalue"], out["stat"], f"results_device lfcThreshold 0 (T {T})")
    check_padj(out, res["baseMean"])
    for alt in ALTS:
        out = DP.results_device(res, y, x, name=1, lfcThreshold=T, altHypothesis=alt, cooksCutoff=False,
                                pAdjustMethod="BY" if alt == "lessAbs" else "BH")
        lfc, se = _np(out["log2FoldChange"]), _np(out["lfcSE"])
        assert np.array_equal(lfc, _np(res["betaMatrix"][:, 1]), equal_nan=True)
        stat, refs = threshold_ref(alt, lfc, se, T)
        assert np.array_equal(_np(out["stat"]), stat, equal_nan=True), alt
        check_tails(_np(out["pvalue"]), refs, f"results_device {alt} T {T}", stat)
        check_padj(out, res["baseMean"], "BY" if alt == "lessAbs" else "BH")


def test_padj_methods(backend):
    """p_value_adjustment with every method, with and without independent filtering, on p-values that span 1e-300
    to 1 with ties and NaN."""
    DP, dev, _ = backend
    rng = np.random.default_rng(8)
    n = 1300                                                     # more than two 512-thread chunks
    p = 10.0 ** -rng.uniform(0, 300, n)
    p[::7] = rng.uniform(0, 1, len(p[::7]))
    p[::29] = p[5]
    p[::31] = NAN
    filt = rng.uniform(0, 100, n)
    filt[::11] = 0.0
    for method in ("BH", "BY", "holm", "hochberg", "bonferroni", "none"):
        for indep in (False, True):
            padj, meta = DP.p_value_adjustment(torch.tensor(p, device=dev), torch.tensor(filt, device=dev),
                                               independentFiltering=indep, pAdjustMethod=method)
            check_padj({"pvalue": p, "padj": padj, "metadata": meta}, filt, method, indep)


# ---------------------------------------------------------------- 3. end to end

def _planted(n, m, x, seed):
    """An ordinary synthetic set with planted rows whose condition effect runs from 0 to 2^14 at base counts from a
    few to thousands: |stat| from 0 to about 60.  Condition is column 1 of x."""
    d = synth.make_example_counts(n, m, x=x, seed=seed)
    K = d["counts"].copy()
    cond = x[:, 1] == 1
    jitter = 1.0 + 0.04 * np.cos(np.arange(m))
    rows = []
    for c in (3, 30, 300, 3000):
        for L in (0.0, 0.5, 1.0, 2.0, 3.0, 4.0, 6.0, 8.0, 10.0, 12.0, 14.0):
            rows.append(np.round(c * jitter * np.where(cond, 2.0 ** L, 1.0)))
    P = np.asarray(rows)
    K[:len(P)] = np.minimum(P, 2 ** 31 - 1).astype(np.int32)
    return K, d["sizeFactors"]


def _e2e_case(big):
    if big:
        n, m = 50000, 100
    else:
        n, m = 160, 12
    factors = [np.tile([0, 1], m // 2), np.repeat([0, 1], m // 2)]
    x = pipeline.factorDesign(factors)[0]                       # intercept, condition, batch
    K, sf = _planted(n, m, x, seed=23)
    return K, sf, x, factors


def _span(stat, what):
    a = np.abs(_np(stat))
    a = a[np.isfinite(a)]
    assert a.max() > 35 and np.any((a > 8.3) & (a < 30)), (what, "the planted rows no longer reach the far tail")


@pytest.fixture(params=[False, pytest.param(True, marks=pytest.mark.gpu)], ids=["small", "C2"])
def e2e(request, backend):
    """(device_pipeline, device, counts, gene-major y, size factors, x, factors): small on the emulator and the GPU,
    C2 (50 000 x 100) on the GPU only."""
    DP, dev, gpu = backend
    if request.param and not gpu:
        pytest.skip("C2 size runs on the GPU only")
    K, sf, x, factors = _e2e_case(request.param)
    return DP, dev, K, gm(K, dev), sf, x, factors


def test_deseq_wald_results_and_shrink(e2e):
    """DESeq_device's WaldPvalue (every column), results_device by name and by contrast (getContrast_device), padj,
    getContrast_device itself and lfcShrink_device."""
    DP, dev, K, y, sf, x, factors = e2e
    res = DP.DESeq_device(y, x, sf)
    _span(res["WaldStatistic"][:, 1], "Wald")
    check_wald(res["WaldPvalue"], res["WaldStatistic"], "DESeq_device WaldPvalue")
    out = DP.results_device(res, y, x, name=1, factors=factors)
    check_wald(out["pvalue"], out["stat"], "results_device by name", na=True)
    check_padj(out, out["baseMean"])
    con = np.array([0.0, 1.0, 0.5])
    out = DP.results_device(res, y, x, contrast=con, factors=factors)
    check_wald(out["pvalue"], out["stat"], "results_device by contrast", na=True)
    check_padj(out, out["baseMean"])
    ynz = y[res["idx"]].contiguous()
    g = DP.getContrast_device(ynz, x, sf, res["dispersion"], res["betaMatrix"], con)
    check_wald(g["pvalue"], g["stat"], "getContrast_device")
    sh = DP.lfcShrink_device(res, y, x, coef=1, factors=factors)
    check_wald(sh["pvalue"], sh["stat"], "lfcShrink_device", na=True)
    sh = DP.lfcShrink_device(res, y, x, coef=1, factors=factors, lfcThreshold=0.5)
    lfc, se = _np(sh["log2FoldChange"]), _np(sh["lfcSE"])
    stat, refs = threshold_ref("greaterAbs", lfc, se, 0.5)
    assert np.array_equal(_np(sh["stat"]), stat, equal_nan=True)
    check_tails(_np(sh["pvalue"]), refs, "lfcShrink_device lfcThreshold 0.5", stat, na=True)


@pytest.mark.parametrize("reduced", ["intercept", "batch"])
def test_deseq_lrt(e2e, reduced):
    """DESeq_device(test="LRT") against ~1 (R's closed form, df 2) and ~batch + condition against ~batch (df 1):
    LRTPvalue and results_device of the LRT result, with its padj."""
    DP, dev, K, y, sf, x, factors = e2e
    xr = x[:, :1] if reduced == "intercept" else x[:, [0, 2]]
    res = DP.DESeq_device(y, x, sf, test="LRT", reduced=xr)
    df = res["df"]
    assert df == x.shape[1] - xr.shape[1]
    check_chisq(res["LRTPvalue"], res["LRTStatistic"], df, f"DESeq_device LRT ~{reduced} df {df}")
    s = _np(res["LRTStatistic"])
    assert np.nanmax(s) > 1000 and np.any(s < 1)
    out = DP.results_device(res, y, x, name=1, factors=factors)
    check_chisq(out["pvalue"], out["stat"], df, "results_device of an LRT result", na=True)
    check_padj(out, out["baseMean"])


@pytest.mark.parametrize("variant", ["betaPrior", "weights", "nf"])
def test_deseq_variants(e2e, variant):
    """WaldPvalue of the betaPrior, weights and normalization-factor paths, and results_device on each."""
    DP, dev, K, y, sf, x, factors = e2e
    rng = np.random.default_rng(5)
    kw, rkw = {}, {}
    if variant == "betaPrior":
        kw = dict(betaPrior=True, factors=factors)
    elif variant == "weights":
        kw = dict(weights=gm(rng.uniform(0.5, 1.0, K.shape), dev, np.float64))
        rkw = dict(weights=kw["weights"])
    else:
        nf = sf[None, :] * np.exp(rng.normal(0, 0.1, K.shape))
        kw = dict(normalizationFactors=gm(nf, dev, np.float64))
        sf = None
    res = DP.DESeq_device(y, x, sf, **kw)
    check_wald(res["WaldPvalue"], res["WaldStatistic"], f"DESeq_device {variant} WaldPvalue")
    out = DP.results_device(res, y, x, factors=factors, **rkw)
    check_wald(out["pvalue"], out["stat"], f"results_device {variant}", na=True)
    check_padj(out, out["baseMean"])


# ---------------------------------------------------------------- 4. the host mirror

def test_host_mirror(oracle):
    """pipeline.nbinomWaldTest / nbinomLRT / getContrast, the reference of the other device tests, on the oracle."""
    K, sf, x, factors = _e2e_case(False)
    K = K[K.sum(axis=1) > 0]
    nf = np.broadcast_to(sf[None, :], K.shape)
    alpha = np.clip(0.05 + 1.0 / (K / sf).mean(axis=1), 1e-8, 10.0)
    w = pipeline.nbinomWaldTest(K, nf, x, alpha, engine=oracle)
    _span(w["WaldStatistic"][:, 1], "host Wald")
    check_wald(w["WaldPvalue"], w["WaldStatistic"], "pipeline.nbinomWaldTest")
    lr = pipeline.nbinomLRT(K, nf, x, x[:, [0, 2]], alpha, engine=oracle)
    check_chisq(lr["LRTPvalue"], lr["LRTStatistic"], 1, "pipeline.nbinomLRT")
    g = pipeline.getContrast(K, nf, x, alpha, w["betaMatrix"], np.array([0.0, 1.0, 0.5]), engine=oracle)
    check_wald(g["pvalue"], g["stat"], "pipeline.getContrast")
