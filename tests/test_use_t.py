"""DESeq(useT = TRUE) on the device: the Student t tail device_pipeline.t_upper / t_wald_pvalue and its numpy twin
pipeline.r_pt_upper against a 50-digit mpmath tail, the host mirror against R's formulas (R/core.R:1478-1508,
R/results.R:414, 477-518, 812-816, refitWithoutOutliers :2484-2565), the device against the host mirror, invariants
that need no mirror, and the gene shards.  The CPU tests run the engine on the SIMT emulator (`emu_dev`) and the ranks
over gloo; the `-m gpu` tests run on the H100 and the ranks over NCCL.

Tail accuracy contract: |p - p*| <= (C + kappa) 2^-52 p* wherever p* >= DBL_MIN, with p* the 50-digit tail at the
float64 arguments, kappa = |q f(q) / (1 - F(q))| its condition number (also at 50 digits) and C = 64; below DBL_MIN any
0 <= p <= DBL_MIN."""
import math

import mpmath as mp
import numpy as np
import pytest
import torch
from scipy import special as sps

from helpers import DEV, emu_dev, gm  # noqa: F401
from deseq2_b200 import pipeline, synth
from ranks import DEVICE, nccl_world, run_ranks

DBL_MIN = 2.2250738585072014e-308
ULP = 2.0 ** -52
C_TAIL = 64
NUS = [0.3, 0.5, 1.0, 1.5, 2.0, 3.0, 7.25, 10.0, 98.0, 1000.0, 35000.0, 1e6]
COLS = ("baseMean", "log2FoldChange", "lfcSE", "stat", "pvalue", "padj")


# ---------------------------------------------------------------- the 50-digit reference

def _two_sided_ref(q, nu):
    """2 (1 - F_nu(|q|)) at 50 significant digits: I_x(nu/2, 1/2) = x^a y^(1/2) / (a B(a, 1/2)) 2F1(a + 1/2, 1; a + 1; x)
    for y = q^2 / (nu + q^2) >= 1/2, else 1 - I_y(1/2, a) with 2F1(a + 1/2, 1; 3/2; y) (both sums of positive terms),
    worked with enough digits that the subtraction keeps 50."""
    q, nu = mp.mpf(abs(float(q))), mp.mpf(float(nu))
    if q == 0:
        return mp.mpf(1)
    h, a = mp.mpf(1) / 2, nu / 2
    L = float(mp.log1p(q * q / nu))
    small_y = float(q * q / (nu + q * q)) < 0.5
    with mp.workdps(70 + (int(float(a) * L / 2.3) if small_y else 0)):
        y, x = q * q / (nu + q * q), nu / (nu + q * q)
        if small_y:
            return +(1 - mp.sqrt(y) * mp.power(x, a) / (h * mp.beta(h, a)) * mp.hyp2f1(a + h, 1, h + 1, y,
                                                                                          maxterms=10 ** 7))
        return +(mp.power(x, a) * mp.sqrt(y) / (a * mp.beta(a, h)) * mp.hyp2f1(a + h, 1, a + 1, x, maxterms=10 ** 7))


def _upper_ref(q, nu):
    """(pt(q, nu, lower.tail = FALSE), its condition number), or None when the tail is surely below DBL_MIN."""
    qq, n = mp.mpf(float(q)), mp.mpf(float(nu))
    if float(n / 2 * mp.log1p(qq * qq / n)) > 800:
        return None
    mp.mp.dps = 50
    two = _two_sided_ref(q, nu)
    p = two / 2 if q >= 0 else 1 - two / 2
    lf = mp.loggamma((n + 1) / 2) - mp.log(mp.sqrt(n * mp.pi)) - mp.loggamma(n / 2) - (n + 1) / 2 * mp.log1p(qq * qq / n)
    return p, abs(qq * mp.exp(lf) / p)


def _grid(nu):
    q = np.r_[-np.geomspace(1e-3, 30.0, 9), 0.0, np.linspace(0.05, 5.0, 34), np.geomspace(5.0, 1e300, 60)]
    return q[np.log1p(q * q / nu) * nu / 2 < 820]


def _check_tail(values, qs, nu, C=C_TAIL):
    worst = 0.0
    for q, v in zip(qs, values):
        r = _upper_ref(q, nu)
        if r is None or r[0] < DBL_MIN:
            assert 0.0 <= v <= DBL_MIN, (nu, q, v)
            continue
        p, kappa = r
        err = float(abs(mp.mpf(float(v)) - p) / p) / ULP
        assert err <= C + float(kappa), (nu, q, v, float(p), err, float(kappa))
        worst = max(worst, err - float(kappa))
    return worst


@pytest.mark.parametrize("nu", NUS)
def test_t_upper_against_50_digits_cpu(nu):
    from deseq2_b200 import device_pipeline as DP
    qs = _grid(nu)
    v = DP.t_upper(torch.tensor(qs), torch.full((qs.size,), nu, dtype=torch.float64)).numpy()
    _check_tail(v, qs, nu)


@pytest.mark.parametrize("nu", NUS)
def test_numpy_twin_against_50_digits(nu):
    qs = _grid(nu)
    _check_tail(pipeline.r_pt_upper(qs, nu), qs, nu)


@pytest.mark.gpu
@pytest.mark.parametrize("nu", NUS)
def test_t_upper_against_50_digits_gpu(nu):
    from deseq2_b200 import device_pipeline as DP
    qs = _grid(nu)
    v = DP.t_upper(torch.tensor(qs, device=DEV), torch.full((qs.size,), nu, dtype=torch.float64, device=DEV))
    _check_tail(v.cpu().numpy(), qs, nu)


def _check_special_values(dev):
    from deseq2_b200 import device_pipeline as DP
    z = torch.tensor(np.r_[0.0, 1e-300, 0.3, 1.0, 2.5, 8.3, 9.0, 20.0, 37.5, 38.5, 1e3, np.inf, -np.inf, -3.0, np.nan],
                     device=dev)
    inf = torch.full_like(z, math.inf)
    # df = Inf: wald_pvalue's bits, and the normal tail for the one-sided form
    assert torch.equal(torch.nan_to_num(DP.t_wald_pvalue(z, inf), nan=-1.0),
                       torch.nan_to_num(DP.wald_pvalue(z), nan=-1.0))
    assert torch.equal(torch.nan_to_num(DP.t_upper(z, inf), nan=-1.0),
                       torch.nan_to_num(0.5 * torch.erfc(z * 0.7071067811865476), nan=-1.0))
    # df NaN or <= 0: NaN, as R's NA
    for bad in (math.nan, 0.0, -1.0, -math.inf):
        d = torch.full_like(z, bad)
        assert torch.isnan(DP.t_upper(z, d)).all() and torch.isnan(DP.t_wald_pvalue(z, d)).all()
    d = torch.full_like(z, 7.25)
    u = DP.t_upper(z, d).cpu().numpy()
    assert u[0] == 0.5 and u[11] == 0.0 and u[12] == 1.0 and np.isnan(u[-1])
    w = DP.t_wald_pvalue(z, d).cpu().numpy()
    assert w[0] == 1.0 and w[11] == 0.0 and w[12] == 0.0
    # a (p, n) statistic with per-gene df broadcast along the genes, as DESeq_device calls it
    s = torch.linspace(-6.0, 6.0, 12, dtype=torch.float64, device=dev).reshape(2, 6)
    df = torch.tensor([0.4, 3.0, 17.5, 98.0, math.inf, math.nan], dtype=torch.float64, device=dev)
    got = DP.t_wald_pvalue(s, df).cpu().numpy()
    want = pipeline.waldPvalue(s.cpu().numpy().T, df.cpu().numpy()).T
    assert np.allclose(got, want, rtol=1e-13, atol=0, equal_nan=True)


def test_special_values_cpu():
    _check_special_values("cpu")


@pytest.mark.gpu
def test_special_values_gpu():
    _check_special_values(DEV)


def test_t_tail_is_heavier_than_the_normal_tail():
    """2 pt(|z|, df, lower = FALSE) >= 2 pnorm(|z|, lower = FALSE) at every z, and increases toward it as df grows."""
    from deseq2_b200 import device_pipeline as DP
    z = torch.tensor(np.r_[np.linspace(0.01, 12.0, 200), 20.0, 30.0], dtype=torch.float64)
    norm = DP.wald_pvalue(z)
    prev = None
    for nu in (0.5, 2.0, 10.0, 98.0, 1e4, 1e8):
        t = DP.t_wald_pvalue(z, torch.full_like(z, nu))
        assert bool((t >= norm * (1 - 80 * ULP * (1 + z * z))).all()), nu
        if prev is not None:
            assert bool((t <= prev * (1 + 80 * ULP * (1 + z * z))).all()), nu
        prev = t


# ---------------------------------------------------------------- the host mirror against R's formulas

def _case(kind, seed=7):
    """(counts, x, factors, DESeq kwargs) of a named design, with all-zero rows."""
    if kind == "replace":
        factors = [np.repeat([0, 1, 2], 7)]
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(240, 21, x=x, seed=seed)
        K = d["counts"].copy()
        K[0] = np.repeat([100, 200, 400], 7)
        K[0, 9] = 20000
        K[1] = 0
        K[1, 16] = 500
        K[3:5] = 0
        return K, x, factors, dict(sizeFactors=d["sizeFactors"], minReplicatesForReplace=7)
    factors = [np.tile([0, 1], 5), np.repeat([0, 1], 5)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(240, 10, x=x, seed=seed)
    K = d["counts"].copy()
    K[3:6] = 0
    return K, x, factors, dict(sizeFactors=d["sizeFactors"])


def _weights(K, seed=5):
    w = np.random.default_rng(seed).uniform(0.05, 1.0, K.shape)
    w[:, 0] = 1.0
    return w


def test_host_degrees_of_freedom(emu_dev):
    E = dict(engine=emu_dev)
    K, x, factors, kw = _case("batch")
    N, m = K.shape
    p = x.shape[1]
    nz = K.sum(axis=1) > 0
    plain = pipeline.DESeq(K, x, useT=True, **kw, **E)
    assert np.array_equal(plain["tDegreesFreedom"][nz], np.full(nz.sum(), float(m - p)))
    assert np.isnan(plain["tDegreesFreedom"][~nz]).all()
    # 2 pt(|z|, df, lower = FALSE), R's formula at df = m - p
    want = 2.0 * sps.stdtr(m - p, -np.abs(plain["WaldStatistic"][nz]))
    assert np.allclose(plain["WaldPvalue"][nz], want, rtol=1e-12, atol=0)
    # given df: a scalar, and one per input row subset to the tested rows; df <= 0 is NA
    df = np.linspace(-1.0, 30.0, N)
    per = pipeline.DESeq(K, x, useT=True, df=df, **kw, **E)
    want_df = np.where(df > 0, df, np.nan)
    assert np.array_equal(per["tDegreesFreedom"][nz], want_df[nz], equal_nan=True)
    assert np.isnan(per["WaldPvalue"][nz & (df <= 0)]).all()
    assert np.array_equal(pipeline.DESeq(K, x, useT=True, df=4.5, **kw, **E)["tDegreesFreedom"][nz], np.full(nz.sum(), 4.5))
    with pytest.raises(ValueError, match="one value per row"):
        pipeline.DESeq(K, x, useT=True, df=np.ones(N - 1), **kw, **E)
    # weights: rowSums of the normalised weights minus p
    w = _weights(K)
    wt = pipeline.DESeq(K, x, useT=True, weights=w, **kw, **E)
    keep = nz & ~wt["weightsFail"]
    wn = w / w.max(axis=1, keepdims=True)
    assert np.allclose(wt["tDegreesFreedom"][keep], wn[keep].sum(axis=1) - p, rtol=1e-14, atol=0)
    # betaPrior: the standard design's p, not the expanded matrix's
    bp = pipeline.DESeq(K, x, useT=True, betaPrior=True, factors=factors, **kw, **E)
    assert np.array_equal(bp["tDegreesFreedom"][nz], np.full(nz.sum(), float(m - p)))
    assert bp["WaldStatistic"].shape[1] > p
    # the LRT ignores useT and adds no column
    lrt = pipeline.DESeq(K, x, useT=True, test="LRT", reduced=x[:, :-1], **kw, **E)
    assert "tDegreesFreedom" not in lrt
    # useT=False is the normal tail
    assert "tDegreesFreedom" not in pipeline.DESeq(K, x, **kw, **E)


def test_host_outlier_refit_quirk(emu_dev):
    """refitWithoutOutliers does not pass useT: the refitted rows get normal p-values and keep the first fit's df; a
    row all zero once replaced gets NA in every results column, df included."""
    K, x, _, kw = _case("replace")
    m, p = x.shape
    r = pipeline.DESeq(K, x, useT=True, engine=emu_dev, **kw)
    rep = r["replace"]
    assert rep.sum() >= 2 and rep[0] and rep[1]
    refit = rep & (r["baseMean"] > 0)
    assert np.array_equal(r["WaldPvalue"][refit], 2.0 * sps.ndtr(-np.abs(r["WaldStatistic"][refit])))
    assert np.array_equal(r["tDegreesFreedom"][refit], np.full(refit.sum(), float(m - p)))
    assert np.isnan(r["tDegreesFreedom"][1]) and np.isnan(r["WaldPvalue"][1]).all()
    other = ~rep & (K.sum(axis=1) > 0)
    assert np.allclose(r["WaldPvalue"][other], 2.0 * sps.stdtr(m - p, -np.abs(r["WaldStatistic"][other])),
                       rtol=1e-12, atol=0)


def _threshold_restated(lfc, se, T, alt, df):
    """R/results.R:477-518 with useT, stated with scipy's stdtr (pt(q, df) = stdtr(df, q)), each gene at its df."""
    pt = lambda q: sps.stdtr(df, q)
    up = lambda q: sps.stdtr(df, -q)
    with np.errstate(divide="ignore", invalid="ignore"):
        if alt == "greaterAbs":
            return pt((-np.abs(lfc) + T) / se) + pt((-np.abs(lfc) - T) / se)
        if alt == "greaterAbs2014":
            return np.minimum(1.0, 2.0 * up((np.abs(lfc) - T) / se))
        if alt == "lessAbs":
            return np.maximum(up((T - lfc) / se), up((lfc + T) / se))
        if alt == "greater":
            return up((lfc - T) / se)
        return up((-T - lfc) / se)


@pytest.mark.parametrize("alt", pipeline.ALT_HYPOTHESES)
def test_host_threshold_matches_restatement(emu_dev, alt):
    K, x, factors, kw = _case("batch")
    dds = pipeline.DESeq(K, x, useT=True, df=np.linspace(0.5, 40.0, K.shape[0]), engine=emu_dev, **kw)
    res = pipeline.results(dds, K, x, name=2, lfcThreshold=0.5, altHypothesis=alt, cooksCutoff=False, factors=factors,
                           engine=emu_dev)
    f = ~np.isnan(res["pvalue"])
    want = _threshold_restated(res["log2FoldChange"], res["lfcSE"], 0.5, alt, dds["tDegreesFreedom"])
    assert f.sum() > 100
    assert np.allclose(res["pvalue"][f], want[f], rtol=1e-12, atol=1e-300)
    with pytest.raises(ValueError, match="useT is not supported"):
        pipeline.results(dds, K, x, name=2, useT=True, engine=emu_dev)


# ---------------------------------------------------------------- the device against the host mirror

def _host_dds(res, K, x, w=None):
    N, m = K.shape
    idx = res["idx"].cpu().numpy()

    def full(v, fill=np.nan):
        v = v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        a = np.full((N,) + v.shape[1:], fill)
        a[idx] = v
        return a

    keys = ["betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "maxCooks", "dispersion", "dispFit",
            "tDegreesFreedom"]
    dds = {k: full(res[k]) for k in keys if k in res}
    dds["baseMean"] = full(res["baseMean"], 0.0)
    dds["allZero"] = np.ones(N, bool)
    dds["allZero"][idx] = False
    dds["sizeFactors"] = res["sizeFactors"]
    dds["test"] = "Wald"
    if res.get("modelMatrix") is not None:
        dds["modelMatrix"], dds["betaPriorVar"] = res["modelMatrix"], res["betaPriorVar"]
    if w is not None:
        dds["weights"] = res["weights"][:, :m].cpu().numpy()
        dds["weightsFail"] = res["weightsFail"].cpu().numpy()
        dds["baseMean"][dds["weightsFail"]] = pipeline.getBaseMeansAndVariances(
            K, res["sizeFactors"], w)["baseMean"][dds["weightsFail"]]
    return dds


def _close(a, b, tol, what):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    assert np.array_equal(np.isnan(a), np.isnan(b)), what
    f = ~np.isnan(b)
    err = np.abs(a[f] - b[f]) / np.maximum(np.abs(b[f]), 1e-300)
    assert np.all(err <= tol), (what, float(err.max()))


DEVICE_CASES = {
    "plain": (dict(), dict(name=2)),
    "df_vector": (dict(df="vector"), dict(name=1)),
    "weights": (dict(w=True), dict(name=2)),
    "nf": (dict(nf=True), dict(name=1)),
    "beta_prior": (dict(betaPrior=True), dict(contrast=(1, 1, 0))),
    "fit_type_mean": (dict(fitType="mean"), dict(name=2)),
    "contrast": (dict(), dict(contrast=np.array([0.0, 1.0, -1.0]))),
    "threshold": (dict(), dict(name=2, lfcThreshold=0.4)),
    "threshold_less": (dict(), dict(name=1, lfcThreshold=0.3, altHypothesis="less")),
    "threshold_contrast": (dict(), dict(contrast=np.array([0.0, 1.0, -1.0]), lfcThreshold=0.3,
                                        altHypothesis="greaterAbs2014")),
}


def _device_vs_host(dev, engine, case):
    from deseq2_b200 import device_pipeline as DP
    dkw, rkw = DEVICE_CASES[case]
    dkw = dict(dkw)
    K, x, factors, kw = _case("batch")
    N, m = K.shape
    y = gm(K, dev)
    w = nf = None
    if dkw.pop("w", False):
        w = _weights(K)
        kw["weights"] = gm(w, dev)
    if dkw.pop("nf", False):
        nf = np.exp(np.random.default_rng(2).normal(0, 0.2, K.shape))
        kw["normalizationFactors"], kw["sizeFactors"] = gm(nf, dev), None
    if dkw.get("df") == "vector":
        dkw["df"] = np.linspace(-2.0, 25.0, N)
    if dkw.get("betaPrior"):
        kw["factors"] = factors
    res = DP.DESeq_device(y, x, useT=True, **dkw, **kw)
    hkw = {k: v for k, v in kw.items() if k not in ("weights", "normalizationFactors")}
    host = pipeline.DESeq(K, x, useT=True, weights=w, normalizationFactors=nf, engine=engine, **dkw, **hkw)
    idx = res["idx"].cpu().numpy()
    assert np.array_equal(res["tDegreesFreedom"].cpu().numpy(), host["tDegreesFreedom"][idx], equal_nan=True) or \
        np.allclose(res["tDegreesFreedom"].cpu().numpy(), host["tDegreesFreedom"][idx], rtol=1e-14, equal_nan=True)
    # the device's p-values at its own statistics: the tail bound against the numpy twin at the same arguments
    z = res["WaldStatistic"].cpu().numpy()
    _close(res["WaldPvalue"], pipeline.waldPvalue(z, res["tDegreesFreedom"].cpu().numpy()), 1e-12, "WaldPvalue")
    # the whole pipeline against the mirror: the fits agree to the IRLS tolerance on nearly every gene
    a, b = res["WaldPvalue"].cpu().numpy(), host["WaldPvalue"][idx]
    assert np.array_equal(np.isnan(a), np.isnan(b))
    f = ~np.isnan(b)
    assert np.median(np.abs(a[f] - b[f]) / b[f]) < 1e-8 and np.mean(np.abs(a[f] - b[f]) <= 1e-4 * b[f]) > 0.97
    # results(): the device table against the host mirror fed the device's fit
    dds = _host_dds(res, K, x, w)
    tab = DP.results_device(res, y, x, factors=factors, weights=kw.get("weights"), cooksCutoff=False, **rkw)
    ht = pipeline.results(dds, K, x, factors=factors, engine=engine, cooksCutoff=False, **rkw)
    for k in COLS:
        _close(tab[k], ht[k], 1e-9, k)
    return res, tab


@pytest.mark.parametrize("case", list(DEVICE_CASES))
def test_device_matches_host_emulated(emu_dev, case):
    _device_vs_host("cpu", emu_dev, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(DEVICE_CASES))
def test_device_matches_host_gpu(engine, case):
    _device_vs_host(DEV, engine, case)


def _check_refit_and_shrink(dev, engine):
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("replace")
    m, p = x.shape
    y = gm(K, dev)
    res = DP.DESeq_device(y, x, useT=True, **kw)
    idx = res["idx"].cpu().numpy()
    host = pipeline.DESeq(K, x, useT=True, engine=engine, **kw)
    rep = res["replace"].cpu().numpy()
    refit = rep & (res["baseMean"].cpu().numpy() > 0)
    z = res["WaldStatistic"].cpu().numpy()
    pv = res["WaldPvalue"].cpu().numpy()
    tdf = res["tDegreesFreedom"].cpu().numpy()
    assert refit.sum() >= 1
    assert np.array_equal(pv[refit], DP.wald_pvalue(res["WaldStatistic"][torch.as_tensor(refit)]).cpu().numpy())
    assert np.array_equal(tdf[refit], np.full(refit.sum(), float(m - p)))
    assert np.array_equal(np.isnan(tdf), np.isnan(host["tDegreesFreedom"][idx]))
    _close(pv, host["WaldPvalue"][idx], 1e-4, "WaldPvalue")
    _close(pv[~rep], pipeline.waldPvalue(z[~rep], tdf[~rep]), 1e-12, "first fit")
    # lfcShrink: the shrunk table's test is normal (its MAP refit's nbinomWaldTest drops tDegreesFreedom)
    K2, x2, factors2, kw2 = _case("batch")
    y2 = gm(K2, dev)
    r2 = DP.DESeq_device(y2, x2, useT=True, **kw2)
    plain = DP.DESeq_device(y2, x2, **kw2)
    for kwl in (dict(coef=2), dict(coef=2, lfcThreshold=0.3)):
        a = DP.lfcShrink_device(r2, y2, x2, factors=factors2, **kwl)
        b = DP.lfcShrink_device(plain, y2, x2, factors=factors2, **kwl)
        for k in ("log2FoldChange", "lfcSE"):
            assert torch.equal(torch.nan_to_num(a[k], nan=-7.0), torch.nan_to_num(b[k], nan=-7.0)), k
        if kwl.get("lfcThreshold"):
            assert torch.equal(torch.nan_to_num(a["pvalue"], nan=-7.0), torch.nan_to_num(b["pvalue"], nan=-7.0))
        else:                                           # the default table is results() of the useT fit
            want = DP.results_device(r2, y2, x2, factors=factors2, name=2)
            assert torch.equal(torch.nan_to_num(a["pvalue"], nan=-7.0), torch.nan_to_num(want["pvalue"], nan=-7.0))
        dds = _host_dds(r2, K2, x2)
        hs = pipeline.lfcShrink(dds, K2, x2, factors=factors2, engine=engine, cooks=np.zeros(K2.shape), **kwl)
        for k in COLS:
            _close(a[k], hs[k], 1e-6, ("shrink", k))


def test_refit_and_shrink_emulated(emu_dev):
    _check_refit_and_shrink("cpu", emu_dev)


@pytest.mark.gpu
def test_refit_and_shrink_gpu(engine):
    _check_refit_and_shrink(DEV, engine)


# ---------------------------------------------------------------- invariants

def _eq(a, b):
    return torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0))


def _check_invariants(dev, n=240, m=10):
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("batch")
    if n != 240:
        factors = [np.tile([0, 1], m // 2), np.repeat([0, 1], m // 2)]
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(n, m, x=x, seed=3)
        K, kw = d["counts"], dict(sizeFactors=d["sizeFactors"])
    y = gm(K, dev)
    base = DP.DESeq_device(y, x, **kw)
    off = DP.DESeq_device(y, x, useT=False, df=3.0, **kw)
    inf = DP.DESeq_device(y, x, useT=True, df=math.inf, **kw)
    t = DP.DESeq_device(y, x, useT=True, **kw)
    for k in ("WaldStatistic", "WaldPvalue", "betaMatrix", "betaSE", "dispersion", "deviance"):
        assert _eq(off[k], base[k]) and _eq(inf[k], base[k]), k
    assert "tDegreesFreedom" not in off
    z = base["WaldStatistic"]
    assert bool((t["WaldPvalue"] >= base["WaldPvalue"] * (1 - 80 * ULP * (1 + z * z))).all())
    assert bool((t["WaldPvalue"] > base["WaldPvalue"])[z.abs() > 0.5].all())
    for rkw in (dict(name=2), dict(contrast=np.array([0.0, 1.0, -1.0])), dict(name=1, lfcThreshold=0.3),
                dict(name=1, lfcThreshold=0.3, altHypothesis="lessAbs")):
        a = DP.results_device(inf, y, x, factors=factors, **rkw)
        b = DP.results_device(base, y, x, factors=factors, **rkw)
        for k in COLS:
            assert _eq(a[k], b[k]), (rkw, k)
    return K, x, base, t


def test_invariants_emulated(emu_dev):
    _check_invariants("cpu")


@pytest.mark.gpu
def test_invariants_gpu_c2():
    """C2 size: 50 000 genes x 100 samples."""
    _check_invariants(DEV, 50000, 100)


def test_errors(emu_dev):
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("batch")
    y = gm(K, "cpu")
    with pytest.raises(ValueError, match="one value per row"):
        DP.DESeq_device(y, x, useT=True, df=np.ones(3), **kw)
    res = DP.DESeq_device(y, x, useT=True, **kw)
    with pytest.raises(ValueError, match="tDegreesFreedom"):
        DP.getContrast_device(y[res["idx"]].contiguous(), x, kw["sizeFactors"], res["dispersion"], res["betaMatrix"],
                              np.array([0.0, 1.0, 0.0]), useT=True)
    lrt = DP.DESeq_device(y, x, useT=True, test="LRT", reduced=x[:, :-1], **kw)
    assert "tDegreesFreedom" not in lrt
    plain = DP.DESeq_device(y, x, test="LRT", reduced=x[:, :-1], **kw)
    w1 = DP.results_device(lrt, y, x, factors=factors, name=2, test="Wald")
    w2 = DP.results_device(plain, y, x, factors=factors, name=2, test="Wald")
    assert _eq(w1["pvalue"], w2["pvalue"])


# ---------------------------------------------------------------- gene shards

def _sharded_case(n):
    factors = [np.tile([0, 1], 6), np.repeat([0, 1, 2], 4)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(n, 12, x=x, seed=41)
    K = d["counts"].copy()
    K[[5, n // 2]] = 0
    w = np.random.default_rng(9).uniform(0.2, 1.0, K.shape)
    w[:, 0] = 1.0
    return K, x, factors, d["sizeFactors"], w


def _bounds(n, world, tiny):
    """shard_bounds' shards, or with `tiny` three unequal shards whose middle one holds two rows."""
    if tiny:
        cuts = [0, n // 2, n // 2 + 2, n]
        return [(cuts[r], cuts[r + 1]) for r in range(world)]
    from deseq2_b200 import sharded
    return [sharded.shard_bounds(n, world, r) for r in range(world)]


_SHARD_CALLS = (("coef", dict(name=3)), ("contrast", dict(contrast=(1, 1, 2))),
                ("threshold", dict(name=2, lfcThreshold=0.4)))


def _sharded_rank(rank, world, dev, n, weighted, tiny):
    from deseq2_b200 import sharded
    K, x, factors, sf, w = _sharded_case(n)
    lo, hi = _bounds(n, world, tiny)[rank]
    y = gm(K[lo:hi], dev)
    kw = dict(weights=gm(w[lo:hi], dev)) if weighted else {}
    res = sharded.sharded_DESeq_device(y, x, sf, useT=True, df=np.linspace(1.0, 30.0, n)[lo:hi], **kw)
    out = {"WaldPvalue": res["WaldPvalue"], "tDegreesFreedom": res["tDegreesFreedom"],
           "collectives": res["collectives"]}
    if not tiny:                                     # sharded_results_device needs shard_bounds' layout
        for name, rkw in _SHARD_CALLS:
            r = sharded.sharded_results_device(res, y, x, factors=factors, weights=kw.get("weights"), **rkw)
            out[name] = {k: r[k] for k in COLS}
        r = sharded.sharded_lfcShrink_device(res, y, x, factors=factors, coef=3, weights=kw.get("weights"))
        out["shrink"] = {k: r[k] for k in COLS}
    return out


def _check_sharded(backend, n, world, weighted=False, tiny=False):
    from deseq2_b200 import device_pipeline as DP, sharded
    got = run_ranks(_sharded_rank, n, weighted, tiny, world=world, backend=backend)
    K, x, factors, sf, w = _sharded_case(n)
    dev = DEVICE[backend]
    y = gm(K, dev)
    kw = dict(weights=gm(w, dev)) if weighted else {}
    whole = DP.DESeq_device(y, x, sf, useT=True, df=np.linspace(1.0, 30.0, n), **kw)
    for g in got:
        assert g["collectives"] == 3                 # size agreement, global step, result gather: unchanged by useT
    for k in ("WaldPvalue", "tDegreesFreedom"):
        cat = np.concatenate([g[k] for g in got])
        assert np.array_equal(cat, whole[k].cpu().numpy(), equal_nan=True), k
    if tiny:
        return
    for name, rkw in _SHARD_CALLS:
        want = DP.results_device(whole, y, x, factors=factors, weights=kw.get("weights"), **rkw)
        for k in COLS:
            cat = np.concatenate([g[name][k] for g in got])
            assert np.array_equal(cat, want[k].cpu().numpy(), equal_nan=True), (name, k)
    want = DP.lfcShrink_device(whole, y, x, factors=factors, coef=3, weights=kw.get("weights"))
    for k in COLS:
        assert np.array_equal(np.concatenate([g["shrink"][k] for g in got]), want[k].cpu().numpy(), equal_nan=True), k


@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharded_equals_whole(emu_dev, world):
    _check_sharded("gloo", 301, world, weighted=world == 2)


def test_sharded_unequal_shards(emu_dev):
    _check_sharded("gloo", 301, 3, tiny=True)


@pytest.mark.gpu
def test_sharded_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, nccl_world(), weighted=True)
