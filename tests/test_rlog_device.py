"""rlog() on the device: the fit kernel (b200nb_rlog_fit_dev, csrc/rlog.cuh) against the reference's own fitBeta on
the design [1 | I_m] (I_m when the intercept is frozen), the prior-variance kernel (b200nb_rlog_prior_var_dev) against
pipeline.matchWeightedUpperQuantileForVariance, rlog_device against the host mirror (pipeline.rlog driving the
oracle), the frozen rlog, and the error cases.  The CPU tests run the engine's CUDA source on the SIMT emulator (`emu`
fixture); the `-m gpu` tests run on a GPU, or on the emulator when B200NB_LIB points at it."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm

LN2 = np.log(2.0)


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as R
    R.lib()
    return R


def _stream(dev):
    return None if dev == "cpu" else C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _within(got, want, bound=1e-6):
    return np.all(np.abs(got - want) <= bound * np.maximum(1.0, np.abs(want)))


# ---------------------------------------------------------------- the fit kernel against the reference's fitBeta

def _ref_rlog_fit(ref, K, nf, disp, bpv, intercept=None, maxit=100):
    """The reference's fitBeta (QR branch) with rlogData's design, lambdas and fitNbinomGLMs' start values; returns
    (values on the log2 scale, fitted log2 intercept or None, iter) over the rows R fits."""
    n, m = K.shape
    if intercept is None:
        x = np.c_[np.ones(m), np.eye(m)]
        lam = np.r_[1e-6, np.full(m, 1.0 / bpv)]
        beta0 = np.zeros((n, m + 1))
        beta0[:, 0] = np.log((K / nf).mean(axis=1))
        nfp = nf
    else:
        x = np.eye(m)
        lam = np.full(m, 1.0 / bpv)
        nfp = nf * 2.0 ** intercept[:, None]
        beta0 = np.log(K / nfp + 0.1)
    r = ref.fitBeta(K, x, nfp, disp, np.r_[1.0, np.zeros(x.shape[1] - 1)], beta0, lam / LN2 ** 2, None, False, 1e-4,
                    maxit, True, 0.5)
    b = r["beta_mat"] / LN2
    vals = b @ x.T
    if intercept is not None:
        vals = vals + intercept[:, None]
    return vals, (b[:, 0] if intercept is None else None), r["iter"]


def _fit_case(n, m, seed, f64=False):
    rng = np.random.default_rng(seed)
    mean = np.exp(rng.uniform(-1.0, 8.0, n))
    disp = 0.02 + 2.0 / mean + rng.uniform(0.0, 0.1, n)
    sf = np.exp(rng.normal(0.0, 0.3, m))
    nf = sf[None, :] * np.exp(rng.normal(0.0, 0.2, (n, m)))
    mu = mean[:, None] * nf
    K = rng.negative_binomial(1.0 / disp[:, None], 1.0 / (1.0 + disp[:, None] * mu)).astype(np.float64)
    K[1] = 0.0
    K[2, :] = 0.0
    K[2, 0] = 40.0                                      # zero-heavy rows
    K[3, ::2] = 0.0
    return K, sf, nf, disp                              # float64 counts too: integer values (dnbinom is 0 otherwise)


def _call_fit(y, m, disp, bpv, sf=None, nf=None, intercept=None, ld_out=None, maxit=100):
    """b200nb_rlog_fit_dev into an (n, ld_out) buffer prefilled with -7 (the padding must stay)."""
    from deseq2_b200 import _lib
    n, ld = y.shape
    ld_out = m if ld_out is None else ld_out
    dev = y.device
    out = torch.full((n, ld_out), -7.0, dtype=torch.float64, device=dev)
    icpt = torch.full((n,), -7.0, dtype=torch.float64, device=dev)
    it = torch.empty(n, dtype=torch.float64, device=dev)
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    rc = _lib.lib().b200nb_rlog_fit_dev(P(y), 1 if y.dtype == torch.float64 else 0, P(sf), P(nf), P(intercept),
                                        P(disp), n, m, ld, bpv, 1e-4, maxit, 0.5, P(out), ld_out, P(icpt), P(it),
                                        _stream(dev.type))
    _lib.check(rc, "rlog_fit")
    return out.cpu().numpy(), icpt.cpu().numpy(), it.cpu().numpy()


def _check_fit(ref, n, m, seed, f64, use_nf, frozen, dev="cpu", bpv=0.8):
    K, sf, nf, disp = _fit_case(n, m, seed, f64)
    nfm = nf if use_nf else np.broadcast_to(sf, K.shape).copy()
    icpt = None
    if frozen:
        icpt = np.log2((K / nfm).mean(axis=1) + 0.5) + np.random.default_rng(seed).normal(0.0, 0.2, n)
        icpt[5 % n] = -np.inf                           # left out: 0
    if not f64:
        K = K.astype(np.int32)
    y = gm(K, dev)
    kw = dict(nf=gm(nfm, dev)) if use_nf else dict(sf=torch.as_tensor(sf, device=dev))
    itd = None if icpt is None else torch.as_tensor(icpt, device=dev)
    got, gicpt, git = _call_fit(y, m, torch.as_tensor(disp, device=dev), bpv, intercept=itd, ld_out=m + 3, **kw)
    assert np.all(got[:, m:] == -7.0)
    got = got[:, :m]
    fitted = (K.sum(axis=1) > 0) if icpt is None else np.isfinite(icpt)
    want, wicpt, wit = _ref_rlog_fit(ref, K[fitted].astype(np.float64), nfm[fitted], disp[fitted], bpv,
                                     None if icpt is None else icpt[fitted])
    assert np.array_equal(git[fitted], wit), (git[fitted], wit)
    assert _within(got[fitted], want), np.max(np.abs(got[fitted] - want))
    assert np.all(got[~fitted] == 0.0) and np.all(git[~fitted] == 0.0)
    if icpt is None:
        assert _within(gicpt[fitted], wicpt) and np.all(gicpt[~fitted] == -np.inf)
    else:
        assert np.all(gicpt == -7.0)                    # not written with a frozen intercept
    return git


@pytest.mark.parametrize("m", [2, 6, 12, 40])
@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("use_nf", [False, True])
@pytest.mark.parametrize("frozen", [False, True])
def test_fit_kernel_matches_reference(emu_dev, ref, m, f64, use_nf, frozen):
    """Equal iteration counts on every row and values within 1e-6 relative-or-absolute of the reference's fitBeta;
    y padded to ld = 4k, out written with ld_out = m + 3; an all-zero row (0, intercept -Inf, iter 0) and zero-heavy
    rows; with a frozen intercept a row with -Inf (0)."""
    _check_fit(ref, 24, m, 10 + m, f64, use_nf, frozen)


@pytest.mark.parametrize("m", [160, 400])
def test_fit_kernel_many_samples(emu_dev, ref, m):
    """A warp per gene (m > 160) and 16 lanes at its boundary, on a handful of genes."""
    _check_fit(ref, 6, m, 3, False, False, False)
    _check_fit(ref, 6, m, 4, True, True, True)


def test_fit_kernel_divergence(emu_dev, ref):
    """A row whose intercept passes 30 (counts ~ 2e13) and, frozen, a row whose sample coefficients must pass -30
    (intercept 50): iter = maxit and the diverged coefficients kept, as the reference does."""
    m = 6
    K, sf, nf, disp = _fit_case(8, m, 21, f64=True)
    K[4] = 2e13 * np.arange(1, m + 1)
    y = gm(K, "cpu")
    sfd = torch.as_tensor(sf)
    nfm = np.broadcast_to(sf, K.shape).copy()
    got, gicpt, git = _call_fit(y, m, torch.as_tensor(disp), 0.8, sf=sfd)
    fitted = K.sum(axis=1) > 0
    want, wicpt, wit = _ref_rlog_fit(ref, K[fitted], nfm[fitted], disp[fitted], 0.8)
    assert git[4] == 100 and np.array_equal(git[fitted], wit)
    assert _within(got[fitted], want) and abs(gicpt[4] * LN2) > 30
    K, sf, nf, disp = _fit_case(8, m, 22, f64=True)
    y = gm(K, "cpu")
    sfd = torch.as_tensor(sf)
    nfm = np.broadcast_to(sf, K.shape).copy()
    icpt = np.log2((K / nfm).mean(axis=1) + 0.5)
    icpt[2] = 50.0
    got, _, git = _call_fit(y, m, torch.as_tensor(disp), 1e6, sf=sfd, intercept=torch.as_tensor(icpt))
    want, _, wit = _ref_rlog_fit(ref, K, nfm, disp, 1e6, icpt)
    assert git[2] == 100 and np.array_equal(git, wit)
    assert _within(got, want) and np.max(np.abs(got[2] - 50.0) * LN2) > 30


# ---------------------------------------------------------------- the prior-variance kernel

def _prior_case(n, m, seed):
    rng = np.random.default_rng(seed)
    K = rng.negative_binomial(2, 0.01, (n, m))
    K[rng.random((n, m)) < 0.3] = 0
    K[:20, 0] = 0
    K[:20, 1:] = 5000                                   # zeros in highly expressed rows: |x| > 10
    K[30:60] = K[30]                                    # tied rows
    K[70] = 0                                           # an all-zero row: weight 0
    sf = np.exp(rng.normal(0.0, 0.3, m))
    disp = 0.05 + rng.uniform(0.0, 0.2, n)
    return K.astype(np.int32), sf, disp


def _host_prior(K, div, disp):
    from deseq2_b200 import pipeline
    bm = (K / pipeline._div(div)).mean(axis=1)
    nz = K.sum(axis=1) > 0
    x = np.log2(K[nz] / np.broadcast_to(pipeline._div(div), K.shape)[nz] + 0.5) - np.log2(bm[nz] + 0.5)[:, None]
    w = 1.0 / (1.0 / bm[nz] + disp[nz])
    return pipeline.matchWeightedUpperQuantileForVariance(x.ravel(order="F"), np.tile(w, K.shape[1])), bm, x


@pytest.mark.parametrize("use_nf", [False, True])
@pytest.mark.parametrize("m", [6, 100])
def test_prior_var_matches_host(emu_dev, use_nf, m):
    """Within 1e-12 relative of the host quantile; entries with |x| >= 10 and ties are present, the histogram grid has
    several CTAs, and two calls give the same bits."""
    from deseq2_b200 import device_pipeline as DP
    n = 2000
    K, sf, disp = _prior_case(n, m, m)
    div = sf[None, :] * np.exp(np.random.default_rng(1).normal(0.0, 0.2, (n, m))) if use_nf else sf
    want, bm, x = _host_prior(K, div, disp)
    assert np.any(np.abs(x) >= 10)
    y = gm(K, "cpu")
    sfd = gm(div, "cpu") if use_nf else torch.as_tensor(sf)
    bmd, dd = torch.as_tensor(bm), torch.as_tensor(disp)
    got = DP.rlog_prior_var(y, m, sfd, bmd, dd)
    assert abs(got.item() - want) <= 1e-12 * want
    assert torch.equal(got, DP.rlog_prior_var(y, m, sfd, bmd, dd))
    assert (n + 1023 // m - 1) // (1024 // m) > 1        # several histogram CTAs


def test_prior_var_nothing_kept(emu_dev):
    from deseq2_b200 import device_pipeline as DP
    y = gm(np.zeros((5, 3), dtype=np.int32), "cpu")
    v = DP.rlog_prior_var(y, 3, torch.ones(3, dtype=torch.float64), torch.zeros(5, dtype=torch.float64),
                          torch.ones(5, dtype=torch.float64))
    assert torch.isnan(v)


# ---------------------------------------------------------------- rlog_device against the host mirror

def _counts(n, m, seed, x=None):
    from deseq2_b200 import synth
    d = synth.make_example_counts(n, m, x=synth.design_condition(m) if x is None else x, seed=seed, betaSD=0.5)
    K = d["counts"].copy()
    K[[3, 17]] = 0
    return K, d["sizeFactors"]


def _compare(dv, host, frozen=False):
    n, m = host["rlog"].shape
    v = dv["rlog"].cpu().numpy()
    assert v.shape == (n, m) and dv["rlog"].is_contiguous()
    assert abs(dv["betaPriorVar"] - host["betaPriorVar"]) <= 1e-6 * host["betaPriorVar"]
    assert np.array_equal(dv["betaIter"].cpu().numpy(), host["betaIter"])
    assert np.max(np.abs(v - host["rlog"])) < 1e-6 * max(1.0, np.max(np.abs(host["rlog"])))
    if frozen:
        assert dv["intercept"] is None and host["intercept"] is None
    else:
        gi, hi = dv["intercept"].cpu().numpy(), host["intercept"]
        assert np.array_equal(np.isinf(gi), np.isinf(hi))
        assert np.max(np.abs(gi[np.isfinite(hi)] - hi[np.isfinite(hi)])) < 1e-6
    assert dv["n_nonfinite"] == 0


@pytest.mark.parametrize("blind", [True, False])
@pytest.mark.parametrize("fitType", ["parametric", "mean"])
def test_rlog_matches_host(emu_dev, oracle, blind, fitType):
    """Blind (~1) and blind=False with the design, parametric and mean trends, given size factors, all-zero rows."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_batch_condition(12, 3)
    K, sf = _counts(200, 12, 41, x)
    host = pipeline.rlog(K, x=x, blind=blind, fitType=fitType, sizeFactors=sf, engine=oracle)
    dv = DP.rlog_device(gm(K, "cpu"), 12, x=x, blind=blind, fitType=fitType, sizeFactors=sf)
    _compare(dv, host)
    assert dv["fitType"] == fitType and np.all(dv["rlog"].numpy()[[3, 17]] == 0.0)
    nz = K.sum(axis=1) > 0
    assert np.max(np.abs(dv["dispFit"].numpy()[nz] - host["dispFit"][nz])) < 1e-6 * np.max(host["dispFit"][nz])


def test_rlog_factors(emu_dev, oracle):
    """Estimated size factors, a gene-specific nf matrix, and the nf avgTxLength estimates."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, sf = _counts(200, 8, 43)
    y = gm(K, "cpu")
    dv = DP.rlog_device(y, 8)
    host = pipeline.rlog(K, engine=oracle)
    assert np.max(np.abs(dv["sizeFactors"] - host["sizeFactors"]) / host["sizeFactors"]) < 1e-12
    _compare(dv, host)
    nf = sf[None, :] * np.exp(np.random.default_rng(2).normal(0.0, 0.25, K.shape))
    dv = DP.rlog_device(y, 8, normalizationFactors=gm(nf, "cpu"))
    _compare(dv, pipeline.rlog(K, sizeFactors=nf, engine=oracle))
    tx = gm(np.exp(np.random.default_rng(3).normal(7.0, 0.5, K.shape)), "cpu")
    dv = DP.rlog_device(y, 8, avgTxLength=tx)
    nfe = DP.normalization_factors(y, 8, avgTxLength=tx)["normalizationFactors"]
    assert torch.equal(dv["normalizationFactors"], nfe)
    _compare(dv, pipeline.rlog(K, sizeFactors=nfe[:, :8].numpy(), engine=oracle))


def test_frozen_rlog(emu_dev, oracle):
    """The vignette's frozen rlog: intercept, betaPriorVar and dispFit of a first call applied to the same data and to
    a second dataset with another sample count (m = 5 and m = 1), against the host mirror; without betaPriorVar the
    prior is estimated on nf 2^intercept."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, sf = _counts(200, 10, 45)
    y = gm(K, "cpu")
    res = DP.rlog_device(y, 10, sizeFactors=sf)
    icpt, disp = res["intercept"], res["dispFit"]
    for K2, sf2 in ((K, sf), _counts(200, 5, 46), (K[:, :1], np.array([1.0]))):
        m2 = K2.shape[1]
        kw = dict(intercept=icpt, dispFit=disp, blind=False, sizeFactors=sf2)
        dv = DP.rlog_device(gm(K2, "cpu"), m2, betaPriorVar=res["betaPriorVar"], **kw)
        host = pipeline.rlog(K2, intercept=icpt.numpy(), betaPriorVar=res["betaPriorVar"], dispFit=disp.numpy(),
                             blind=False, sizeFactors=sf2, engine=oracle)
        _compare(dv, host, frozen=True)
        assert np.all(dv["rlog"].numpy()[[3, 17]] == 0.0)             # -Inf intercepts of the first call
    dv = DP.rlog_device(y, 10, **dict(kw, sizeFactors=sf))
    host = pipeline.rlog(K, intercept=icpt.numpy(), dispFit=disp.numpy(), blind=False, sizeFactors=sf, engine=oracle)
    _compare(dv, host, frozen=True)


def test_rlog_with_deseq_dispfit(emu_dev, oracle):
    """dispFit from DESeq_device's result (its non-zero rows), scattered to the N rows, with blind=False."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_condition(8)
    K, sf = _counts(200, 8, 47, x)
    y = gm(K, "cpu")
    ds = DP.DESeq_device(y, x, sizeFactors=sf)
    disp = torch.full((200,), float("nan"), dtype=torch.float64)
    disp[torch.as_tensor(ds["idx"])] = ds["dispFit"]
    dv = DP.rlog_device(y, 8, blind=False, dispFit=disp, sizeFactors=sf)
    host = pipeline.rlog(K, blind=False, dispFit=disp.numpy(), sizeFactors=sf, engine=oracle)
    _compare(dv, host)
    assert "fitType" not in dv


# ---------------------------------------------------------------- errors

def test_rlog_errors(emu_dev, oracle):
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, sf = _counts(100, 6, 49)
    y = gm(K, "cpu")
    with pytest.raises(ValueError, match="intercept should be as long"):
        DP.rlog_device(y, 6, intercept=np.zeros(99))
    with pytest.raises(ValueError, match="intercept should be as long"):
        pipeline.rlog(K, intercept=np.zeros(99), dispFit=np.ones(100), blind=False, engine=oracle)
    with pytest.raises(ValueError, match="dispFit should be as long"):
        DP.rlog_device(y, 6, blind=False, dispFit=np.ones(99))
    bad = np.full(100, 0.1)
    bad[5] = np.nan
    with pytest.raises(ValueError, match="dispFit"):
        DP.rlog_device(y, 6, blind=False, dispFit=bad)
    with pytest.raises(ValueError, match="dispFit"):
        pipeline.rlog(K, blind=False, dispFit=bad, engine=oracle)
    with pytest.raises(ValueError, match="blind=False"):
        DP.rlog_device(y, 6, blind=False)
    with pytest.raises(ValueError, match="blind=False"):
        pipeline.rlog(K, blind=False, engine=oracle)
    with pytest.raises(ValueError, match="local"):
        DP.rlog_device(y, 6, fitType="local")
    with pytest.raises(ValueError, match="one row per sample"):
        DP.rlog_device(y, 6, x=np.ones((5, 1)), blind=False)
    zero_heavy = np.zeros((300, 6), dtype=np.int64)
    zero_heavy[:, 0] = 1000
    zero_heavy[:, 1] = 1
    for f in (lambda: DP.rlog_device(gm(zero_heavy, "cpu"), 6, sizeFactors=np.ones(6), betaPriorVar=1.0,
                                     blind=False, dispFit=np.full(300, 0.1)),
              lambda: pipeline.rlog(zero_heavy, sizeFactors=np.ones(6), betaPriorVar=1.0, blind=False,
                                    dispFit=np.full(300, 0.1), engine=oracle)):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            f()
        assert any("negative binomial" in str(e.message) for e in w)


def test_rlog_abi_rejects_bad_arguments(emu_dev):
    from deseq2_b200 import _lib
    L = _lib.lib()
    y = gm(np.ones((5, 3)), "cpu")
    sf = torch.ones(3, dtype=torch.float64)
    nf = gm(np.ones((5, 3)), "cpu")
    disp = torch.full((5,), 0.1, dtype=torch.float64)
    icpt = torch.zeros(5, dtype=torch.float64)
    out = torch.empty((5, 3), dtype=torch.float64)
    oi, it, var = (torch.empty(5, dtype=torch.float64) for _ in range(3))
    P = lambda t: C.c_void_p(t.data_ptr())
    good = dict(y=P(y), sf=P(sf), nf=None, icpt=None, disp=P(disp), n=5, m=3, ld=4, bpv=0.5, tol=1e-4, maxit=100,
                minmu=0.5, out=P(out), ld_out=3, oi=P(oi), it=P(it))

    def fit(**kw):
        g = dict(good, **kw)
        return L.b200nb_rlog_fit_dev(g["y"], 1, g["sf"], g["nf"], g["icpt"], g["disp"], g["n"], g["m"], g["ld"],
                                     g["bpv"], g["tol"], g["maxit"], g["minmu"], g["out"], g["ld_out"], g["oi"],
                                     g["it"], None)

    assert fit() == 0 and fit(n=0) == 0
    assert fit(sf=None, nf=P(nf)) == 0 and fit(icpt=P(icpt), oi=None) == 0
    nan, inf = float("nan"), float("inf")
    for bad in (dict(n=-1), dict(m=0), dict(ld=2), dict(ld_out=2), dict(nf=P(nf)), dict(sf=None),
                dict(bpv=0.0), dict(bpv=-1.0), dict(bpv=nan), dict(bpv=inf), dict(tol=0.0), dict(tol=nan),
                dict(minmu=0.0), dict(minmu=inf), dict(maxit=0), dict(y=None), dict(disp=None), dict(out=None),
                dict(it=None), dict(oi=None)):
        assert fit(**bad) != 0, bad
        assert L.b200nb_last_error()
    bm = torch.ones(5, dtype=torch.float64)
    pv = dict(y=P(y), sf=P(sf), nf=None, bm=P(bm), disp=P(disp), n=5, m=3, ld=4, out=P(var))

    def prior(**kw):
        g = dict(pv, **kw)
        return L.b200nb_rlog_prior_var_dev(g["y"], 1, g["sf"], g["nf"], g["bm"], g["disp"], g["n"], g["m"], g["ld"],
                                           g["out"], None)

    assert prior() == 0 and prior(sf=None, nf=P(nf)) == 0
    for bad in (dict(n=0), dict(m=0), dict(ld=2), dict(nf=P(nf)), dict(sf=None), dict(y=None), dict(bm=None),
                dict(disp=None), dict(out=None)):
        assert prior(**bad) != 0, bad
        assert L.b200nb_last_error()


def test_fit_kernel_bad_dispersion_gives_nan(emu_dev):
    """A fitted row whose dispersion is not finite and > 0 gets NaN (the entry point does not read device data)."""
    y = gm(np.full((3, 4), 10, dtype=np.int32), "cpu")
    disp = torch.tensor([0.1, -1.0, float("nan")], dtype=torch.float64)
    out, icpt, it = _call_fit(y, 4, disp, 0.5, sf=torch.ones(4, dtype=torch.float64))
    assert np.all(np.isfinite(out[0])) and np.all(np.isnan(out[1:])) and np.all(np.isnan(it[1:]))


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("m", [3, 12, 31])
def test_fit_kernel_against_general_fit_beta_gpu(engine, m):
    """An independent implementation: the engine's general-p b200nb_fit_beta_dev (p = m + 1 <= 32) on the same
    [1 | I_m] design and start values: equal iteration counts and coefficients within 1e-6."""
    from deseq2_b200 import device as D
    n = 3000 if DEV == "cuda" else 60
    K, sf, _, disp = _fit_case(n, m, 7 + m)
    K = K.astype(np.int32)
    fitted = K.sum(axis=1) > 0
    K, disp = K[fitted], disp[fitted]
    n = K.shape[0]
    y = gm(K, DEV)
    sfd = torch.as_tensor(sf, device=DEV)
    dd = torch.as_tensor(disp, device=DEV)
    bpv = 0.7
    got, gicpt, git = _call_fit(y, m, dd, bpv, sf=sfd)
    x = np.c_[np.ones(m), np.eye(m)]
    beta0 = np.zeros((m + 1, n))
    beta0[0] = np.log((K / sf).mean(axis=1))
    lam = np.r_[1e-6, np.full(m, 1.0 / bpv)] / LN2 ** 2
    r = D.fit_beta(y, D.x_to_device(x, torch.device(DEV)), sfd, dd,
                   torch.as_tensor(np.r_[1.0, np.zeros(m)], device=DEV), torch.as_tensor(beta0, device=DEV),
                   torch.as_tensor(lam, device=DEV), 1e-4, 100, minmu=0.5, want_hat=False, want_mu=False)
    b = r["beta_mat"].cpu().numpy().T / LN2                  # (n, p)
    assert np.array_equal(git, r["iter"].cpu().numpy())
    assert _within(got, b @ x.T)
    assert _within(gicpt, b[:, 0])


def _config(config):
    """BASELINE C2 (50 000 x 100) and C4 (50 000 x 1000); on the emulator 400 x 20 and 400 x 56."""
    from deseq2_b200 import synth
    m = 100 if config == "C2" else 1000
    n = 50000
    if DEV != "cuda":
        n, m = 400, m // 25 + 16
    d = synth.make_example_counts(n, m, x=synth.design_condition(m), seed=13)
    K = d["counts"].copy()
    K[[3, 11]] = 0
    return K


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C2", "C4"])
def test_rlog_at_config_against_reference_gpu(engine, ref, config):
    """rlog_device at the C2 / C4 shapes; a random subset of its fitted rows refitted by the reference's own fitBeta
    with the same dispFit and betaPriorVar: equal iteration counts and values within 1e-6; the prior variance against
    the host quantile over all entries.  At C4 (m = 1000) one reference IRLS step of one gene is a QR of a 2001 x 1001
    matrix and a whole fit takes minutes, so there one gene is compared after maxit = 2 iterations of both fits."""
    from deseq2_b200 import device_pipeline as DP
    K = _config(config)
    n, m = K.shape
    y = gm(K, DEV)
    dv = DP.rlog_device(y, m)
    sf = dv["sizeFactors"]
    disp = dv["dispFit"].cpu().numpy()
    want, _, _ = _host_prior(K, sf, disp)
    assert abs(dv["betaPriorVar"] - want) <= 1e-12 * want
    assert dv["n_nonfinite"] == 0
    big = m > 500
    rows = np.random.default_rng(5).choice(np.flatnonzero(K.sum(axis=1) > 0), 1 if big else 64, replace=False)
    rows.sort()
    got = dv
    if big:
        got = DP.rlog_fit(y, m, torch.as_tensor(sf, device=DEV), dv["dispFit"], dv["betaPriorVar"], maxit=2)
    nfm = np.broadcast_to(sf, (len(rows), m)).copy()
    vals, icpt, it = _ref_rlog_fit(ref, K[rows].astype(np.float64), nfm, disp[rows], dv["betaPriorVar"],
                                   maxit=2 if big else 100)
    assert np.array_equal(got["betaIter"].cpu().numpy()[rows], it)
    assert _within(got["rlog"].cpu().numpy()[rows], vals)
    assert _within(got["intercept"].cpu().numpy()[rows], icpt)
