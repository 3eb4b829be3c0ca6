"""vst(), varianceStabilizingTransformation() and normTransform() on the device: the transform kernel
(b200nb_transform_dev, csrc/transform.cuh) against numpy and against the closed-form property of a VST, vst()'s gene
subset (pipeline.vstSubsetPositions), the device functions against the host mirror (pipeline.vst /
varianceStabilizingTransformation / normTransform driving the oracle), the frozen VST, and the error cases.
The CPU tests run the engine's CUDA source on the SIMT emulator (`emu` fixture); the `-m gpu` tests run on a GPU, or on
the emulator when B200NB_LIB points at it."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, rel_err

LN2 = np.log(2.0)
MODES = {"parametric": (0, 0.05, 2.0), "mean": (1, 0.07, 0.0), "log2": (2, 1.0, 0.0)}


def _numpy_transform(K, div, mode, c0, c1):
    from deseq2_b200 import pipeline
    if mode == "parametric":
        return pipeline.getVarianceStabilizedData(K, div, {"fitType": "parametric", "trendCoefs": [c0, c1]})
    if mode == "mean":
        return pipeline.getVarianceStabilizedData(K, div, {"fitType": "mean", "meanDisp": c0})
    return pipeline.normTransform(K, div, pc=c0)


def _within(got, want, bound=1e-13):
    return np.all(np.abs(got - want) <= bound * np.maximum(1.0, np.abs(want)))


def _kernel_case(n, m, seed, f64):
    rng = np.random.default_rng(seed)
    K = rng.negative_binomial(2, 0.02, (n, m)).astype(np.float64)
    K[rng.random((n, m)) < 0.2] = 0.0
    K[0] = 0.0
    K[1 % n, 0] = 1e7
    if f64:
        K = K * rng.uniform(0.5, 1.5, (n, m))
    sf = np.exp(rng.normal(0.0, 0.4, m))
    nf = sf[None, :] * np.exp(rng.normal(0.0, 0.3, (n, m)))
    return (K if f64 else K.astype(np.int32)), sf, nf


def _call(y, m, mode, c0, c1, sf=None, nf=None, ld_out=None):
    """b200nb_transform_dev into an (n, ld_out) buffer prefilled with -7 (the padding must stay)."""
    from deseq2_b200 import _lib
    n, ld = y.shape
    ld_out = m if ld_out is None else ld_out
    out = torch.full((n, ld_out), -7.0, dtype=torch.float64, device=y.device)
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    rc = _lib.lib().b200nb_transform_dev(P(y), 1 if y.dtype == torch.float64 else 0, P(sf), P(nf), n, m, ld, mode,
                                         c0, c1, P(out), ld_out, None if y.device.type == "cpu" else
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "transform")
    return out.cpu().numpy()


def _check_kernel(n, m, mode, f64, use_nf, dev, seed=1, ld_out_pad=0):
    K, sf, nf = _kernel_case(n, m, seed, f64)
    code, c0, c1 = MODES[mode]
    y = gm(K, dev)
    if use_nf:
        got = _call(y, m, code, c0, c1, nf=gm(nf, dev), ld_out=m + ld_out_pad)
        want = _numpy_transform(K, nf, mode, c0, c1)
    else:
        got = _call(y, m, code, c0, c1, sf=torch.as_tensor(sf, device=dev), ld_out=m + ld_out_pad)
        want = _numpy_transform(K, sf, mode, c0, c1)
    assert _within(got[:, :m], want), np.max(np.abs(got[:, :m] - want))
    assert np.all(got[:, m:] == -7.0)


# ---------------------------------------------------------------- the transform kernel

@pytest.mark.parametrize("mode", ["parametric", "mean", "log2"])
@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("use_nf", [False, True])
@pytest.mark.parametrize("m", [1, 6, 100])
def test_transform_kernel_matches_numpy(emu_dev, mode, f64, use_nf, m):
    """Every entry within 1e-13 max(1, |v|) of numpy; zero counts and a 1e7 count; y's ld pads m = 1, 6 and out is
    written with ld_out = m + 3, whose padding stays untouched."""
    _check_kernel(37, m, mode, f64, use_nf, "cpu", seed=m, ld_out_pad=3)


def test_transform_many_rows_per_cta(emu_dev):
    """m = 1 packs 2048 rows into one CTA: 5000 rows leave a partial last CTA."""
    _check_kernel(5000, 1, "parametric", False, False, "cpu")


@pytest.mark.parametrize("mode", ["parametric", "mean"])
def test_vst_closed_form_property(emu_dev, mode):
    """For Var(q) = q + disp(q) q^2 with disp(q) = a0 + a1 / q (parametric) or alpha (mean), the derivative of the VST
    times sqrt(Var(q)) is the constant sqrt(a0) / ln 2 (sqrt(alpha) / ln 2): a central difference of the device
    output, independent of the formula's algebra.  For large q the VST tends to log2(q)."""
    code, c0, c1 = MODES[mode]
    q = np.exp(np.linspace(0.0, np.log(1e5), 40))
    h = 1e-4 * q
    pts = np.stack([q - h, q + h], axis=1).reshape(1, -1)
    out = _call(gm(pts, "cpu"), pts.shape[1], code, c0, c1, sf=torch.ones(pts.shape[1], dtype=torch.float64))[0]
    deriv = (out[1::2] - out[0::2]) / (2 * h)
    disp = c0 + c1 / q if mode == "parametric" else c0
    const = deriv * np.sqrt(q + disp * q ** 2)
    assert np.max(np.abs(const / (np.sqrt(c0) / LN2) - 1.0)) < 1e-6
    big = np.array([[1e9, 1e11, 1e13]])
    v = _call(gm(big, "cpu"), 3, code, c0, c1, sf=torch.ones(3, dtype=torch.float64))[0]
    assert np.all(np.abs(v - np.log2(big[0])) < 1e-6)
    assert abs(v[-1] - np.log2(1e13)) < 1e-10


def test_transform_abi_rejects_bad_arguments(emu_dev):
    from deseq2_b200 import _lib
    L = _lib.lib()
    y = gm(np.ones((5, 3)), "cpu")
    sf = torch.ones(3, dtype=torch.float64)
    nf = gm(np.ones((5, 3)), "cpu")
    out = torch.empty((5, 3), dtype=torch.float64)
    P = lambda t: C.c_void_p(t.data_ptr())
    good = dict(y=P(y), sf=P(sf), nf=None, n=5, m=3, ld=4, mode=0, c0=0.05, c1=2.0, out=P(out), ld_out=3)

    def call(**kw):
        g = dict(good, **kw)
        return L.b200nb_transform_dev(g["y"], 1, g["sf"], g["nf"], g["n"], g["m"], g["ld"], g["mode"], g["c0"], g["c1"],
                                      g["out"], g["ld_out"], None)

    assert call() == 0
    assert call(n=0) == 0 and call(m=0, ld_out=0) == 0
    assert call(sf=None, nf=P(nf)) == 0
    assert call(mode=1, c1=float("nan")) == 0 and call(mode=2, c0=0.0) == 0
    nan, inf = float("nan"), float("inf")
    for bad in (dict(n=-1), dict(m=-1), dict(ld=2), dict(ld_out=2), dict(nf=P(nf)), dict(sf=None),
                dict(c0=0.0), dict(c0=-1.0), dict(c0=nan), dict(c0=inf), dict(c1=0.0), dict(c1=nan), dict(c1=inf),
                dict(mode=1, c0=0.0), dict(mode=1, c0=nan), dict(mode=1, c0=inf),
                dict(mode=2, c0=-1e-9), dict(mode=2, c0=nan), dict(mode=2, c0=inf), dict(mode=3),
                dict(y=None), dict(out=None)):
        assert call(**bad) != 0, bad
        assert L.b200nb_last_error()


# ---------------------------------------------------------------- the gene subset of vst()

def test_subset_positions_by_hand():
    from deseq2_b200 import pipeline
    P = lambda L, k: list(pipeline.vstSubsetPositions(L, k) + 1)       # 1-based, as R prints them
    assert P(4, 3) == [1, 2, 4]                                        # 1, 2.5, 4: 2.5 -> 2
    assert P(6, 3) == [1, 4, 6]                                        # 1, 3.5, 6: 3.5 -> 4
    assert P(10, 4) == [1, 4, 7, 10]
    assert P(11, 5) == [1, 4, 6, 8, 11]                                # 1, 3.5, 6, 8.5, 11
    assert P(7, 7) == [1, 2, 3, 4, 5, 6, 7]                            # nsub = L
    assert P(9, 2) == [1, 9] and P(9, 1) == [1]
    for L, k in ((0, 1), (3, 4), (5, 0)):
        with pytest.raises(ValueError):
            pipeline.vstSubsetPositions(L, k)


def _vst_counts(n, m, seed, ties=True, zero_rows=(3, 17)):
    from deseq2_b200 import synth
    d = synth.make_example_counts(n, m, x=synth.design_condition(m), seed=seed, betaSD=0.5)
    K = d["counts"].copy()
    if ties:
        src = np.argsort(K.sum(axis=1))[n // 2:]                        # rows well above baseMean 5
        K[20:31] = K[src[0]]                                            # eleven rows with one baseMean
        K[50:53] = K[src[1]]
    K[list(zero_rows)] = 0
    return K, d["sizeFactors"]


def test_device_subset_equals_host(emu_dev, oracle):
    """Tied baseMeans keep their row order (a stable sort, as R's order()); the device subset is the host's, index for
    index, with estimated and with given size factors."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, sf = _vst_counts(300, 6, 5)
    for given in (None, sf):
        host = pipeline.vst(K, nsub=120, sizeFactors=given, engine=oracle)
        dv = DP.vst_device(gm(K, "cpu"), 6, nsub=120, sizeFactors=given)
        assert np.array_equal(dv["subset"].numpy(), host["subset"])
    tied = host["subset"][np.isin(host["subset"], np.arange(20, 31))]
    assert len(tied) >= 2 and np.all(np.diff(tied) > 0)


# ---------------------------------------------------------------- device against the host mirror

def _design(name):
    from deseq2_b200 import synth
    return {"condition12": lambda: synth.design_condition(12),
            "batch_condition36": lambda: synth.design_batch_condition(36, 3),
            "factor6_40": lambda: synth.design_factor(40, 6),
            "continuous40": lambda: np.c_[np.ones(40), np.linspace(-1.0, 1.0, 40)]}[name]()


def _nf_for(K, sf, seed):
    rng = np.random.default_rng(seed)
    return sf[None, :] * np.exp(rng.normal(0.0, 0.25, K.shape))


def _compare(dv, host, n_rows, fitType):
    assert dv["fitType"] == host["fitType"] == fitType
    if fitType == "mean":
        assert abs(dv["meanDisp"] - host["meanDisp"]) < 1e-6 * host["meanDisp"]
    else:
        assert np.max(rel_err(dv["trendCoefs"].cpu().numpy(), host["trendCoefs"])) < 1e-6
    v = dv["vst"].cpu().numpy()
    assert v.shape == (n_rows, host["vst"].shape[1]) and dv["vst"].is_contiguous()
    assert np.max(np.abs(v - host["vst"])) < 1e-6


@pytest.mark.parametrize("design", ["condition12", "batch_condition36", "factor6_40", "continuous40"])
@pytest.mark.parametrize("blind", [True, False])
@pytest.mark.parametrize("fitType", ["parametric", "mean"])
def test_vst_functions_match_host(emu_dev, oracle, design, blind, fitType):
    """vst (nsub = 150) and varianceStabilizingTransformation against the host mirror with the oracle, given size
    factors, two all-zero rows."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = _design(design)
    m = x.shape[0]
    d = synth.make_example_counts(240, m, x=x, seed=41, betaSD=0.3)
    K = d["counts"].copy()
    K[[5, 77]] = 0
    sf = d["sizeFactors"]
    y = gm(K, "cpu")
    host = pipeline.varianceStabilizingTransformation(K, x=x, blind=blind, fitType=fitType, sizeFactors=sf,
                                                      engine=oracle)
    dv = DP.varianceStabilizingTransformation_device(y, m, x=x, blind=blind, fitType=fitType, sizeFactors=sf)
    _compare(dv, host, 240, fitType)
    assert np.array_equal(dv["sizeFactors"], sf)
    host = pipeline.vst(K, x=x, blind=blind, nsub=150, fitType=fitType, sizeFactors=sf, engine=oracle)
    dv = DP.vst_device(y, m, x=x, blind=blind, nsub=150, fitType=fitType, sizeFactors=sf)
    assert np.array_equal(dv["subset"].numpy(), host["subset"])
    _compare(dv, host, 240, fitType)


@pytest.mark.parametrize("fitType", ["parametric", "mean"])
@pytest.mark.parametrize("blind", [True, False])
def test_vst_functions_match_host_nf(emu_dev, oracle, fitType, blind):
    """Gene-specific normalization factors: q = K / nf, and xim over the fitted rows (the subset's for vst)."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_batch_condition(12, 3)
    d = synth.make_example_counts(240, 12, x=x, seed=43, betaSD=0.3)
    K = d["counts"].copy()
    K[9] = 0
    nf = _nf_for(K, d["sizeFactors"], 2)
    y, nfd = gm(K, "cpu"), gm(nf, "cpu")
    host = pipeline.varianceStabilizingTransformation(K, x=x, blind=blind, fitType=fitType, sizeFactors=nf,
                                                      engine=oracle)
    dv = DP.varianceStabilizingTransformation_device(y, 12, x=x, blind=blind, fitType=fitType,
                                                     normalizationFactors=nfd)
    _compare(dv, host, 240, fitType)
    assert "sizeFactors" not in dv and dv["normalizationFactors"] is nfd
    host = pipeline.vst(K, x=x, blind=blind, nsub=120, fitType=fitType, sizeFactors=nf, engine=oracle)
    dv = DP.vst_device(y, 12, x=x, blind=blind, nsub=120, fitType=fitType, normalizationFactors=nfd)
    assert np.array_equal(dv["subset"].numpy(), host["subset"])
    _compare(dv, host, 240, fitType)


def test_estimated_factors_and_avg_tx_length(emu_dev, oracle):
    """No factors given: the median-of-ratios size factors; avgTxLength: the nf DESeq_device estimates."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, _ = _vst_counts(300, 8, 7, ties=False)
    y = gm(K, "cpu")
    dv = DP.varianceStabilizingTransformation_device(y, 8)
    host = pipeline.varianceStabilizingTransformation(K, engine=oracle)
    assert np.max(rel_err(dv["sizeFactors"], host["sizeFactors"])) < 1e-12
    _compare(dv, host, 300, "parametric")
    tx = np.exp(np.random.default_rng(3).normal(7.0, 0.5, K.shape))
    txd = gm(tx, "cpu")
    nf = DP.normalization_factors(y, 8, avgTxLength=txd)["normalizationFactors"]
    dv = DP.vst_device(y, 8, nsub=120, avgTxLength=txd)
    assert torch.equal(dv["normalizationFactors"], nf)
    host = pipeline.vst(K, nsub=120, sizeFactors=nf[:, :8].numpy(), engine=oracle)
    assert np.array_equal(dv["subset"].numpy(), host["subset"])
    _compare(dv, host, 300, "parametric")


@pytest.mark.parametrize("use_nf", [False, True])
def test_norm_transform_matches_host(emu_dev, use_nf):
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, sf = _vst_counts(200, 7, 9, ties=False)
    y = gm(K, "cpu")
    if use_nf:
        nf = _nf_for(K, sf, 4)
        got = DP.normTransform_device(y, 7, normalizationFactors=gm(nf, "cpu"), pc=0.5).numpy()
        want = pipeline.normTransform(K, nf, pc=0.5)
    else:
        got = DP.normTransform_device(y, 7).numpy()
        want = pipeline.normTransform(K)
    assert np.max(np.abs(got - want)) < 1e-13 * max(1.0, np.max(np.abs(want)))


# ---------------------------------------------------------------- frozen VST

@pytest.mark.parametrize("fitType", ["parametric", "mean"])
def test_frozen_vst(emu_dev, oracle, fitType):
    """vst_transform with DESeq_device's dispersion function is the transform with those coefficients, bit for bit;
    applied to a second dataset with another sample count it matches the host mirror."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_condition(12)
    d = synth.make_example_counts(240, 12, x=x, seed=45, betaSD=0.3)
    y = gm(d["counts"], "cpu")
    res = DP.DESeq_device(y, x, sizeFactors=d["sizeFactors"], fitType=fitType)
    got = DP.vst_transform(y, 12, res, sizeFactors=res["sizeFactors"])
    if fitType == "parametric":
        a0, a1 = (float(v) for v in res["trendCoefs"])
        want = DP.transform(y, 12, "parametric", a0, a1, torch.as_tensor(res["sizeFactors"]))
    else:
        want = DP.transform(y, 12, "mean", res["meanDisp"], 0.0, torch.as_tensor(res["sizeFactors"]))
    assert torch.equal(got, want)
    d2 = synth.make_example_counts(150, 5, x=synth.design_condition(5), seed=46)
    K2 = d2["counts"].copy()
    K2[4] = 0
    y2 = gm(K2, "cpu")
    fn = {k: res[k] for k in ("fitType", "trendCoefs", "meanDisp") if k in res}
    frozen = DP.varianceStabilizingTransformation_device(y2, 5, blind=False, dispersionFunction=fn)
    host_fn = {k: (v.numpy() if isinstance(v, torch.Tensor) else v) for k, v in fn.items()}
    host = pipeline.varianceStabilizingTransformation(K2, blind=False, dispersionFunction=host_fn)
    assert np.max(np.abs(frozen["vst"].numpy() - host["vst"])) < 1e-13 * np.max(np.abs(host["vst"]))
    assert torch.equal(frozen["vst"], DP.vst_transform(y2, 5, fn, sizeFactors=frozen["sizeFactors"]))


# ---------------------------------------------------------------- errors

def test_vst_errors(emu_dev, oracle):
    from deseq2_b200 import _lib, device_pipeline as DP, pipeline
    K, sf = _vst_counts(300, 6, 11, ties=False)
    y = gm(K, "cpu")
    with pytest.raises(ValueError, match="less than 'nsub' rows,"):
        DP.vst_device(y, 6, nsub=301)
    with pytest.raises(ValueError, match="less than 'nsub' rows,"):
        pipeline.vst(K, nsub=301, engine=oracle)
    low = np.minimum(K, 3)
    with pytest.raises(ValueError, match="mean normalized count > 5"):
        DP.vst_device(gm(low, "cpu"), 6, nsub=100)
    with pytest.raises(ValueError, match="mean normalized count > 5"):
        pipeline.vst(low, nsub=100, engine=oracle)
    for f in (lambda: DP.vst_device(y, 6, nsub=100, fitType="local"),
              lambda: DP.varianceStabilizingTransformation_device(y, 6, fitType="local"),
              lambda: DP.vst_transform(y, 6, {"fitType": "local"}, sizeFactors=sf),
              lambda: pipeline.getVarianceStabilizedData(K, sf, {"fitType": "local"})):
        with pytest.raises(ValueError, match="local"):
            f()
    with pytest.raises(ValueError, match="blind=False"):
        DP.varianceStabilizingTransformation_device(y, 6, blind=False)
    with pytest.raises(ValueError, match="blind=False"):
        DP.vst_device(y, 6, blind=False, nsub=100)
    with pytest.raises(ValueError, match="blind=False"):
        pipeline.varianceStabilizingTransformation(K, blind=False, engine=oracle)
    with pytest.raises(ValueError, match="one row per sample"):
        DP.varianceStabilizingTransformation_device(y, 6, x=np.ones((5, 1)), blind=False)
    bad = np.ones(K.shape)
    bad[2, 1] = 0.0
    with pytest.raises(ValueError, match="normalizationFactors"):
        DP.varianceStabilizingTransformation_device(y, 6, normalizationFactors=gm(bad, "cpu"))
    with pytest.raises(ValueError, match="normalizationFactors"):
        DP.normTransform_device(y, 6, normalizationFactors=torch.ones((300, 6), dtype=torch.float64))
    with pytest.raises(ValueError, match="not both"):
        DP.vst_transform(y, 6, {"fitType": "mean", "meanDisp": 0.1}, sizeFactors=sf,
                         normalizationFactors=gm(np.ones(K.shape), "cpu"))
    with pytest.raises(ValueError, match="sizeFactors or normalizationFactors"):
        DP.vst_transform(y, 6, {"fitType": "mean", "meanDisp": 0.1})
    with pytest.raises(_lib.EngineError, match="pc"):
        DP.normTransform_device(y, 6, sizeFactors=sf, pc=-1.0)


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

def _config(config):
    """BASELINE C2 (50 000 x 100) and C4 (50 000 x 1000); on the emulator 1000 x 20 and 1000 x 40."""
    from deseq2_b200 import synth
    m = 100 if config == "C2" else 1000
    n = 50000
    if DEV != "cuda":
        n, m = 1000, m // 25 + 16
    d = synth.make_example_counts(n, m, x=synth.design_condition(m), seed=13)
    K = d["counts"].copy()
    K[[3, 11]] = 0
    return K, d["sizeFactors"]


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C2", "C4"])
def test_transform_kernel_at_config_gpu(engine, config):
    K, sf = _config(config)
    n, m = K.shape
    y = gm(K, DEV)
    sfd = torch.as_tensor(sf, device=DEV)
    for mode, (code, c0, c1) in MODES.items():
        got = _call(y, m, code, c0, c1, sf=sfd)
        assert _within(got, _numpy_transform(K, sf, mode, c0, c1)), mode


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C2", "C4"])
def test_vst_end_to_end_at_config_gpu(engine, oracle, config):
    """vst (nsub = 1000) and the blind varianceStabilizingTransformation against the host mirror driving the oracle."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    K, _ = _config(config)
    n, m = K.shape
    y = gm(K, DEV)
    nsub = 1000 if DEV == "cuda" else 200
    dv = DP.vst_device(y, m, nsub=nsub)
    host = pipeline.vst(K, nsub=nsub, engine=oracle)
    assert np.array_equal(dv["subset"].cpu().numpy(), host["subset"])
    _compare(dv, host, n, "parametric")
    dv = DP.varianceStabilizingTransformation_device(y, m)
    host = pipeline.varianceStabilizingTransformation(K, engine=oracle)
    _compare(dv, host, n, "parametric")
    assert np.max(np.abs(DP.normTransform_device(y, m).cpu().numpy() - pipeline.normTransform(K))) < 1e-12
