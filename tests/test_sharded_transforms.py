"""Size factors, normalization factors and the transforms on gene shards (deseq2_b200/sharded.py): on every rank the
result equals the single-device function run on the whole matrix, bit for bit, for the rows that rank owns, and every
value all ranks hold (size factors, trend coefficients, meanDisp, the vst subset) is the same on all of them.  The
CPU tests run the ranks over gloo with the emulated engine, the `-m gpu` tests over NCCL with one GPU per rank
(tests/ranks.py).  The shards are cut unequally on purpose, and the collective count of every call is asserted.

One exception to "bit for bit": with normalization factors the moments dispersion's xim sums nf columns per rank, so its
last bit can depend on where the shards split.  The nf cases that compare bit for bit use factors with few significant
bits (every partial sum exact); estimated nf, whose values are arbitrary, are compared bit for bit themselves and the
VST built on them to 1e-9."""
import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm  # noqa: F401
from ranks import DEVICE, nccl_world, run_ranks

SF_COLLECTIVES = 9                  # the agreement all-reduce and 8 histogram rounds


def _cuts(n, world):
    """Unequal shards: rank 0 gets a short block, the others split the rest."""
    if world == 1:
        return [0, n]
    first = max(1, n // (3 * world))
    rest = np.linspace(first, n, world).round().astype(int)
    return [0] + list(rest)


# ---------------------------------------------------------------- size factors

def _sf_counts(case, n, m):
    from deseq2_b200 import synth
    K = synth.make_example_counts(n, m, seed=61, betaSD=0.5)["counts"].copy()
    rng = np.random.default_rng(7)
    K[rng.random(K.shape) < min(0.05, 1.0 / m)] = 0           # genes with zeros
    src = n // 2 + int(np.argmax((K[n // 2:] > 0).all(axis=1)))
    for cut in (_cuts(n, 2)[1], _cuts(n, 3)[1]):
        K[cut - 3:cut + 3] = K[src]                            # tied ratios across the first cut
    if case in ("odd", "even"):
        pos = np.nonzero((K > 0).all(axis=1))[0]
        if (len(pos) % 2 == 1) != (case == "odd"):
            K[pos[-1], 0] = 0
    elif case == "nan_sample":
        K[:, 2] = 0                                            # no usable ratio in sample 2 (poscounts)
    elif case == "empty_shard":
        K[:_cuts(n, 2)[1] + 3, 1] = 0                          # no finite loggeomean on rank 0
    elif case == "all_zero":
        K[np.arange(n), np.arange(n) % m] = 0                  # every gene has a zero
    return K


SF_CASES = [("odd", "ratio", False), ("even", "ratio", True), ("odd", "poscounts", True),
            ("even", "poscounts", False), ("nan_sample", "poscounts", False), ("empty_shard", "ratio", False),
            ("all_zero", "ratio", False)]


def _sf_rank(rank, world, dev, n, m, cases):
    from deseq2_b200 import sharded
    cuts = _cuts(n, world)
    out = []
    for case, type_, f64 in cases:
        K = _sf_counts(case, n, m)[cuts[rank]:cuts[rank + 1]]
        y = gm(K, dev, np.float64 if f64 else None)
        try:
            out.append(sharded.sharded_size_factors_device(y, m, type=type_))
        except ValueError as e:
            out.append({"error": str(e)})
        if case == "nan_sample":
            # the medians before the poscounts rescaling, which turns every factor into NaN: where does the NaN go?
            r = sharded._local_ratios(y, m, True)
            nv, _, _, entries = sharded._agree(r)
            out[-1]["unscaled"] = sharded._sizes_of(sharded._global_median(entries, nv)[0], nv)
    return out


def _whole_sf(K, m, type_, f64, dev):
    from deseq2_b200 import device_pipeline as DP
    y = gm(K, dev, np.float64 if f64 else None)
    r = DP.size_factors(y, m, type=type_)
    sf = r["sizeFactors"]
    if type_ == "poscounts":
        sf = sf / torch.exp(torch.log(sf).mean())              # as DESeq_device rescales them
    return sf.cpu().numpy(), r["loggeomeans"].cpu().numpy()


def _check_sf(backend, n, m, world):
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sf_rank, n, m, SF_CASES, world=world, backend=backend)
    cuts = _cuts(n, world)
    assert world == 1 or len(set(np.diff(cuts))) > 1
    for i, (case, type_, f64) in enumerate(SF_CASES):
        K = _sf_counts(case, n, m)
        if case == "all_zero":
            with pytest.raises(ValueError, match="every gene contains at least one zero"):
                DP.size_factors(gm(K, DEVICE[backend]), m)
            assert all("every gene contains at least one zero" in g[i]["error"] for g in got)
            continue
        sf, lg = _whole_sf(K, m, type_, f64, DEVICE[backend])
        if case == "nan_sample":
            assert np.isnan(sf).all()
            whole = DP.size_factors(gm(K, DEVICE[backend]), m, type="poscounts")["sizeFactors"].cpu().numpy()
            assert np.isnan(whole[2]) and np.isfinite(np.delete(whole, 2)).all()
            for g in got:
                assert np.array_equal(g[i]["unscaled"], whole, equal_nan=True)
        else:
            assert np.isfinite(sf).all(), case
        for r, g in enumerate(got):
            r_i = g[i]
            assert np.array_equal(r_i["sizeFactors"], sf, equal_nan=True), (case, type_, r)
            assert np.array_equal(r_i["loggeomeans"], lg[cuts[r]:cuts[r + 1]]), (case, r)
            assert r_i["collectives"] == SF_COLLECTIVES
        if case == "empty_shard" and world > 1:
            assert np.isinf(got[0][i]["loggeomeans"]).all()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_size_factors_equal_whole(emu_dev, world):
    _check_sf("gloo", 301, 8, world)


def test_usable_ratio_parity(emu_dev):
    """The cases really have an odd and an even number of usable ratios per sample."""
    for case, want in (("odd", 1), ("even", 0)):
        K = _sf_counts(case, 301, 8)
        assert (K > 0).all(axis=1).sum() % 2 == want


# ---------------------------------------------------------------- normalization factors

def _nf_inputs(n, m):
    from deseq2_b200 import synth
    K = synth.make_example_counts(n, m, seed=63, betaSD=0.5)["counts"].copy()
    rng = np.random.default_rng(9)
    K[rng.random(K.shape) < 0.03] = 0
    nm = np.exp(rng.normal(0.0, 0.3, K.shape))
    tx = np.exp(rng.normal(7.0, 0.5, K.shape))
    return K, nm, tx


NF_CASES = [("normMatrix", "ratio"), ("avgTxLength", "ratio"), ("normMatrix", "poscounts")]


def _nf_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    cuts = _cuts(n, world)
    K, nm, tx = _nf_inputs(n, m)
    s = slice(cuts[rank], cuts[rank + 1])
    y = gm(K[s], dev)
    out = []
    for source, type_ in NF_CASES:
        kw = {"normMatrix_local": gm(nm[s], dev)} if source == "normMatrix" else {"avgTxLength_local": gm(tx[s], dev)}
        r = sharded.sharded_normalization_factors(y, m, type=type_, **kw)
        out.append({"nf": r["normalizationFactors"][:, :m], "sf": r["sizeFactors"], "collectives": r["collectives"]})
    bad = nm[s].copy()
    if rank == world - 1:
        bad[0, 0] = 0.0                                        # fails its check on the last rank only
    try:
        sharded.sharded_normalization_factors(y, m, normMatrix_local=gm(bad, dev))
        out.append("no error")
    except ValueError as e:
        out.append(str(e))
    return out


def _check_nf(backend, n, m, world):
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_nf_rank, n, m, world=world, backend=backend)
    cuts = _cuts(n, world)
    K, nm, tx = _nf_inputs(n, m)
    dev = DEVICE[backend]
    y = gm(K, dev)
    for i, (source, type_) in enumerate(NF_CASES):
        kw = {"normMatrix": gm(nm, dev)} if source == "normMatrix" else {"avgTxLength": gm(tx, dev)}
        w = DP.normalization_factors(y, m, type=type_, **kw)
        nf, sf = w["normalizationFactors"][:, :m].cpu().numpy(), w["sizeFactors"].cpu().numpy()
        for r, g in enumerate(got):
            assert np.array_equal(g[i]["sf"], sf), (source, type_, r)
            assert np.array_equal(g[i]["nf"], nf[cuts[r]:cuts[r + 1]]), (source, type_, r)
            assert g[i]["collectives"] == SF_COLLECTIVES
    assert "finite and positive" in got[-1][-1]
    assert all("other rank" in g[-1] for g in got[:-1])


def test_sharded_normalization_factors_equal_whole(emu_dev):
    _check_nf("gloo", 240, 8, 2)


# ---------------------------------------------------------------- the transforms

def _tie(n):
    """Half the length of each run of tied rows: long enough that the vst subset takes several of them."""
    return max(4, n // 100)


def _tf_inputs(n, m, seed=65):
    """Counts with all-zero rows, a run of tied rows across the first cut (equal baseMean), nf with 7 significant bits
    (every column sum exact) and a transcript-length matrix."""
    from deseq2_b200 import synth
    x = synth.design_batch_condition(m, 3)
    d = synth.make_example_counts(n, m, x=x, seed=seed, betaSD=0.4)
    K = d["counts"].copy()
    src = np.argsort(K.sum(axis=1))[3 * n // 4]
    for cut in (_cuts(n, 2)[1], _cuts(n, 3)[1]):
        K[cut - _tie(n):cut + _tie(n)] = K[src]
    K[[5, _cuts(n, 2)[1] + 9]] = 0
    rng = np.random.default_rng(seed)
    nf_exact = rng.integers(32, 129, K.shape) / 64.0
    tx = np.exp(rng.normal(7.0, 0.5, K.shape))
    return K, x, d["sizeFactors"], nf_exact, tx


def _tf_calls(y, m, x, sf, nfd, txd, nsub, sharded):
    """(name, call, whether the VST is compared bit for bit) for the single-device and the sharded functions alike:
    `sharded` picks the module functions."""
    from deseq2_b200 import device_pipeline as DP, sharded as S
    vt = S.sharded_varianceStabilizingTransformation_device if sharded else DP.varianceStabilizingTransformation_device
    vs = S.sharded_vst_device if sharded else DP.vst_device
    nt = S.sharded_normTransform_device if sharded else DP.normTransform_device
    return [
        ("vt_estimated", lambda: vt(y, m)),
        ("vt_mean_sf", lambda: vt(y, m, fitType="mean", sizeFactors=sf)),
        ("vt_design", lambda: vt(y, m, x=x, blind=False, sizeFactors=sf)),
        ("vt_design_mean", lambda: vt(y, m, x=x, blind=False, fitType="mean")),
        ("vt_nf", lambda: vt(y, m, normalizationFactors=nfd)),
        ("vt_avgtx", lambda: vt(y, m, avgTxLength=txd)),
        ("vt_frozen", lambda: vt(y, m, blind=False, sizeFactors=sf,
                                 dispersionFunction={"fitType": "parametric", "trendCoefs": [0.04, 1.5]})),
        ("vst_estimated", lambda: vs(y, m, nsub=nsub)),
        ("vst_mean_design", lambda: vs(y, m, x=x, blind=False, nsub=nsub, fitType="mean", sizeFactors=sf)),
        ("vst_nf", lambda: vs(y, m, nsub=nsub, normalizationFactors=nfd)),
        ("nt_estimated", lambda: nt(y, m)),
        ("nt_sf", lambda: nt(y, m, sizeFactors=sf, pc=0.5)),
        ("nt_nf", lambda: nt(y, m, normalizationFactors=nfd)),
    ]


TF_COLLECTIVES = {"vt_estimated": SF_COLLECTIVES + 2, "vt_mean_sf": 2, "vt_design": 2,
                  "vt_design_mean": SF_COLLECTIVES + 2, "vt_nf": 4, "vt_avgtx": SF_COLLECTIVES + 3, "vt_frozen": 0,
                  "vst_estimated": SF_COLLECTIVES + 3, "vst_mean_design": 3, "vst_nf": 5, "nt_estimated": SF_COLLECTIVES,
                  "nt_sf": 0, "nt_nf": 1}
KEPT = ("vst", "normTransform", "trendCoefs", "meanDisp", "sizeFactors", "subset", "fitType", "collectives")


def _tf_rank(rank, world, dev, n, m, nsub):
    from deseq2_b200 import sharded
    cuts = _cuts(n, world)
    K, x, sf, nf, tx = _tf_inputs(n, m)
    s = slice(cuts[rank], cuts[rank + 1])
    out = {}
    for name, call in _tf_calls(gm(K[s], dev), m, x, sf, gm(nf[s], dev), gm(tx[s], dev), nsub, True):
        r = call()
        out[name] = {k: v for k, v in r.items() if k in KEPT}
        if "normalizationFactors" in r:
            out[name]["nf"] = r["normalizationFactors"][:, :m]
    bad = nf[s].copy()
    if rank == world - 1:
        bad[0, 0] = -1.0                                       # fails its check on the last rank only
    try:
        sharded.sharded_varianceStabilizingTransformation_device(gm(K[s], dev), m, normalizationFactors=gm(bad, dev))
        out["bad_nf"] = "no error"
    except ValueError as e:
        out["bad_nf"] = str(e)
    for name, kw in (("too_few_rows", {"nsub": n + 1}), ("too_few_above_5", {"nsub": nsub})):
        yk = gm(K[s] if name == "too_few_rows" else np.minimum(K[s], 1), dev)
        try:
            sharded.sharded_vst_device(yk, m, sizeFactors=sf, **kw)
            out[name] = "no error"
        except ValueError as e:
            out[name] = str(e)
    return out


def _same(a, b):
    if isinstance(b, torch.Tensor):
        b = b.cpu().numpy()
    if isinstance(b, np.ndarray):
        return np.array_equal(np.asarray(a), b, equal_nan=True)
    return a == b


def _check_tf(backend, n, m, nsub, world):
    from deseq2_b200 import device_pipeline as DP  # noqa: F401
    got = run_ranks(_tf_rank, n, m, nsub, world=world, backend=backend)
    cuts = _cuts(n, world)
    K, x, sf, nf, tx = _tf_inputs(n, m)
    dev = DEVICE[backend]
    for name, call in _tf_calls(gm(K, dev), m, x, sf, gm(nf, dev), gm(tx, dev), nsub, False):
        w = call()
        if isinstance(w, torch.Tensor):
            w = {"normTransform": w}
        rows = w.get("vst", w.get("normTransform")).cpu().numpy()
        for r, g in enumerate(got):
            gr = g[name]
            assert gr["collectives"] == TF_COLLECTIVES[name], (name, gr["collectives"])
            mine = gr.get("vst", gr.get("normTransform"))
            if name == "vt_avgtx":
                # estimated nf: the factors are exact, xim over them may differ in the last bit
                assert np.array_equal(gr["nf"], w["normalizationFactors"][:, :m].cpu().numpy()[cuts[r]:cuts[r + 1]])
                assert np.max(np.abs(mine - rows[cuts[r]:cuts[r + 1]])) < 1e-9, name
                assert np.max(np.abs(gr["trendCoefs"] / w["trendCoefs"].cpu().numpy() - 1)) < 1e-9, name
                assert np.array_equal(gr["trendCoefs"], got[0][name]["trendCoefs"])
                continue
            assert np.array_equal(mine, rows[cuts[r]:cuts[r + 1]]), (name, r)
            for k in ("trendCoefs", "meanDisp", "sizeFactors", "subset", "fitType"):
                if k in w:
                    assert _same(gr[k], w[k]), (name, k, r)
        if name.startswith("vst"):
            sub = w["subset"].cpu().numpy()
            assert len(set(np.searchsorted(cuts[1:], sub, side="right"))) == world, name   # spans every rank
    # the tied rows straddle the first cut and sit next to each other in the fit order
    cut = _cuts(n, max(world, 2))[1]
    tied = np.arange(cut - _tie(n), cut + _tie(n))
    sub = got[0]["vst_estimated"]["subset"]
    pos = np.nonzero(np.isin(sub, tied))[0]
    assert len(pos) >= 2 and np.all(np.diff(pos) == 1) and np.all(np.diff(sub[pos]) > 0)
    if world > 1:
        assert sub[pos].min() < cut <= sub[pos].max()
    assert "finite and positive" in got[-1]["bad_nf"]
    assert all("other rank" in g["bad_nf"] for g in got[:-1])
    for g in got:
        assert g["too_few_rows"].startswith("less than 'nsub' rows,")
        assert "mean normalized count > 5" in g["too_few_above_5"]


def test_sharded_transforms_equal_whole(emu_dev):
    _check_tf("gloo", 300, 12, 120, 2)


def test_sharded_transforms_equal_whole_three_ranks(emu_dev):
    _check_tf("gloo", 300, 12, 120, 3)


# ---------------------------------------------------------------- size factors of all ranks into sharded_DESeq_device

def _deseq_data(n, m):
    from deseq2_b200 import synth
    x = synth.design_condition(m)
    return synth.make_example_counts(n, m, x=x, seed=67)["counts"], x


def _deseq_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    cuts = _cuts(n, world)
    K, x = _deseq_data(n, m)
    y = gm(K[cuts[rank]:cuts[rank + 1]], dev)
    sf = sharded.sharded_size_factors_device(y, m)["sizeFactors"]      # a device tensor, passed on as it is
    r = sharded.sharded_DESeq_device(y, x, sf)
    return {"sizeFactors": r["sizeFactors"], "trendCoefs": r["trendCoefs"], "gathered": r["gathered"],
            "collectives": r["collectives"]}


def _check_deseq(backend, n, m, world):
    """sharded_size_factors_device followed by sharded_DESeq_device equals DESeq_device on the whole matrix with the
    size factors of the whole matrix, bit for bit."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_deseq_rank, n, m, world=world, backend=backend)
    K, x = _deseq_data(n, m)
    y = gm(K, DEVICE[backend])
    whole = DP.DESeq_device(y, x, DP.size_factors(y, m)["sizeFactors"])
    assert np.array_equal(whole["sizeFactors"], DP.DESeq_device(y, x)["sizeFactors"])
    for g in got:
        assert np.array_equal(g["sizeFactors"], whole["sizeFactors"])
        assert np.array_equal(g["trendCoefs"], whole["trendCoefs"].cpu().numpy())
        assert g["collectives"] == 3
        for k in ("dispersion", "betaMatrix", "betaSE", "WaldPvalue"):
            assert np.array_equal(g["gathered"][k], whole[k].cpu().numpy(), equal_nan=True), k


def test_sharded_size_factors_into_sharded_deseq(emu_dev):
    _check_deseq("gloo", 400, 12, 2)


# ---------------------------------------------------------------- NCCL

@pytest.mark.gpu
def test_sharded_size_factors_over_nccl(engine):
    _check_sf("nccl", 20000, 100, nccl_world(3))


@pytest.mark.gpu
def test_sharded_normalization_factors_over_nccl(engine):
    _check_nf("nccl", 20000, 40, nccl_world())


@pytest.mark.gpu
def test_sharded_size_factors_into_sharded_deseq_over_nccl(engine):
    _check_deseq("nccl", 20000, 40, nccl_world(3))


@pytest.mark.gpu
def test_sharded_transforms_over_nccl(engine):
    _check_tf("nccl", 20000, 40, 1000, nccl_world(3))


@pytest.mark.gpu
def test_sharded_one_rank_over_nccl(engine):
    """One NCCL rank on one GPU, so that a one-GPU host checks the radix select, the exp and the gathers on the device
    against the single-device calls, bit for bit."""
    if DEV != "cuda" or torch.cuda.device_count() < 1:
        pytest.skip("needs a GPU")
    _check_sf("nccl", 20000, 100, 1)
    _check_nf("nccl", 20000, 40, 1)
    _check_tf("nccl", 20000, 40, 1000, 1)
    _check_deseq("nccl", 20000, 40, 1)
