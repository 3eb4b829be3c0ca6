"""Size factors and normalization factors from control genes and given geometric means (estimateSizeFactorsForMatrix's
`controlGenes` and `geoMeans`, R/core.R:535-578; estimateNormFactors, :2159-2163): the host mirror against a
column-by-column restatement of the R function, the device functions against the host mirror, the gene-sharded
functions against the single-device ones bit for bit, a spike-in experiment end to end, and the frozen-normalization
round trip.  The CPU tests run the engine on the SIMT emulator (emu_dev) and the ranks over gloo; the `-m gpu` tests
run on the H100 and the ranks over NCCL."""
import math

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, rel_err  # noqa: F401
from ranks import DEVICE, nccl_world, run_ranks

SF_COLLECTIVES = 9


# ---------------------------------------------------------------- an independent restatement of R/core.R:535-578

def _r_median(v):
    v = sorted(v)
    if not v:
        return math.nan
    h = len(v) // 2
    return v[h] if len(v) % 2 else (v[h - 1] + v[h]) / 2


def _r_log(g):
    return math.log(g) if g > 0 else (-math.inf if g == 0 else math.nan)


def _restated(counts, geoMeans=None, controlGenes=None, poscounts=False, normMatrix=None):
    """estimateSizeFactorsForMatrix (estimateNormFactors' size factors with normMatrix) one sample at a time, in plain
    Python: loggeomeans, the stop on all rows, the median over the control rows, the incoming-geoMeans rescaling."""
    K = np.asarray(counts, dtype=np.float64)
    n, m = K.shape
    cn = K if normMatrix is None else K / np.asarray(normMatrix)
    if geoMeans is not None:
        lg = [_r_log(float(g)) for g in geoMeans]
    elif poscounts:
        lg = [_r_log(math.exp(sum(math.log(c) for c in row if c > 0) / m)) if (row > 0).any() else -math.inf
              for row in K]
    else:
        lg = [sum(_r_log(c) for c in row) / m for row in cn]
    if all(math.isinf(v) for v in lg):
        raise ValueError("every gene contains at least one zero")
    if controlGenes is None:
        rows = list(range(n))
    elif np.asarray(controlGenes).dtype == bool:
        rows = [i for i in range(n) if controlGenes[i]]
    else:
        rows = [int(i) for i in controlGenes]
    sf = [math.exp(_r_median([math.log(cn[i, j]) - lg[i] for i in rows if math.isfinite(lg[i]) and cn[i, j] > 0]))
          for j in range(m)]
    sf = np.array(sf)
    if geoMeans is not None or poscounts:
        sf = sf / math.exp(sum(math.log(s) for s in sf) / m)
    return sf


def _base_counts(n=40, m=6, seed=3):
    rng = np.random.default_rng(seed)
    K = rng.negative_binomial(4, 4 / (4 + rng.gamma(2.0, 40.0, (n, 1)) * rng.uniform(0.5, 2.0, (1, m))))
    K[rng.random(K.shape) < 0.06] = 0
    return K.astype(np.int32)


def _host_cases():
    K = _base_counts()
    n, m = K.shape
    full = np.flatnonzero((K > 0).all(axis=1))
    rng = np.random.default_rng(5)
    gmeans = np.exp(rng.normal(3.5, 1.0, n))
    bad = gmeans.copy()
    bad[[0, 3]] = 0.0
    bad[[1, 7]] = -2.0
    bad[9] = np.nan
    zero_ctl = np.flatnonzero(~(K > 0).all(axis=1))[:5]
    return K, [
        ("duplicated", dict(controlGenes=np.r_[full[:3], full[:3], full[5]])),
        ("geo_bad_values", dict(geoMeans=bad)),
        ("geo_and_control", dict(geoMeans=bad, controlGenes=np.r_[np.arange(12), 0, 1, 9])),
        ("zero_controls", dict(controlGenes=zero_ctl)),
        ("all_negative_geo", dict(geoMeans=-gmeans)),
        ("empty_control", dict(controlGenes=np.zeros(0, dtype=np.int64))),
        ("even_usable", dict(controlGenes=full[:4])),
        ("odd_usable", dict(controlGenes=full[:5])),
        ("mask", dict(controlGenes=np.isin(np.arange(n), full[::2]))),
        ("poscounts_control", dict(controlGenes=zero_ctl, poscounts=True)),
    ]


@pytest.mark.parametrize("case", [c for c, _ in _host_cases()[1]])
def test_host_mirror_matches_restatement(case):
    from deseq2_b200 import pipeline
    K, cases = _host_cases()
    kw = dict(cases)[case]
    want = _restated(K, **kw)
    type_ = "poscounts" if kw.get("poscounts") else "ratio"
    got = pipeline.estimateSizeFactorsForMatrix(K, type=type_, geoMeans=kw.get("geoMeans"),
                                                controlGenes=kw.get("controlGenes"))
    assert np.array_equal(np.isnan(got), np.isnan(want)), case
    ok = ~np.isnan(want)
    assert np.max(rel_err(got[ok], want[ok]), initial=0.0) < 1e-14, case
    if case in ("zero_controls", "all_negative_geo", "empty_control"):
        assert np.isnan(got).all(), case
    else:
        assert np.isfinite(got).all(), case
    nm = np.exp(np.random.default_rng(11).normal(0.0, 0.3, K.shape))
    want_nf_sf = _restated(K, normMatrix=nm, **kw)
    nf = pipeline.estimateNormFactors(K, nm, type=type_, geoMeans=kw.get("geoMeans"),
                                      controlGenes=kw.get("controlGenes"))
    ref = nm * want_nf_sf[None, :]
    ref = ref / np.exp(np.log(ref).mean(axis=1))[:, None]
    assert np.array_equal(np.isnan(nf), np.isnan(ref)), case
    assert np.nanmax(rel_err(nf, ref), initial=0.0) < 1e-13, case


def test_host_mirror_usable_ratio_parity():
    """The even / odd cases really take an even and an odd number of ratios in every sample."""
    K, cases = _host_cases()
    c = dict(cases)
    assert (K[c["even_usable"]["controlGenes"]] > 0).all() and len(c["even_usable"]["controlGenes"]) == 4
    assert (K[c["odd_usable"]["controlGenes"]] > 0).all() and len(c["odd_usable"]["controlGenes"]) == 5


def test_host_mirror_stops_and_refusals():
    from deseq2_b200 import pipeline
    K = _base_counts()
    n = K.shape[0]
    Z = K.copy()
    Z[np.arange(n), np.arange(n) % K.shape[1]] = 0
    with pytest.raises(ValueError, match="every gene contains at least one zero"):
        pipeline.estimateSizeFactorsForMatrix(Z, controlGenes=np.arange(5))
    with pytest.raises(ValueError, match="every gene contains at least one zero"):
        pipeline.estimateSizeFactorsForMatrix(K, geoMeans=np.zeros(n))
    with pytest.raises(ValueError, match="geoMeans should be as long as the number of rows"):
        pipeline.estimateSizeFactorsForMatrix(K, geoMeans=np.ones(n - 1))
    with pytest.raises(ValueError, match="poscounts"):
        pipeline.estimateSizeFactorsForMatrix(K, type="poscounts", geoMeans=np.ones(n))
    with pytest.raises(ValueError, match="poscounts"):
        pipeline.estimateNormFactors(K, np.ones(K.shape), type="poscounts", geoMeans=np.ones(n))
    for bad in (np.ones(n - 1, dtype=bool), np.array([0, -1]), np.array([n]), np.array([0.0, 1.0]),
                np.ones((2, 2), dtype=int)):
        with pytest.raises(ValueError, match="controlGenes"):
            pipeline.estimateSizeFactorsForMatrix(K, controlGenes=bad)


def test_host_mirror_every_row_is_the_plain_call():
    from deseq2_b200 import pipeline
    K = _base_counts()
    n = K.shape[0]
    for type_ in ("ratio", "poscounts"):
        plain = pipeline.estimateSizeFactorsForMatrix(K, type=type_)
        for ctl in (np.ones(n, dtype=bool), np.arange(n)):
            assert np.array_equal(pipeline.estimateSizeFactorsForMatrix(K, type=type_, controlGenes=ctl), plain)


# ---------------------------------------------------------------- device against the host mirror

def _device_counts(n, m, seed):
    from deseq2_b200 import synth
    K = synth.make_example_counts(n, m, seed=seed, betaSD=0.5, interceptMean=5.0)["counts"].copy()
    rng = np.random.default_rng(seed)
    K[rng.random(K.shape) < 0.02] = 0
    K[::17] = 0                                                  # all-zero rows
    return K


def _control_forms(n, seed):
    """(name, controlGenes) pairs: a 10 % mask, 92 (or n // 4) indices with duplicates, and every row both ways."""
    rng = np.random.default_rng(seed)
    k = min(92, n // 4)
    idx = rng.choice(n, k, replace=False)
    return [("mask", rng.random(n) < 0.1), ("index", np.r_[idx, idx[:3]]),
            ("all_mask", np.ones(n, dtype=bool)), ("all_index", np.arange(n))]


def _check_device(dev, n, m, seed):
    from deseq2_b200 import device_pipeline as DP, pipeline
    K = _device_counts(n, m, seed)
    rng = np.random.default_rng(seed + 1)
    nm = np.exp(rng.normal(0.0, 0.3, K.shape))
    tx = np.exp(rng.normal(7.0, 0.5, K.shape))
    geo = np.exp(rng.normal(4.5, 1.0, n))
    geo[:5] = 0.0
    geo[5:8] = -1.0
    for f64 in (False, True):
        y = gm(K, dev, np.float64 if f64 else None)
        for type_ in ("ratio", "poscounts"):
            plain = DP.size_factors(y, m, type=type_)
            for name, ctl in _control_forms(n, seed):
                got = DP.size_factors(y, m, type=type_, controlGenes=ctl)
                rows = pipeline.controlGeneRows(ctl, n)
                sub = DP.size_factors(y[torch.as_tensor(rows, device=y.device)].contiguous(), m, type=type_)
                assert torch.equal(got["sizeFactors"], sub["sizeFactors"]), (name, type_, f64)
                assert torch.equal(got["loggeomeans"], plain["loggeomeans"]), (name, type_, f64)
                if name.startswith("all"):
                    assert torch.equal(got["sizeFactors"], plain["sizeFactors"]), (name, type_, f64)
                host = pipeline.estimateSizeFactorsForMatrix(K, type=type_, controlGenes=ctl)
                sf = got["sizeFactors"]
                if type_ == "poscounts":
                    sf = sf / torch.exp(torch.log(sf).mean())            # the host mirror rescales poscounts
                assert np.max(rel_err(sf.cpu().numpy(), host)) < 1e-12, (name, type_, f64)
                # a device tensor of indices or a mask is taken as well
                t = DP.size_factors(y, m, type=type_, controlGenes=torch.as_tensor(ctl, device=y.device))
                assert torch.equal(t["sizeFactors"], got["sizeFactors"])
        for name, ctl in [("none", None)] + _control_forms(n, seed)[:2]:
            for g in (geo, torch.as_tensor(geo, device=y.device)):
                got = DP.size_factors(y, m, controlGenes=ctl, geoMeans=g)["sizeFactors"].cpu().numpy()
                host = pipeline.estimateSizeFactorsForMatrix(K, controlGenes=ctl, geoMeans=geo)
                assert np.max(rel_err(got, host)) < 1e-13, (name, f64)
        # normalization factors, both sources
        for src in ("normMatrix", "avgTxLength"):
            mat = nm if src == "normMatrix" else tx
            hm = mat if src == "normMatrix" else tx / np.exp(np.log(tx).mean(axis=1))[:, None]
            for type_, ctl, g in (("ratio", _control_forms(n, seed)[0][1], None),
                                  ("poscounts", _control_forms(n, seed)[1][1], None),
                                  ("ratio", None, geo), ("ratio", _control_forms(n, seed)[1][1], geo)):
                w = DP.normalization_factors(y, m, type=type_, controlGenes=ctl, geoMeans=g, **{src: gm(mat, dev)})
                host = pipeline.estimateNormFactors(K, hm, type=type_, controlGenes=ctl, geoMeans=g)
                nf = w["normalizationFactors"][:, :m].cpu().numpy()
                assert np.max(rel_err(nf, host)) < 1e-12, (src, type_, ctl is None, g is None)
                assert np.all(w["normalizationFactors"][:, m:].cpu().numpy() == 1.0)
                if g is None:
                    rows = torch.as_tensor(pipeline.controlGeneRows(ctl, n), device=y.device)
                    sub = DP.normalization_factors(y[rows].contiguous(), m, type=type_,
                                                   **{src: gm(mat, dev)[rows].contiguous()})
                    assert torch.equal(w["sizeFactors"], sub["sizeFactors"]), (src, type_)
            for type_ in ("ratio", "poscounts"):
                plain = DP.normalization_factors(y, m, type=type_, **{src: gm(mat, dev)})
                for _, ctl in _control_forms(n, seed)[2:]:
                    w = DP.normalization_factors(y, m, type=type_, controlGenes=ctl, **{src: gm(mat, dev)})
                    assert torch.equal(w["sizeFactors"], plain["sizeFactors"]), (src, type_)
                    assert torch.equal(w["normalizationFactors"], plain["normalizationFactors"]), (src, type_)


def test_device_matches_host_mirror(emu_dev):
    _check_device("cpu", 300, 7, 21)


def _check_device_edges(dev):
    from deseq2_b200 import device_pipeline as DP
    K = _base_counts()
    n, m = K.shape
    y = gm(K, dev)
    zero_ctl = np.flatnonzero(~(K > 0).all(axis=1))[:5]
    assert np.isnan(DP.size_factors(y, m, controlGenes=zero_ctl)["sizeFactors"].cpu().numpy()).all()
    assert np.isnan(DP.size_factors(y, m, controlGenes=[])["sizeFactors"].cpu().numpy()).all()
    assert np.isnan(DP.size_factors(y, m, geoMeans=-np.ones(n))["sizeFactors"].cpu().numpy()).all()
    ctl_empty = DP.normalization_factors(y, m, normMatrix=gm(np.ones(K.shape), dev), controlGenes=np.zeros(n, bool))
    assert np.isnan(ctl_empty["sizeFactors"].cpu().numpy()).all()
    Z = K.copy()
    Z[np.arange(n), np.arange(n) % m] = 0
    with pytest.raises(ValueError, match="every gene contains at least one zero"):
        DP.size_factors(gm(Z, dev), m, controlGenes=np.arange(4))
    with pytest.raises(ValueError, match="every gene contains at least one zero"):
        DP.size_factors(y, m, geoMeans=np.r_[np.zeros(n - 1), np.inf])
    with pytest.raises(ValueError, match="geoMeans should be as long"):
        DP.size_factors(y, m, geoMeans=np.ones(n + 1))
    with pytest.raises(ValueError, match="poscounts"):
        DP.size_factors(y, m, type="poscounts", geoMeans=np.ones(n))
    with pytest.raises(ValueError, match="poscounts"):
        DP.normalization_factors(y, m, normMatrix=gm(np.ones(K.shape), dev), type="poscounts", geoMeans=np.ones(n))
    for bad in (np.ones(n - 1, dtype=bool), [0, -1], [n], [0.5]):
        with pytest.raises(ValueError, match="controlGenes"):
            DP.size_factors(y, m, controlGenes=bad)


def test_device_edges(emu_dev):
    _check_device_edges("cpu")


def _check_frozen_round_trip(dev, n, m, seed):
    """geoMeans from a reference's own loggeomeans put the reference's counts back on its scale: its factors rescaled
    to geometric mean 1."""
    from deseq2_b200 import device_pipeline as DP
    y = gm(_device_counts(n, m, seed), dev)
    ref = DP.size_factors(y, m)
    want = ref["sizeFactors"] / torch.exp(torch.log(ref["sizeFactors"]).mean())
    got = DP.size_factors(y, m, geoMeans=torch.exp(ref["loggeomeans"]))
    assert np.max(rel_err(got["sizeFactors"].cpu().numpy(), want.cpu().numpy())) < 1e-13
    assert torch.equal(torch.isinf(got["loggeomeans"]), torch.isinf(ref["loggeomeans"]))


def test_frozen_round_trip(emu_dev):
    _check_frozen_round_trip("cpu", 300, 7, 23)


# ---------------------------------------------------------------- gene shards

def _shard_cuts(n, world):
    """Rank 0 of a multi-rank world gets no row at all with 3 ranks, and no control row with 2."""
    if world == 1:
        return [0, n]
    if world == 2:
        return [0, n // 5, n]
    return [0, 0, n // 2, n]


def _shard_inputs(n, m):
    rng = np.random.default_rng(71)
    K = _device_counts(n, m, 73)
    nm = np.exp(rng.normal(0.0, 0.3, K.shape))
    tx = np.exp(rng.normal(7.0, 0.5, K.shape))
    geo = np.exp(rng.normal(4.5, 1.0, n))
    geo[[3, n // 2]] = 0.0
    geo[[4, n - 2]] = -1.0
    mask = np.zeros(n, dtype=bool)
    mask[n // 5:] = rng.random(n - n // 5) < 0.3                 # none in the first fifth
    idx = np.flatnonzero(rng.random(n) < 0.2)
    return K, nm, tx, geo, mask, idx


SHARD_CASES = [("sf", "ratio", "mask", False), ("sf", "poscounts", "index", False), ("sf", "ratio", None, True),
               ("sf", "ratio", "index", True), ("normMatrix", "ratio", "mask", False),
               ("normMatrix", "poscounts", "index", False), ("avgTxLength", "ratio", "mask", True)]


def _local_control(form, mask, idx, lo, hi):
    if form == "mask":
        return mask[lo:hi]
    if form == "index":
        return idx[(idx >= lo) & (idx < hi)] - lo
    return None


def _ctl_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    cuts = _shard_cuts(n, world)
    lo, hi = cuts[rank], cuts[rank + 1]
    K, nm, tx, geo, mask, idx = _shard_inputs(n, m)
    y = gm(K[lo:hi], dev)
    out = []
    for src, type_, form, use_geo in SHARD_CASES:
        kw = {"controlGenes_local": _local_control(form, mask, idx, lo, hi),
              "geoMeans_local": geo[lo:hi] if use_geo else None}
        if src == "sf":
            r = sharded.sharded_size_factors_device(y, m, type=type_, **kw)
            out.append({"sf": r["sizeFactors"], "lg": r["loggeomeans"], "collectives": r["collectives"]})
        else:
            mat = gm((nm if src == "normMatrix" else tx)[lo:hi], dev)
            r = sharded.sharded_normalization_factors(y, m, type=type_, **{src + "_local": mat}, **kw)
            out.append({"sf": r["sizeFactors"], "nf": r["normalizationFactors"][:, :m],
                        "collectives": r["collectives"]})
    errors = []
    for fn in ("sf", "nf"):
        bad = _local_control("index", mask, idx, lo, hi)
        if rank == world - 1:
            bad = np.r_[bad, hi - lo]                             # one past this rank's rows, on the last rank only
        try:
            if fn == "sf":
                sharded.sharded_size_factors_device(y, m, controlGenes_local=bad)
            else:
                sharded.sharded_normalization_factors(y, m, normMatrix_local=gm(nm[lo:hi], dev),
                                                      controlGenes_local=bad)
            errors.append("no error")
        except ValueError as e:
            errors.append(str(e))
    out.append(errors)
    return out


def _check_shards(backend, n, m, world):
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_ctl_rank, n, m, world=world, backend=backend)
    cuts = _shard_cuts(n, world)
    K, nm, tx, geo, mask, idx = _shard_inputs(n, m)
    dev = DEVICE[backend]
    y = gm(K, dev)
    if world > 1:
        assert not mask[cuts[0]:cuts[1]].any()                    # rank 0 holds no control row of the mask
    for i, (src, type_, form, use_geo) in enumerate(SHARD_CASES):
        ctl = {"mask": mask, "index": idx, None: None}[form]
        g = geo if use_geo else None
        if src == "sf":
            w = DP.size_factors(y, m, type=type_, controlGenes=ctl, geoMeans=g)
            sf = w["sizeFactors"]
            if type_ == "poscounts":
                sf = sf / torch.exp(torch.log(sf).mean())          # as the sharded estimate (and DESeq_device) rescale
            lg = w["loggeomeans"].cpu().numpy()
        else:
            w = DP.normalization_factors(y, m, type=type_, controlGenes=ctl, geoMeans=g,
                                         **{src: gm(nm if src == "normMatrix" else tx, dev)})
            sf, nf = w["sizeFactors"], w["normalizationFactors"][:, :m].cpu().numpy()
        sf = sf.cpu().numpy()
        assert np.isfinite(sf).all(), i
        for r, gr in enumerate(got):
            c = gr[i]
            assert np.array_equal(c["sf"], sf), (i, r)
            assert c["collectives"] == SF_COLLECTIVES, (i, r)
            if src == "sf":
                assert np.array_equal(c["lg"], lg[cuts[r]:cuts[r + 1]], equal_nan=True), (i, r)
            else:
                assert np.array_equal(c["nf"], nf[cuts[r]:cuts[r + 1]]), (i, r)
    for gr in got[:-1]:
        assert all("other rank" in e for e in gr[-1]), gr[-1]
    assert all("controlGenes indices" in e for e in got[-1][-1]), got[-1][-1]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharded_control_genes_equal_whole(emu_dev, world):
    _check_shards("gloo", 240, 6, world)


# ---------------------------------------------------------------- spike-ins end to end

def _spike_in_set(seed=2024):
    """2000 endogenous genes and 92 spike-ins, 6 + 6 samples with known library sizes; 40 % of the endogenous genes are
    raised 2x in the second condition, the spike-ins follow the library size only."""
    rng = np.random.default_rng(seed)
    m, n_endo, n_spike = 12, 2000, 92
    lib = np.exp(rng.normal(0.0, 0.35, m))
    cond = np.r_[np.zeros(6), np.ones(6)]
    base = np.exp(rng.uniform(3.0, 8.0, n_endo + n_spike))
    raised = np.zeros(n_endo + n_spike, dtype=bool)
    raised[rng.choice(n_endo, int(0.4 * n_endo), replace=False)] = True
    mu = base[:, None] * lib[None, :] * np.where(raised[:, None] & (cond[None, :] == 1), 2.0, 1.0)
    disp = 0.02
    K = rng.negative_binomial(1 / disp, 1 / (1 + disp * mu)).astype(np.int32)
    spikes = np.arange(n_endo, n_endo + n_spike)
    return K, lib, cond, raised, spikes, disp


def _sampling_bound(K, spikes, lib):
    """Four standard errors of the median of 92 spike-in log ratios: s is the spread of one ratio, measured on the
    spike-ins against the true library sizes, and the median's standard error is 1.2533 s / sqrt(92).  A factor off by
    more than that (after centring) is not sampling noise."""
    lr = np.log(K[spikes]) - np.log(K[spikes]).mean(axis=1, keepdims=True) - np.log(lib)[None, :]
    return 4 * 1.2533 * float(lr.std()) / math.sqrt(len(spikes))


def test_spike_ins_recover_library_sizes_host():
    from deseq2_b200 import pipeline
    K, lib, cond, raised, spikes, disp = _spike_in_set()
    bound = _sampling_bound(K, spikes, lib)
    assert bound < 0.1
    for sf, ok in ((pipeline.estimateSizeFactorsForMatrix(K, controlGenes=spikes), True),
                   (pipeline.estimateSizeFactorsForMatrix(K), False)):
        e = np.log(sf) - np.log(lib)
        e = e - e.mean()
        assert (np.max(np.abs(e)) < bound) == ok, (np.max(np.abs(e)), bound)


def _check_spike_ins(dev):
    from deseq2_b200 import device_pipeline as DP
    K, lib, cond, raised, spikes, disp = _spike_in_set()
    bound = _sampling_bound(K, spikes, lib)
    y = gm(K, dev)
    x = np.c_[np.ones(len(cond)), cond]
    endo = np.arange(K.shape[0]) < spikes[0]
    medians = {}
    for name, sf in (("spikes", DP.size_factors(y, len(cond), controlGenes=spikes)["sizeFactors"]),
                     ("all", DP.size_factors(y, len(cond))["sizeFactors"])):
        e = np.log(sf.cpu().numpy()) - np.log(lib)
        e = e - e.mean()
        assert (np.max(np.abs(e)) < bound) == (name == "spikes"), (name, np.max(np.abs(e)), bound)
        r = DP.DESeq_device(y, x, sizeFactors=sf)
        lfc = np.full(K.shape[0], np.nan)
        lfc[r["idx"].cpu().numpy()] = r["betaMatrix"][:, 1].cpu().numpy()
        medians[name] = (np.nanmedian(lfc[endo & ~raised]), np.nanmedian(lfc[endo & raised]))
    # the median of 1200 (800) fold changes: its spread is far below 0.05 at these means
    assert abs(medians["spikes"][0]) < 0.05 and abs(medians["spikes"][1] - 1) < 0.05, medians
    assert medians["all"][0] < -0.15 and medians["all"][1] < 0.85, medians


# ---------------------------------------------------------------- on the H100

@pytest.mark.gpu
def test_device_matches_host_mirror_c2(engine):
    """At C2 size (50 000 x 100)."""
    _check_device(DEV, 50000, 100, 31)


@pytest.mark.gpu
def test_device_edges_gpu(engine):
    _check_device_edges(DEV)


@pytest.mark.gpu
def test_frozen_round_trip_c2(engine):
    _check_frozen_round_trip(DEV, 50000, 100, 33)


@pytest.mark.gpu
def test_spike_ins_end_to_end(engine):
    _check_spike_ins(DEV)


@pytest.mark.gpu
def test_sharded_control_genes_over_nccl(engine):
    _check_shards("nccl", 20000, 100, nccl_world(3))


@pytest.mark.gpu
def test_sharded_control_genes_one_rank_over_nccl(engine):
    """One NCCL rank, so that a one-GPU host checks the sharded estimate against the single-device one on the device."""
    if DEV != "cuda" or torch.cuda.device_count() < 1:
        pytest.skip("needs a GPU")
    _check_shards("nccl", 20000, 100, 1)
