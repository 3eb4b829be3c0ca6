"""Gene-sharded multi-GPU driver for the Wald path: one process per GPU (torch.distributed), contiguous
gene blocks per rank exactly as the reference's BiocParallel driver chunks them (R/parallel.R:9-10:
`sort(rep(seq_len(nworkers), length.out=nrow))`), two global synchronisation points where the reference has
them (R/parallel.R:25-28: dispersion trend + prior variance need every gene's dispGeneEst / baseMean) and one
final all-gather of the per-gene results so rank 0 holds what results()/lfcShrink() consume (R/parallel.R:54-66).
The n x m matrices (mu, H) stay on their shard: they never cross NVLink.

Backend: "nccl" on GPUs (tensors on the rank's device), "gloo" for the CPU tests.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.distributed as dist

from . import pipeline


def shard_bounds(n: int, world: int, rank: int):
    """Contiguous block of genes owned by `rank` (first n % world ranks get one extra gene)."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def _dev():
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")


def all_gather_rows(local: np.ndarray, n_total: int) -> np.ndarray:
    """All-gather a per-gene array (first axis = genes of this rank's shard) into the full (n_total, ...) array
    on every rank.  Shards are padded to the largest shard so a single all_gather_into_tensor suffices."""
    world, rank = dist.get_world_size(), dist.get_rank()
    local = np.ascontiguousarray(local, dtype=np.float64)
    tail = local.shape[1:]
    width = int(np.prod(tail)) if tail else 1
    cap = max(shard_bounds(n_total, world, r)[1] - shard_bounds(n_total, world, r)[0] for r in range(world))
    buf = torch.zeros((cap, width), dtype=torch.float64, device=_dev())
    if local.shape[0]:
        buf[: local.shape[0]] = torch.from_numpy(local.reshape(local.shape[0], width)).to(buf.device)
    out = torch.empty((world * cap, width), dtype=torch.float64, device=buf.device)
    dist.all_gather_into_tensor(out, buf)
    out = out.cpu().numpy().reshape(world, cap, width)
    parts = []
    for r in range(world):
        lo, hi = shard_bounds(n_total, world, r)
        parts.append(out[r, : hi - lo])
    return np.concatenate(parts, axis=0).reshape((n_total,) + tail)


def sharded_DESeq(counts, x, sizeFactors, engine=None):
    """DESeq() Wald path on this rank's gene shard with the reference's two global steps.
    `counts` is the FULL matrix on every rank (synthetic benchmarks generate it everywhere; a real loader
    would read only the shard); returns the full per-gene result dict (identical on every rank)."""
    world, rank = dist.get_world_size(), dist.get_rank()
    counts = np.asarray(counts)
    N, m = counts.shape
    p = x.shape[1]
    lo, hi = shard_bounds(N, world, rank)
    mine = counts[lo:hi]
    mv = pipeline.getBaseMeansAndVariances(mine, sizeFactors)
    nz = ~mv["allZero"]
    cnz = mine[nz]
    mvnz = {k: v[nz] for k, v in mv.items()}
    ge = pipeline.estimateDispersionsGeneEst(cnz, sizeFactors, x, engine=engine, mv=mvnz)

    def full_local(v, fill=np.nan):
        out = np.full((hi - lo,) + v.shape[1:], fill)
        out[nz] = v
        return out

    # ---- global step 1 (R/parallel.R:25-28): trend + prior variance from ALL genes
    g1 = all_gather_rows(np.stack([full_local(ge["dispGeneEst"]), full_local(ge["baseMean"])], axis=1), N)
    ok = ~np.isnan(g1[:, 0])
    tf = pipeline.estimateDispersionsFit(g1[ok, 0], g1[ok, 1])
    dispPriorVar = pipeline.estimateDispersionsPriorVar(tf["varLogDispEsts"], m, p, g1[ok, 0], tf["dispFit"])
    dispFit_mine = tf["coefs"][0] + tf["coefs"][1] / ge["baseMean"]
    mp = pipeline.estimateDispersionsMAP(cnz, x, ge["mu"], ge["dispGeneEst"], dispFit_mine, dispPriorVar,
                                         tf["varLogDispEsts"], engine=engine)
    nf = np.broadcast_to(sizeFactors[None, :], cnz.shape)
    wt = pipeline.nbinomWaldTest(cnz, nf, x, mp["dispersion"], engine=engine)
    # ---- final gather (R/parallel.R:54-66): per-gene scalars only
    cols = [full_local(ge["dispGeneEst"]), full_local(dispFit_mine), full_local(mp["dispMAP"]),
            full_local(mp["dispersion"]), full_local(wt["betaIter"]), full_local(wt["deviance"])]
    packed = np.concatenate([np.stack(cols, axis=1), full_local(wt["betaMatrix"]), full_local(wt["betaSE"]),
                             full_local(wt["WaldStatistic"]), full_local(wt["WaldPvalue"])], axis=1)
    allp = all_gather_rows(packed, N)
    k = len(cols)
    return {"dispGeneEst": allp[:, 0], "dispFit": allp[:, 1], "dispMAP": allp[:, 2], "dispersion": allp[:, 3],
            "betaIter": allp[:, 4], "deviance": allp[:, 5], "betaMatrix": allp[:, k:k + p],
            "betaSE": allp[:, k + p:k + 2 * p], "WaldStatistic": allp[:, k + 2 * p:k + 3 * p],
            "WaldPvalue": allp[:, k + 3 * p:k + 4 * p], "dispPriorVar": dispPriorVar, "trendCoefs": tf["coefs"]}


class PackedGather:
    """ONE collective per exchange: several per-gene 1-D vectors of this rank (all of the same, rank-dependent length)
    travel as one (1 + ncols) x cap buffer -- row 0 carries the shard's length -- through a single
    all_gather_into_tensor, and come back concatenated over the ranks in rank order (R/parallel.R:54-66's rbind).
    `cap` (rows of the largest shard) is agreed once per run with one 8-byte all-reduce, or given by a caller to whom
    every rank's row count is already known (no collective then)."""

    def __init__(self, n_local_rows: int, device, cap=None):
        self.world = dist.get_world_size()
        if cap is None:
            c = torch.tensor([int(n_local_rows)], dtype=torch.int64, device=device)
            dist.all_reduce(c, op=dist.ReduceOp.MAX)
            cap, self.collectives = int(c.item()), 1
        else:
            self.collectives = 0
        self.cap = max(int(cap), 1)

    def __call__(self, cols):
        single = isinstance(cols, torch.Tensor)
        cols = [cols] if single else list(cols)
        n = cols[0].numel()
        dev = cols[0].device
        buf = torch.zeros((len(cols) + 1, self.cap), dtype=torch.float64, device=dev)
        buf[0, 0] = float(n)
        for k, c in enumerate(cols):
            buf[k + 1, :n] = c.to(torch.float64)
        out = torch.empty((self.world * buf.shape[0], self.cap), dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(out, buf)       # rank r's buffer = rows [r (1 + ncols), (r + 1)(1 + ncols))
        out = out.view(self.world, buf.shape[0], self.cap)
        self.collectives += 1
        sizes = [int(v) for v in out[:, 0, 0].tolist()]
        self.sizes = sizes
        res = [torch.cat([out[r, k + 1, :sizes[r]] for r in range(self.world)]) for k in range(len(cols))]
        return res[0] if single else res


def allgather_1d(t: torch.Tensor) -> torch.Tensor:
    """Concatenate a 1-D tensor of rank-dependent length over the ranks (rank order): a PackedGather of one column."""
    return PackedGather(t.numel(), t.device)(t)


def gathered_xim(nf_rows, m, pg):
    """momentsDispEstimate's xim = mean(1 / colMeans(nf)) over the rows nf_rows of EVERY rank: ONE all-gather carries
    each rank's m column sums and its row count (m + 1 doubles), summed on every rank in rank order, so every rank gets
    the same bits.  Counted in pg.collectives.  The partial sums make the last bit depend on where the shards split,
    so xim can differ in the last bit from the single-device sum over the same rows."""
    from . import device_pipeline as DP
    colsum, count = DP.nf_column_sums(nf_rows, m)
    mine = torch.cat([colsum, torch.tensor([float(count)], dtype=torch.float64, device=colsum.device)])
    allr = torch.empty(pg.world * (m + 1), dtype=torch.float64, device=mine.device)
    dist.all_gather_into_tensor(allr, mine.contiguous())
    allr = allr.view(pg.world, m + 1)
    pg.collectives += 1
    tot = allr[0].clone()
    for r in range(1, pg.world):                    # rank order: the same bits on every rank
        tot = tot + allr[r]
    return DP.nf_xim(tot[:m], tot[m])


def sharded_DESeq_device(y_local, x, sizeFactors=None, **kw):
    """Device-resident DESeq() on this rank's gene shard (y_local: gene-major counts of the shard, on the rank's GPU)
    with the reference's global step on all genes (dispersion trend + prior variance, R/parallel.R:25-28).  The whole run
    issues TWO per-gene collectives: one packed all-gather of (baseMean, dispGeneEst) for the global step and ONE packed
    all-gather of the results (dispersion, betaMatrix, betaSE, WaldPvalue: 1 + 3p doubles per gene), plus an 8-byte
    all-reduce that agrees on the buffer size; the n x m matrices never leave their shard.  Returns the shard's result
    dict (device tensors) plus "gathered": the results of ALL genes on every rank, in rank order, and "collectives".
    betaPrior=True, factors=... (passed on to DESeq_device): the prior variance is estimated over all genes
    (R/parallel.R:39-40) through ONE more packed all-gather of the p - 1 non-intercept MLE columns; the gathered
    results then carry the expanded matrix's columns.
    weights=w_local (passed on to DESeq_device): this shard's rows of the observation weights, gene-major like
    y_local; no collective is added (the global step's gather carries the weighted baseMean).
    normalizationFactors=nf_local (passed on to DESeq_device): this shard's rows of the normalization factors,
    gene-major like y_local.  The moments dispersion's xim = mean(1 / colMeans(nf)) is over the non-all-zero rows of
    ALL ranks, as a serial DESeq() computes it: ONE more all-gather carries each rank's m column sums and its row count
    (m + 1 doubles), summed on every rank in rank order, so xim does not depend on the number of ranks (the reference's
    DESeqParallel uses each chunk's own xim instead, R/parallel.R:18-20).  Not supported with finite
    minReplicatesForReplace (the refitted rows' xim would need another collective) or avgTxLength: estimate the
    factors with sharded_normalization_factors and pass them.
    sizeFactors=None estimates median-of-ratios size factors from this rank's shard only (unchanged: the ranks then
    differ); pass sharded_size_factors_device(y_local, m)["sizeFactors"] for the size factors of all genes.
    test="LRT", reduced=... (passed on to DESeq_device): the LRT columns are per gene, so no collective is added;
    LRTStatistic and LRTPvalue travel in the result gather in place of WaldPvalue (1 + 2p + 2 doubles per gene).
    useT=True, df=df_local (passed on to DESeq_device): df is this rank's rows (a scalar, or one value per row of
    y_local); the t degrees of freedom and p-values are per gene, so no collective is added, and the gathered
    WaldPvalue columns are the t ones.  sharded_results_device / sharded_lfcShrink_device infer t mode from the
    shard's "tDegreesFreedom" as results_device does."""
    from . import device_pipeline as DP
    if kw.get("sfType") == "iterate":
        raise ValueError("sharded runs do not estimate iterate size factors (every perturbation needs a quantile over "
                         "all genes): estimate them on one device (size_factors_iterate) and pass sizeFactors")
    pg = PackedGather(y_local.shape[0], y_local.device)
    nf = kw.get("normalizationFactors")
    if kw.get("avgTxLength") is not None:
        raise ValueError("sharded runs do not estimate normalization factors: estimate them on one device "
                         "(normalization_factors) or pass normalizationFactors")
    if nf is not None:
        if np.isfinite(kw.get("minReplicatesForReplace", np.inf)):
            raise ValueError("sharded normalization factors are not supported with outlier replacement "
                             "(finite minReplicatesForReplace)")
        m = np.asarray(x).shape[0]
        DP._check_positive_matrix(nf, y_local, m, "normalizationFactors")
        nz = y_local[:, :m].sum(dim=1) != 0
        kw["nfXim"] = gathered_xim(nf[nz], m, pg)
    res = DP.DESeq_device(y_local, x, sizeFactors, allgather=pg, **kw)
    p = res["betaMatrix"].shape[1]
    lrt = res["test"] == "LRT"
    tests = [res["LRTStatistic"], res["LRTPvalue"]] if lrt else [res["WaldPvalue"][:, k] for k in range(p)]
    cols = [res["dispersion"]] + [res["betaMatrix"][:, k] for k in range(p)] \
        + [res["betaSE"][:, k] for k in range(p)] + tests
    g = pg(cols)
    res["gathered"] = {"dispersion": g[0], "betaMatrix": torch.stack(g[1:1 + p], dim=1),
                       "betaSE": torch.stack(g[1 + p:1 + 2 * p], dim=1)}
    if lrt:
        res["gathered"]["LRTStatistic"], res["gathered"]["LRTPvalue"] = g[1 + 2 * p], g[2 + 2 * p]
    else:
        res["gathered"]["WaldPvalue"] = torch.stack(g[1 + 2 * p:1 + 3 * p], dim=1)
    res["collectives"] = pg.collectives
    return res


def sharded_nbinomLRT_device(y_local, x_full, x_reduced, sizeFactors, dispersion_local, **kw):
    """nbinomLRT on this rank's shard (BASELINE config 5's call sequence: full and reduced IRLS fit, LRT statistic) and
    ONE packed all-gather of (LRTStatistic, LRTPvalue, betaMatrix of the full model) to every rank."""
    from . import device_pipeline as DP
    pg = PackedGather(y_local.shape[0], y_local.device)
    res = DP.nbinomLRT_device(y_local, x_full, x_reduced, sizeFactors, dispersion_local, **kw)
    p = res["betaMatrix"].shape[1]
    g = pg([res["LRTStatistic"], res["LRTPvalue"]] + [res["betaMatrix"][:, k] for k in range(p)])
    res["gathered"] = {"LRTStatistic": g[0], "LRTPvalue": g[1], "betaMatrix": torch.stack(g[2:2 + p], dim=1)}
    res["collectives"] = pg.collectives
    return res


def sharded_results_device(res_local, y_local, x, **kw):
    """results() on this rank's shard of a sharded_DESeq_device run (y_local: the shard's rows as shard_bounds splits
    them; res_local: its result).  The per-gene steps stay local; ONE packed all-gather carries [filter, pvalue] of
    every gene, and every rank runs the cutoff, rejection-count and adjusted-column kernels on all genes, then keeps
    its own rows.  Keyword arguments as device_pipeline.results_device (a custom `filter` holds this shard's rows);
    returns its dict for the shard, whose metadata is that of all genes, plus "collectives"."""
    from . import device_pipeline as DP
    pg = PackedGather(y_local.shape[0], y_local.device)
    out = DP.results_device(res_local, y_local, x, allgather=pg, **kw)
    out["collectives"] = pg.collectives
    return out


def sharded_lfcShrink_device(res_local, y_local, x, **kw):
    """lfcShrink(type = "normal") on this rank's shard of a sharded_DESeq_device run (y_local: the shard's rows as
    shard_bounds splits them; res_local: its result).  The prior needs every gene: ONE packed all-gather carries
    baseMean, dispFit and the p - 1 non-intercept MLE columns of every rank's rows (2 + p - 1 doubles per gene), and
    every rank estimates the same prior from them; the MAP fit stays local.  The default results table (when
    results= is not given) and, with lfcThreshold > 0, the shrunk table each take sharded_results_device's one gather
    of [filter, pvalue].  Keyword arguments as device_pipeline.lfcShrink_device; returns its dict for the shard plus
    "collectives" (the size agreement included)."""
    from . import device_pipeline as DP
    pg = PackedGather(y_local.shape[0], y_local.device)
    out = DP.lfcShrink_device(res_local, y_local, x, allgather=pg, **kw)
    out["collectives"] = pg.collectives
    return out


# ---------------------------------------------------------------- size factors, normalization factors and the
# transforms on gene shards (R/core.R:535-578, 2159-2163; R/vst.R; R/helper.R:421-435)

_SIGN = -(1 << 63)                                  # int64 with only the sign bit set
_LOW63 = (1 << 63) - 1


def _order_keys(v):
    """sf_median_kernel's key_of (csrc/size_factors.cu): the order-preserving unsigned 64-bit image of float64 values,
    its bits held in an int64 tensor (compare two keys as unsigned with _below)."""
    b = v.view(torch.int64)
    return torch.where(b < 0, ~b, b | _SIGN)


def _key_values(k):
    """value_of: the float64 values of _order_keys keys."""
    return torch.where(k < 0, k & _LOW63, ~k).view(torch.float64)


def _below(a, b):
    """a < b for unsigned keys held in int64."""
    return (a ^ _SIGN) < (b ^ _SIGN)


_KEY_INF = (0x7ff0000000000000 | (1 << 63)) - (1 << 64)     # _order_keys(+Inf): entries that do not take part


def _exp_as_kernel(v):
    """exp(v) with the bits of sf_median_kernel's exp: CUDA's exp on the GPU (torch's CUDA exp is the same libdevice
    function); where the engine's CUDA source runs on the host (the SIMT emulator), the C library's exp, which
    math.exp calls, as torch's vectorised CPU exp can differ from it in the last bit."""
    if v.device.type == "cuda":
        return torch.exp(v)

    def one(e):
        try:
            return math.exp(e)
        except OverflowError:
            return math.inf
    return torch.tensor([one(e) for e in v.tolist()], dtype=torch.float64, device=v.device)


def _local_ratios(y_local, m, poscounts, divisor=None):
    """The size-factor kernel on this shard (device_pipeline.size_factor_ratios); an empty shard launches nothing."""
    from . import device_pipeline as DP
    if y_local.shape[0] == 0:
        dev = y_local.device
        return {"ratios": torch.empty((m, 0), dtype=torch.float64, device=dev),
                "loggeomeans": torch.empty(0, dtype=torch.float64, device=dev),
                "n_finite": torch.zeros(1, dtype=torch.int32, device=dev)}
    return DP.size_factor_ratios(y_local, m, poscounts=poscounts, divisor=divisor)


def _agree(r, failed=False):
    """ONE integer all-reduce (SUM) of m + 2 int64: the number of ratios that take part in each sample's median, the
    number of genes with a finite log geometric mean and the number of ranks whose arguments failed their checks.
    Returns (per-sample counts as a device tensor, n_finite, failed ranks) -- the same on every rank -- and this
    rank's entries that take part as (keys, sample of each key) for _global_median."""
    ratios = r["ratios"]
    m = ratios.shape[0]
    dev = ratios.device
    keys = _order_keys(ratios)
    use = _below(keys, torch.tensor(_KEY_INF, dtype=torch.int64, device=dev))
    head = torch.cat([use.sum(dim=1), r["n_finite"].to(torch.int64),
                      torch.tensor([int(failed)], dtype=torch.int64, device=dev)])
    dist.all_reduce(head)
    tail = head[-2:].tolist()
    entries = (keys[use], torch.arange(m, dtype=torch.int64, device=dev).view(m, 1).expand_as(keys)[use])
    return head[:-2], int(tail[0]), int(tail[1]), entries


def _global_median(entries, nv):
    """The median of each sample's log ratios over the entries of EVERY rank that take part (not +Inf), as
    sf_median_kernel takes it over one device's: the key of the lower middle element (0-based rank (nv - 1) / 2) and,
    for an even count nv, of the upper middle element are found together by an MSB-first radix select on the
    order-preserving 64-bit keys, 8 bits per round.  entries: this rank's (keys, sample of each key) from _agree.  Each
    round every rank builds the digit histograms of its matching entries (2 targets x m samples x 256 digits, int64;
    in the first round both targets share one) and ONE integer all-reduce (SUM) adds them, so the selected keys
    depend neither on the number of ranks nor on the reduction order; then every rank keeps only the entries under one
    of the two new prefixes.  8 collectives of 2 x m x 256 x 8 bytes; no ratio leaves its rank.  Returns (m,) medians
    0.5 * (lower + upper) (the lower middle for an odd count, NaN for nv = 0) and the number of collectives."""
    kk, jj = entries
    m = nv.numel()
    dev = nv.device
    r0 = torch.clamp(nv - 1, min=0) // 2
    rk = torch.stack([r0, r0 + (nv % 2 == 0).to(torch.int64)])     # residual ranks of the (lower, upper) targets
    prefix = torch.zeros((2, m), dtype=torch.int64, device=dev)
    for rnd in range(7, -1, -1):
        s = 8 * rnd
        idx = jj * 256 + ((kk >> s) & 255)
        hist = torch.empty((2, m * 256), dtype=torch.int64, device=dev)
        if rnd == 7:                                                 # no prefix yet: one histogram for both targets
            hist[0] = torch.bincount(idx, minlength=m * 256)
            hist[1] = hist[0]
        else:
            for t in range(2):
                hist[t] = torch.bincount(idx[(kk >> (s + 8)) == (prefix[t][jj] >> (s + 8))], minlength=m * 256)
        dist.all_reduce(hist)
        cum = hist.view(2, m, 256).cumsum(dim=2)
        b = (cum <= rk.unsqueeze(2)).sum(dim=2).clamp(max=255)       # the first digit whose cumulative count > rank
        rk = rk - torch.where(b > 0, cum.gather(2, (b - 1).clamp(min=0).unsqueeze(2)).squeeze(2), 0)
        prefix = prefix | (b << s)
        top = kk >> s
        keep = (top == (prefix[0][jj] >> s)) | (top == (prefix[1][jj] >> s))
        kk, jj = kk[keep], jj[keep]
    lo, hi = _key_values(prefix[0]), _key_values(prefix[1])
    med = torch.where(nv % 2 == 1, lo, 0.5 * (lo + hi))
    return torch.where(nv == 0, torch.nan, med), 8


def _sizes_of(med, nv):
    sf = _exp_as_kernel(med)
    return torch.where(nv == 0, torch.nan, sf)


def _control_local(y_local, m, type, divisor, controlGenes_local, geoMeans_local):
    """device_pipeline.control_ratios on this shard, with its ValueError held rather than raised, so that the rank
    still joins the agreement all-reduce (which carries the failure to every rank): returns (ratios dict, error)."""
    from . import device_pipeline as DP
    try:
        return DP.control_ratios(y_local, m, type, divisor, controlGenes_local, geoMeans_local), None
    except ValueError as e:
        return _local_ratios(y_local[:0], m, False), e


def _raise_failed(err, failed, what):
    if err is not None:
        raise err
    if failed:
        raise ValueError(f"{what}: the arguments of {failed} other rank(s) failed their checks")


def sharded_size_factors_device(y_local, m, type="ratio", controlGenes_local=None, geoMeans_local=None):
    """estimateSizeFactorsForMatrix (R/core.R:535-578, locfunc = median) over the genes of ALL ranks, y_local being this
    rank's rows (gene-major, split as shard_bounds splits them).  The log geometric means are per gene and the log
    ratios are the size-factor kernel's own (b200nb_size_factors_dev, whose column-major ratio scratch it reads); the
    per-sample median over every rank's ratios is _global_median.  Every rank gets the sizeFactors that
    device_pipeline.size_factors gives for the whole matrix, bit for bit; for "poscounts" they are then rescaled to
    geometric mean 1 (the incoming-geoMeans step, R/core.R:573-576) exactly as DESeq_device does.  A sample with no
    usable ratio gets NaN.  "Every gene contains at least one zero" is decided on the count of finite log geometric
    means of all ranks and raises ValueError on every rank.  Returns {"sizeFactors": (m,) device tensor, "loggeomeans":
    this shard's (n_local,), "collectives": 9 (one agreement all-reduce and 8 histogram rounds)}.
    controlGenes_local (a mask or 0-based indices into this rank's rows) and geoMeans_local (this rank's rows; when
    geoMeans are used every rank passes its part, an empty one for an empty shard) as in device_pipeline.size_factors:
    the ratios are control_ratios' (the kernel's on the gathered control rows, or given_geo_mean_ratios), the median is
    _global_median over the control entries of every rank, the stop count is over every row of every rank, and with
    geoMeans the factors are rescaled to geometric mean 1.  Every rank then gets the single-device size_factors of the
    whole matrix and its control rows, bit for bit (rescaled for "poscounts" as above).  Arguments that fail their
    checks on one rank raise ValueError on every rank; the count of collectives stays 9."""
    from . import device_pipeline as DP
    if controlGenes_local is not None or geoMeans_local is not None:
        r, err = _control_local(y_local, m, type, None, controlGenes_local, geoMeans_local)
        nv, n_finite, failed, entries = _agree(r, failed=err is not None)
        _raise_failed(err, failed, "size_factors")
        if n_finite == 0:
            raise DP._no_finite_loggeomean()
        med, c = _global_median(entries, nv)
        sf = _sizes_of(med, nv)
        if type == "poscounts" or r["incoming"]:
            sf = DP.rescaled_to_geo_mean_one(sf)
        return {"sizeFactors": sf, "loggeomeans": r["loggeomeans"], "collectives": 1 + c}
    if type not in ("ratio", "poscounts"):
        raise ValueError("type must be 'ratio' or 'poscounts'")
    r = _local_ratios(y_local, m, type == "poscounts")
    nv, n_finite, _, entries = _agree(r)
    if n_finite == 0:
        raise DP._no_finite_loggeomean()
    med, c = _global_median(entries, nv)
    sf = _sizes_of(med, nv)
    if type == "poscounts":
        sf = sf / torch.exp(torch.log(sf).mean())
    return {"sizeFactors": sf, "loggeomeans": r["loggeomeans"], "collectives": 1 + c}


def sharded_normalization_factors(y_local, m, normMatrix_local=None, avgTxLength_local=None, type="ratio",
                                  controlGenes_local=None, geoMeans_local=None):
    """device_pipeline.normalization_factors over the genes of ALL ranks (estimateNormFactors, R/core.R:2159-2163, and
    the avgTxLength path): normMatrix_local / avgTxLength_local are this shard's rows, gene-major like y_local.  The size
    factors of K / normMatrix come from the global median of sharded_size_factors_device; everything else is per gene.
    controlGenes_local / geoMeans_local as in sharded_size_factors_device.
    A matrix that fails its checks on any rank raises ValueError on every rank (the failure travels in the agreement
    all-reduce).  Returns {"normalizationFactors": this shard's (n_local, ld), "sizeFactors": (m,), "collectives": 9},
    which sharded_DESeq_device(normalizationFactors=...) and the sharded transforms take."""
    from . import device_pipeline as DP
    err = None
    chosen = controlGenes_local is not None or geoMeans_local is not None
    try:
        nm, d = DP.norm_divisor(y_local, m, normMatrix_local, avgTxLength_local, type)
        if chosen:
            r, err = _control_local(y_local, m, type, d, controlGenes_local, geoMeans_local)
        else:
            r = _local_ratios(y_local, m, type == "poscounts", divisor=d)
    except ValueError as e:
        err = e
        r = _local_ratios(y_local[:0], m, False)
    nv, n_finite, failed, entries = _agree(r, failed=err is not None)
    _raise_failed(err, failed, "normalization_factors")
    if n_finite == 0:
        raise DP._no_finite_loggeomean()
    med, c = _global_median(entries, nv)
    sf = _sizes_of(med, nv)
    if chosen and r["incoming"]:
        sf = DP.rescaled_to_geo_mean_one(sf)
    out = DP.norm_factors_from(nm, d, sf, m, type)
    out["collectives"] = 1 + c
    return out


def _sharded_factors(y_local, m, sizeFactors, normalizationFactors, avgTxLength):
    """device_pipeline._factors with the estimates of every rank: returns (size factors or None, nf rows or None, sfd,
    the collectives of the estimate)."""
    from . import device_pipeline as DP
    n = 0
    if avgTxLength is not None:
        if normalizationFactors is not None:
            raise ValueError("give normalizationFactors or avgTxLength, not both")
        if sizeFactors is not None:
            raise ValueError("avgTxLength estimates normalization factors: sizeFactors must be None")
        r = sharded_normalization_factors(y_local, m, avgTxLength_local=avgTxLength)
        normalizationFactors, n = r["normalizationFactors"], r["collectives"]
    elif normalizationFactors is not None:
        err = None
        try:
            DP._check_positive_matrix(normalizationFactors, y_local, m, "normalizationFactors")
        except ValueError as e:
            err = e
        _fail_together(err, y_local.device, "normalizationFactors")
        n = 1
    elif sizeFactors is None:
        r = sharded_size_factors_device(y_local, m)
        sizeFactors, n = r["sizeFactors"], r["collectives"]
    return DP._factors(y_local, m, sizeFactors, normalizationFactors) + (n,)


def _fail_together(err, dev, what):
    """ONE 8-byte all-reduce (SUM) of the ranks whose arguments failed their checks, so that a check that fails on one
    rank raises ValueError on every rank instead of leaving the others blocked in the next collective."""
    f = torch.tensor([int(err is not None)], dtype=torch.int64, device=dev)
    dist.all_reduce(f)
    if err is not None:
        raise err
    failed = int(f.item())
    if failed:
        raise ValueError(f"{what}: the arguments of {failed} other rank(s) failed their checks")


def _gene_wise(ynz, x, sizeFactors, nfz, xim):
    """device_pipeline.gene_wise_dispersions on this rank's rows; none on a rank without rows."""
    from . import device_pipeline as DP
    if ynz.shape[0] == 0:
        e = torch.empty(0, dtype=torch.float64, device=ynz.device)
        return e, e
    return DP.gene_wise_dispersions(ynz, x, sizeFactors, nfz, xim=xim)


def sharded_varianceStabilizingTransformation_device(y_local, m, x=None, blind=True, fitType="parametric",
                                                     sizeFactors=None, normalizationFactors=None, avgTxLength=None,
                                                     dispersionFunction=None):
    """device_pipeline.varianceStabilizingTransformation_device over the genes of ALL ranks, for this rank's rows
    y_local (gene-major, split as shard_bounds splits them; normalizationFactors / avgTxLength: this shard's rows).
    Factors not given are estimated over all ranks (sharded_size_factors_device, sharded_normalization_factors).  When
    the dispersion function is fitted, GeneEst runs on this shard's non-zero rows, ONE packed all-gather (after the
    8-byte size agreement) brings (baseMean, dispGeneEst) of every rank, and every rank fits the same trend or mean;
    with normalization factors xim is over the non-zero rows of all ranks (gathered_xim, one more all-gather).  The
    transform is local.  Returns the single-device dict for this shard's rows ("vst" is (n_local, m)) plus
    "collectives": 2 with given size factors, 4 with given normalization factors (+ their check and the xim sums),
    11 with estimated size factors, 12 with avgTxLength (the estimate and the xim sums); with a frozen
    dispersionFunction and blind=False 0, 1 or 9 (given size factors, given normalization factors, an estimate).  Given
    normalization factors that fail their check on one rank raise ValueError on every rank."""
    from . import device_pipeline as DP
    refit = blind or dispersionFunction is None
    if refit:
        if not blind and x is None:
            raise ValueError("blind=False needs the design x or a dispersionFunction")
        DP._check_vst_fit_type(fitType)
        x = DP._vst_design(x, m, blind)
    sizeFactors, nf, sfd, n = _sharded_factors(y_local, m, sizeFactors, normalizationFactors, avgTxLength)
    if refit:
        pg = PackedGather(y_local.shape[0], y_local.device)
        idx = torch.nonzero(y_local[:, :m].sum(dim=1) != 0).squeeze(1)
        whole = idx.numel() == y_local.shape[0]
        ynz = y_local if whole else y_local[idx].contiguous()
        nfz = None if nf is None else (nf if whole else nf[idx].contiguous())
        xim = None if nf is None else gathered_xim(nfz, m, pg)
        bm, dge = pg(list(_gene_wise(ynz, x, sizeFactors, nfz, xim)))
        dispersionFunction = DP.dispersion_function_of(bm, dge, fitType)
        n += pg.collectives
    res = DP._vst_result(y_local, m, dispersionFunction, sizeFactors, nf, sfd)
    res["collectives"] = n
    return res


def sharded_vst_device(y_local, m, x=None, blind=True, nsub=1000, fitType="parametric", sizeFactors=None,
                       normalizationFactors=None, avgTxLength=None):
    """device_pipeline.vst_device (R/vst.R:219-267) over the genes of ALL ranks, for this rank's rows y_local
    (gene-major, split as shard_bounds splits them).  Factors as in sharded_varianceStabilizingTransformation_device.
    ONE packed all-gather brings every row's baseMean (1 double per gene); every rank then picks the same subset as
    vst_device: the rows with baseMean > 5 in a stable sort of baseMean (ties in global row order) at
    pipeline.vstSubsetPositions.  Each rank runs GeneEst on its rows of the subset, ONE more packed all-gather brings
    (baseMean, dispGeneEst) of all of them, and they are put back into vst_device's fit order before the trend fit (with
    normalization factors xim is over the subset rows of all ranks: one more all-gather).  R's two stops (fewer than
    nsub rows; fewer than nsub rows with mean > 5) are decided from the gathered baseMean and raise ValueError on every
    rank.  Returns the single-device dict for this shard's rows plus "subset" (global row indices, in fit order) and
    "collectives": 3 with given size factors, 5 with given normalization factors (+ their check and the xim sums),
    12 with estimated size factors, 13 with avgTxLength (the estimate and the xim sums)."""
    from . import device_pipeline as DP
    from .pipeline import vstSubsetPositions
    if not blind and x is None:
        raise ValueError("blind=False needs the design x")
    DP._check_vst_fit_type(fitType)
    x = DP._vst_design(x, m, blind)
    sizeFactors, nf, sfd, n = _sharded_factors(y_local, m, sizeFactors, normalizationFactors, avgTxLength)
    dev = y_local.device
    pg = PackedGather(y_local.shape[0], dev)
    bm_local = DP.prep(y_local, np.ones((m, 1)), sizeFactors, want_mu=False, want_beta0=False,
                       normalizationFactors=nf, xim=1.0)["baseMean"] if y_local.shape[0] else \
        torch.empty(0, dtype=torch.float64, device=dev)
    bm = pg(bm_local)
    if bm.numel() < nsub:
        raise ValueError("less than 'nsub' rows, it is recommended to use varianceStabilizingTransformation directly")
    cand = torch.nonzero(bm > 5).squeeze(1)
    L = cand.numel()
    if L < nsub:
        raise ValueError("less than 'nsub' rows with mean normalized count > 5, it is recommended to use "
                         "varianceStabilizingTransformation directly")
    _, o = torch.sort(bm[cand], stable=True)
    subset = cand[o[torch.as_tensor(vstSubsetPositions(L, nsub), device=dev)]]
    ends = torch.as_tensor(np.cumsum(pg.sizes), device=dev)
    owner = torch.searchsorted(ends, subset, right=True)             # the rank of each subset row, in fit order
    lo = int(ends[dist.get_rank()] - pg.sizes[dist.get_rank()])
    mine = torch.nonzero(owner == dist.get_rank()).squeeze(1)        # this rank's fit positions, ascending
    rows = subset[mine] - lo
    ysub = y_local[rows].contiguous()
    nfsub = None if nf is None else nf[rows].contiguous()
    # every rank knows every rank's subset count: the GeneEst gather is sized for the subset, not the shard
    pg_sub = PackedGather(rows.numel(), dev, cap=int(torch.bincount(owner, minlength=pg.world).max()))
    xim = None if nf is None else gathered_xim(nfsub, m, pg_sub)
    g_bm, g_dge = pg_sub(list(_gene_wise(ysub, x, sizeFactors, nfsub, xim)))
    fit_order = torch.sort(owner, stable=True)[1]                   # the fit position of each gathered entry
    bm_fit, dge_fit = torch.empty_like(g_bm), torch.empty_like(g_dge)
    bm_fit[fit_order], dge_fit[fit_order] = g_bm, g_dge
    res = DP._vst_result(y_local, m, DP.dispersion_function_of(bm_fit, dge_fit, fitType), sizeFactors, nf, sfd)
    res["subset"] = subset
    res["collectives"] = n + pg.collectives + pg_sub.collectives
    return res


def sharded_normTransform_device(y_local, m, sizeFactors=None, normalizationFactors=None, pc=1.0):
    """device_pipeline.normTransform_device (R/helper.R:421-435) for this rank's rows y_local: size factors, when neither
    they nor normalizationFactors (this shard's rows) are given, from sharded_size_factors_device; the transform is
    local.  Returns {"normTransform": (n_local, m) device tensor, "sizeFactors" or "normalizationFactors",
    "collectives": 0, 1 with given normalizationFactors (their check), or 9 for an estimate}.  Given
    normalizationFactors that fail their check on one rank raise ValueError on every rank (in the transforms too)."""
    from . import device_pipeline as DP
    sizeFactors, nf, sfd, n = _sharded_factors(y_local, m, sizeFactors, normalizationFactors, None)
    out = {"normTransform": DP.transform(y_local, m, "log2", pc, 0.0, sfd), "collectives": n}
    if nf is not None:
        out["normalizationFactors"] = nf
    else:
        out["sizeFactors"] = sizeFactors
    return out
