"""Gene-sharded multi-GPU driver for the Wald path: one process per GPU (torch.distributed), contiguous
gene blocks per rank exactly as the reference's BiocParallel driver chunks them (R/parallel.R:9-10:
`sort(rep(seq_len(nworkers), length.out=nrow))`), two global synchronisation points where the reference has
them (R/parallel.R:25-28: dispersion trend + prior variance need every gene's dispGeneEst / baseMean) and one
final all-gather of the per-gene results so rank 0 holds what results()/lfcShrink() consume (R/parallel.R:54-66).
The n x m matrices (mu, H) stay on their shard: they never cross NVLink.

Backend: "nccl" on GPUs (tensors on the rank's device), "gloo" for the CPU tests.
"""
from __future__ import annotations

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
    `cap` (rows of the largest shard) is agreed once per run with one 8-byte all-reduce."""

    def __init__(self, n_local_rows: int, device):
        self.world = dist.get_world_size()
        c = torch.tensor([int(n_local_rows)], dtype=torch.int64, device=device)
        dist.all_reduce(c, op=dist.ReduceOp.MAX)
        self.cap = max(int(c.item()), 1)
        self.collectives = 1

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
        res = [torch.cat([out[r, k + 1, :sizes[r]] for r in range(self.world)]) for k in range(len(cols))]
        return res[0] if single else res


def allgather_1d(t: torch.Tensor) -> torch.Tensor:
    """Concatenate a 1-D tensor of rank-dependent length over the ranks (rank order): a PackedGather of one column."""
    return PackedGather(t.numel(), t.device)(t)


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
    minReplicatesForReplace (the refitted rows' xim would need another collective) or avgTxLength (estimating the
    factors needs a global median): estimate them on one device or pass them.
    test="LRT", reduced=... (passed on to DESeq_device): the LRT columns are per gene, so no collective is added;
    LRTStatistic and LRTPvalue travel in the result gather in place of WaldPvalue (1 + 2p + 2 doubles per gene)."""
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
        colsum, count = DP.nf_column_sums(nf[nz], m)
        mine = torch.cat([colsum, torch.tensor([float(count)], dtype=torch.float64, device=colsum.device)])
        allr = torch.empty(pg.world * (m + 1), dtype=torch.float64, device=mine.device)
        dist.all_gather_into_tensor(allr, mine.contiguous())
        allr = allr.view(pg.world, m + 1)
        pg.collectives += 1
        tot = allr[0].clone()
        for r in range(1, pg.world):                # rank order: the same bits on every rank
            tot = tot + allr[r]
        kw["nfXim"] = DP.nf_xim(tot[:m], tot[m])
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
