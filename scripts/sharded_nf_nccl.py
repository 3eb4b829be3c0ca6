"""Check on 2 GPUs (NCCL; driven by tests/test_norm_factors_device.py): the gene-sharded device pipeline with a
normalization-factor matrix sharded by rows agrees with the single-GPU run within 1e-9 and issues one collective more
than the size-factor run (the xim all-gather).
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29649 \
        scripts/sharded_nf_nccl.py
The same logic runs on CPU in tests/test_norm_factors_device.py (gloo + emulated engine)."""
import os
import sys
import warnings

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deseq2_b200 import device as D, device_pipeline as DP, sharded, synth   # noqa: E402

warnings.simplefilter("ignore")
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
n, m = 20000, 60
x = synth.design_batch_condition(m, 3)
d = synth.make_example_counts(n, m, x=x, seed=5)
eff = np.exp(np.random.default_rng(7).normal(0.0, 0.3, (n, m)))
nf = d["sizeFactors"][None, :] * eff / np.exp(np.log(eff).mean(axis=1))[:, None]
lo, hi = sharded.shard_bounds(n, world, rank)
y = D.to_gene_major(d["counts"][lo:hi], dev)
plain = sharded.sharded_DESeq_device(y, x, d["sizeFactors"])
r = sharded.sharded_DESeq_device(y, x, normalizationFactors=D.to_gene_major(nf[lo:hi], dev))
if rank == 0:
    whole = DP.DESeq_device(D.to_gene_major(d["counts"], dev), x, normalizationFactors=D.to_gene_major(nf, dev))
    err = max(float(((r["gathered"][k] - whole[k]).abs() / whole[k].abs().clamp(min=1e-8)).nan_to_num().max())
              for k in ("dispersion", "betaMatrix", "betaSE", "WaldPvalue"))
    ok = err < 1e-9
    print("sharded ~ whole:", ok, "| max rel err", err, "| genes", int(whole["idx"].numel()),
          "| extra collectives:", int(r["collectives"]) - int(plain["collectives"]))
    assert ok
dist.barrier()
dist.destroy_process_group()
