"""Check on 2 GPUs (NCCL; driven by tests/test_beta_prior_device.py): the gene-sharded device pipeline with
betaPrior=TRUE equals the single-GPU run bit for bit and costs exactly one more collective than without the prior.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29643 \
        scripts/sharded_beta_prior_nccl.py
The same logic runs on CPU in tests/test_beta_prior_device.py (gloo + emulated engine)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deseq2_b200 import device as D, device_pipeline as DP, pipeline, sharded, synth   # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
n, m = 20000, 60
factors = [(np.arange(m) * 6) // m]
x = pipeline.factorDesign(factors)[0]
d = synth.make_example_counts(n, m, x=x, seed=5)
lo, hi = sharded.shard_bounds(n, world, rank)
y = D.to_gene_major(d["counts"][lo:hi], dev)
plain = sharded.sharded_DESeq_device(y, x, d["sizeFactors"])
r = sharded.sharded_DESeq_device(y, x, d["sizeFactors"], betaPrior=True, factors=factors)
if rank == 0:
    whole = DP.DESeq_device(D.to_gene_major(d["counts"], dev), x, d["sizeFactors"], betaPrior=True, factors=factors)
    ok = (np.array_equal(r["betaPriorVar"], whole["betaPriorVar"])
          and all(torch.equal(torch.nan_to_num(r["gathered"][k]), torch.nan_to_num(whole[k]))
                  for k in ("betaMatrix", "betaSE", "WaldPvalue")))
    print("sharded == whole:", ok, "| genes", int(whole["idx"].numel()), "| extra collectives:",
          int(r["collectives"]) - int(plain["collectives"]))
    assert ok
dist.barrier()
dist.destroy_process_group()
