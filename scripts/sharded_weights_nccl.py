"""Check on 2 GPUs (NCCL; driven by tests/test_weights_device.py): the gene-sharded device pipeline with observation
weights sharded by rows equals the single-GPU run bit for bit and issues the same collectives as without weights.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29647 \
        scripts/sharded_weights_nccl.py
The same logic runs on CPU in tests/test_weights_device.py (gloo + emulated engine)."""
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
rng = np.random.default_rng(7)
w = np.where(rng.random((n, m)) < 0.3, 10.0 ** rng.uniform(-4, -2, (n, m)), rng.uniform(0.5, 1.0, (n, m)))
w[:, 0] = 1.0
w[3, x[:, -1] == 1] = 0.0                                   # one row whose weights leave the design rank deficient
lo, hi = sharded.shard_bounds(n, world, rank)
y = D.to_gene_major(d["counts"][lo:hi], dev)
plain = sharded.sharded_DESeq_device(y, x, d["sizeFactors"])
r = sharded.sharded_DESeq_device(y, x, d["sizeFactors"], weights=D.to_gene_major(w[lo:hi], dev))
if rank == 0:
    whole = DP.DESeq_device(D.to_gene_major(d["counts"], dev), x, d["sizeFactors"],
                            weights=D.to_gene_major(w, dev))
    ok = all(torch.equal(torch.nan_to_num(r["gathered"][k]), torch.nan_to_num(whole[k]))
             for k in ("dispersion", "betaMatrix", "betaSE", "WaldPvalue"))
    print("sharded == whole:", ok, "| genes", int(whole["idx"].numel()), "| weightsFail",
          int(whole["weightsFail"].sum()), "| extra collectives:", int(r["collectives"]) - int(plain["collectives"]))
    assert ok
dist.barrier()
dist.destroy_process_group()
