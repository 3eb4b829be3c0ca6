"""Check on 2 GPUs (NCCL; driven by tests/test_lrt_device.py): the gene-sharded DESeq_device(test="LRT") equals the
single-GPU run bit for bit and issues the same collectives as the Wald run.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29651 \
        scripts/sharded_lrt_nccl.py
The same logic runs on CPU in tests/test_lrt_device.py (gloo + emulated engine)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deseq2_b200 import device as D, device_pipeline as DP, sharded, synth   # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
n, m = 20000, 60
x = synth.design_batch_condition(m, 3)
xr = x[:, :3]
d = synth.make_example_counts(n, m, x=x, seed=5)
lo, hi = sharded.shard_bounds(n, world, rank)
y = D.to_gene_major(d["counts"][lo:hi], dev)
wald = sharded.sharded_DESeq_device(y, x, d["sizeFactors"])
r = sharded.sharded_DESeq_device(y, x, d["sizeFactors"], test="LRT", reduced=xr)
if rank == 0:
    whole = DP.DESeq_device(D.to_gene_major(d["counts"], dev), x, d["sizeFactors"], test="LRT", reduced=xr)
    ok = all(torch.equal(torch.nan_to_num(r["gathered"][k]), torch.nan_to_num(whole[k]))
             for k in ("dispersion", "betaMatrix", "betaSE", "LRTStatistic", "LRTPvalue"))
    print("sharded == whole:", ok, "| genes", int(whole["idx"].numel()), "| extra collectives:",
          int(r["collectives"]) - int(wald["collectives"]))
    assert ok
dist.barrier()
dist.destroy_process_group()
