"""deseq2_b200 -- H100-native (sm_90a) batched negative-binomial GLM engine behind DESeq2's native boundary.

Scope: the ONE hot path of thelovelab/DESeq2 -- fitDisp / fitDispGrid / fitBeta
(the reference's src/DESeq2.cpp:164,469,283) -- as hand-written sm_90a kernels in
`csrc/`, exported through the C ABI in `include/b200nb.h` (libb200nb.so), plus the host-side
mirror of the reference's R callers needed to drive and measure it:

  wrappers.py   fitDisp / fitDispGrid / fitBeta + the *Wrapper functions (R/wrappers.R, R/RcppExports.R)
  device.py     the same three calls on device-resident torch tensors (gene-major layout)
  device_pipeline.py  the whole Wald / LRT analysis device-resident: size factors, pre-steps, trend fit, Cook's distances,
                outlier replacement + refit and getContrast as kernels / tensor glue around the three calls; vst(),
                varianceStabilizingTransformation() and normTransform() (R/vst.R) with one transform kernel
  pipeline.py   host glue of DESeq()'s Wald path that feeds/consumes the kernels (R/core.R, R/fitNbinomGLMs.R)
  synth.py      makeExampleDESeqDataSet-style synthetic counts (R/core.R:459-498)
  sharded.py    gene-sharded multi-GPU drivers, host glue and device-resident (R/parallel.R:6-74 is the blueprint)

There is no CPU fallback: importing works without a GPU (so the CPU test-suite can check the ABI),
but every compute call fails loudly if libb200nb.so or a CUDA device is missing.
"""
from ._lib import lib, lib_path, build, EngineError  # noqa: F401

__all__ = ["lib", "lib_path", "build", "EngineError"]
