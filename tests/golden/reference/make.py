"""Record tests/golden/reference/outputs.npz: the outputs of the reference's own src/DESeq2.cpp on the inputs of the
tests that compare with it (tests/test_oracle_vs_reference.py, tests/test_parity_reference_gpu.py and the emulated
cases of tests/test_emulated_kernels.py), kept at a seeded sample of genes (tests/helpers.py, StoredReference).

Needs oracle/_ref/libdeseq2_ref.so (oracle/Makefile `ref`).  The GPU tests are recorded through the SIMT-emulated
engine, so no GPU is needed.  Run from the repo root:  python tests/golden/reference/make.py
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))


def main():
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build_emu
    out = os.path.join(HERE, "outputs.npz")
    if os.path.exists(out):
        os.remove(out)
    env = dict(os.environ, DESEQ2_RECORD_REFERENCE="1")
    pytest = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider"]
    subprocess.check_call(pytest + ["tests/test_oracle_vs_reference.py"], cwd=ROOT, env=env)
    subprocess.check_call(pytest + ["tests/test_emulated_kernels.py", "-k", "reference"], cwd=ROOT, env=env)
    env["B200NB_LIB"] = build_emu.build()
    subprocess.check_call(pytest + ["-m", "gpu", "tests/test_parity_reference_gpu.py"], cwd=ROOT, env=env)


if __name__ == "__main__":
    main()
