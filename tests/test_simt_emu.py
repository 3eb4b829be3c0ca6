"""Known-answer tests of the SIMT emulator itself (tests/simt_emu/): before the emulated engine is trusted as a CPU
check of the product kernels (tests/test_emulated_kernels.py), the emulator's warp collectives, barriers, shared
memory, atomics, poison values and its two bug detectors are pinned here on small kernels written as ordinary CUDA
(tests/simt_emu/selftest_kernels.cu)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "simt_emu"))


@pytest.fixture(scope="module")
def st():
    import build_emu
    return C.CDLL(build_emu.build_selftest())


def _p(a):
    return C.c_void_p(a.ctypes.data)


def test_warp_collectives(st):
    blocks, threads = 3, 96
    sums = np.zeros(blocks * threads // 32)
    misc = np.zeros((blocks * threads, 8), dtype=np.int32)
    assert st.st_warp_collectives(_p(sums), _p(misc), blocks, threads) == 0
    t = np.arange(threads)
    lane = t % 32
    want = np.array([(t[w * 32:(w + 1) * 32] + 1).sum() for w in range(threads // 32)] * blocks, dtype=float)
    assert np.array_equal(sums, want)
    m = misc.reshape(blocks, threads, 8)
    for b in range(blocks):
        assert np.array_equal(m[b, :, 0], np.full(threads, 50))
        assert np.array_equal(m[b, :, 1], np.where(lane + 3 < 32, lane + 3, lane))
        assert np.array_equal(m[b, :, 2], np.where(lane - 2 >= 0, lane - 2, lane))
        assert np.array_equal(m[b, :, 3], lane ^ 1)
        assert np.all(m[b, :, 4].astype(np.uint32) == sum(1 << l for l in range(32) if l % 3 == 0))
        assert np.all(m[b, :, 5] == 1)                      # any(lane == 31) is true, all(lane < 31) is false
        assert np.array_equal(m[b, :, 6], (lane & ~3) | 3)
        assert np.array_equal(m[b, :, 7], np.where((lane % 16) + 1 < 16, lane + 1, lane))


def test_syncthreads_static_and_dynamic_shared(st):
    n = 700
    a = np.arange(n, dtype=np.int32) * 3 + 1
    out = np.full(n, -5, dtype=np.int32)
    assert st.st_cta_reverse(_p(a), _p(out), n) == 0
    pad = np.full(768, -1, dtype=np.int32)
    pad[:n] = a
    want = (2 * pad.reshape(3, 256)[:, ::-1]).reshape(-1)[:n]
    assert np.array_equal(out, want)


def test_atomic_work_queue(st):
    n = 57
    counter = np.zeros(1, dtype=np.uint32)
    owners = np.zeros(2, dtype=np.int32)
    out = np.zeros(n)
    assert st.st_queue(_p(counter), n, _p(owners), _p(out), 2, 64) == 0
    assert np.array_equal(out, (np.arange(n) + 1) * 528.0)
    assert owners.sum() == n and counter[0] == n + 4      # every warp (2 CTAs x 2 warps) overshoots once


def test_missing_syncwarp_is_not_hidden_by_lock_step(st):
    """Lanes do not advance in lock step in the emulator, so a read of another lane's shared-memory write without a
    barrier returns stale data (the bug is visible); with the barrier the result is right."""
    good = np.zeros(32, dtype=np.int32)
    bad = np.zeros(32, dtype=np.int32)
    assert st.st_missing_syncwarp(_p(good), 1) == 0
    assert st.st_missing_syncwarp(_p(bad), 0) == 0
    assert np.array_equal(good, (np.arange(32) + 1) % 32)
    assert not np.array_equal(bad, good) and (bad == -1).sum() >= 30


def test_uninitialised_shared_memory_is_poisoned(st):
    out = np.zeros(64)
    assert st.st_uninitialised_smem(_p(out)) == 0
    assert np.all(np.isnan(out))


def test_divergent_collective_is_reported_as_deadlock(st):
    code = ("import ctypes, numpy as np; l = ctypes.CDLL(%r); o = np.zeros(32, dtype=np.int32); "
            "l.st_divergent_collective(ctypes.c_void_p(o.ctypes.data))" % st._name)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0
    assert "deadlock" in r.stderr and "warp collective" in r.stderr and "__syncthreads" in r.stderr


# sm_90: 48 KB of dynamic shared memory without an opt-in, 232448 bytes (227 KB) at most with one
@pytest.mark.parametrize("bytes_, attr, ok", [
    (48 * 1024, 0, True),              # the default limit, no attribute
    (48 * 1024 + 8, 0, False),         # above it without cudaFuncSetAttribute
    (100 * 1024, 99 * 1024, False),    # above the limit the attribute set
    (232448, 232448, True),            # at the opt-in maximum
    (232448 + 8, 232448, False),       # above it
])
def test_dynamic_shared_memory_limits(st, bytes_, attr, ok):
    """The emulator refuses a launch the H100 refuses, so that a launch plan that only fits on the emulator fails on
    the CPU too; the refused kernel does not run."""
    ran = np.zeros(1, dtype=np.int32)
    rc = st.st_smem_limit(_p(ran), bytes_, attr)
    assert (rc == 0) == ok and ran[0] == int(ok)
    assert st.st_smem_limit(_p(ran), 1024, 0) == 0     # a refusal is not sticky: the next launch runs


def test_shared_memory_attribute_above_the_maximum_is_refused(st):
    ran = np.zeros(1, dtype=np.int32)
    assert st.st_smem_limit(_p(ran), 1024, 232448 + 8) != 0 and ran[0] == 0


@pytest.mark.parametrize("order", ["reverse", "random:7"])
def test_lane_order_is_configurable(st, order):
    """SIMT_EMU_ORDER changes which lane runs first between barriers: correct kernels do not care, the kernel with the
    missing __syncwarp returns a different wrong answer (read in a fresh process: the order is fixed at load time)."""
    code = ("import ctypes, numpy as np, json; l = ctypes.CDLL(%r); "
            "g = np.zeros(32, dtype=np.int32); b = np.zeros(32, dtype=np.int32); "
            "l.st_missing_syncwarp(ctypes.c_void_p(g.ctypes.data), 1); l.st_missing_syncwarp(ctypes.c_void_p(b.ctypes.data), 0); "
            "s = np.zeros(9); m = np.zeros((288, 8), dtype=np.int32); "
            "l.st_warp_collectives(ctypes.c_void_p(s.ctypes.data), ctypes.c_void_p(m.ctypes.data), 3, 96); "
            "print(json.dumps([g.tolist(), b.tolist(), s.tolist()]))" % st._name)
    import json
    outs = {}
    for o in ("forward", order):
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=60,
                           env=dict(os.environ, SIMT_EMU_ORDER=o))
        assert r.returncode == 0, r.stderr
        outs[o] = json.loads(r.stdout)
    good = [(i + 1) % 32 for i in range(32)]
    assert outs["forward"][0] == good and outs[order][0] == good           # with the barrier: right under any order
    assert outs["forward"][2] == outs[order][2]                            # collectives do not depend on the order
    assert outs["forward"][1] != good and outs[order][1] != good           # without it: wrong under both ...
    assert outs["forward"][1] != outs[order][1]                            # ... and differently wrong
