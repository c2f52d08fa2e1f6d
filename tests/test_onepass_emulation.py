"""The one-pass dense GKL kernels (krylovkit.jl_b200/csrc/onepass_kernels.cuh) were written without GPU time, so their
SOURCE is executed here on host threads: tests/emu/onepass_emu.cpp includes the same header nvcc compiles, over
tests/emu/cuda_emu.h (one std::thread per CUDA thread, barriers for __syncthreads, slot exchange for the warp
shuffles, heap buffers for global and dynamic shared memory), with the launch geometries and shared-memory sizes of
the host code in spmv.cu, and checks y = A x, z = A'(A x) against double loops.

  * under AddressSanitizer: every global and shared-memory index of every thread is in range (11 shapes: both
    variants, Float32 / Float64, NZ = 1, 2, 4, 7, ld = 32 mod 64, fewer tiles than CTAs ...);
  * under ThreadSanitizer: no two threads touch a shared-memory word without a barrier between them — removing the
    barrier at the end of the tile loop makes this run fail (tried when the test was written).

  * without a sanitizer (-O2 -ffp-contract=off, the emulator's dump mode): y, the per-CTA partials zpart, the reduced
    dres and z equal oracle/onepass_restate.py bit for bit on the shapes above, on one shape per template instance in
    both types and on grids of more than 32 CTAs (all four running sums of the reduction and its tail); a
    restatement with a sequential warp sum or an in-order sum of the partials differs, so the comparison tells the
    orders apart.  test_gpu_zzz_onepass_restate.py holds the device to the same restatement.

What the emulation cannot see: the inline-PTX streaming loads (replaced by plain loads), performance, and anything
that depends on real warp scheduling."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import onepass_restate as rs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
CSRC = os.path.join(ROOT, "krylovkit.jl_b200", "csrc")


def _build(tmp_path, sanitizer):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    exe = str(tmp_path / f"onepass_emu_{sanitizer}")
    cmd = [gxx, "-std=c++17", "-O1", "-g", f"-fsanitize={sanitizer}", "-fno-omit-frame-pointer", "-Wno-unknown-pragmas",
           "-I", EMU, "-I", CSRC, os.path.join(EMU, "onepass_emu.cpp"), "-o", exe, "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0 and "sanitize" in res.stderr and "cannot find" in res.stderr:
        pytest.skip(f"lib{sanitizer[0]}san not installed")
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def _skip_if_the_sanitizer_cannot_start(res):
    """a sanitizer runtime that cannot set up its shadow memory on this kernel / address-space layout says so before main()
    runs: that is the host's business, not the kernels'"""
    for msg in ("FATAL: ThreadSanitizer", "unexpected memory mapping", "Shadow memory range interleaves",
                "ReserveShadowMemoryRange failed", "failed to allocate", "Resource temporarily unavailable"):   # (pids limit)
        if msg in res.stderr and "ok m=" not in res.stdout:
            pytest.skip("sanitizer runtime cannot start here: " + msg)


def test_kernel_sources_run_clean_under_address_sanitizer(tmp_path):
    exe = _build(tmp_path, "address")
    res = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    _skip_if_the_sanitizer_cannot_start(res)
    assert res.returncode == 0 and "all ok" in res.stdout, res.stdout[-2000:] + res.stderr[-3000:]
    assert res.stdout.count("ok m=") == 11 and "ERROR: AddressSanitizer" not in res.stderr


def test_kernel_sources_have_no_shared_memory_race(tmp_path):
    exe = _build(tmp_path, "thread")
    res = subprocess.run([exe, "1"], capture_output=True, text=True, timeout=900)
    _skip_if_the_sanitizer_cannot_start(res)
    assert res.returncode == 0 and "all ok" in res.stdout, res.stdout[-2000:] + res.stderr[-3000:]
    assert "ThreadSanitizer" not in res.stderr


# (dtype, m, n, grid, variant): the sanitizer shapes, then f64 NZ = 4 and the f64 width limit, and grids past 32 CTAs
DUMP_CASES = [(np.float32, 100, 70, 3, 0), (np.float32, 100, 70, 2, 1), (np.float32, 96, 300, 2, 1),
              (np.float64, 70, 40, 2, 0), (np.float32, 257, 512, 3, 0), (np.float32, 160, 512, 2, 1),
              (np.float32, 33, 600, 1, 0), (np.float32, 64, 1100, 1, 0), (np.float64, 130, 300, 2, 0),
              (np.float32, 4000, 6, 5, 0), (np.float32, 4000, 6, 5, 1),
              (np.float64, 40, 700, 1, 0), (np.float64, 33, 846, 2, 0),
              (np.float32, 4000, 6, 40, 0), (np.float32, 4000, 6, 40, 1), (np.float64, 3000, 9, 45, 0)]


def _case_id(c):
    return f"{np.dtype(c[0]).name}-m{c[1]}-n{c[2]}-g{c[3]}-{'AB'[c[4]]}"


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    """(emulator in dump mode, fma) built without a sanitizer: IEEE arithmetic in program order, no contraction"""
    gxx = shutil.which("g++")
    if gxx is None or shutil.which("gcc") is None:
        pytest.skip("no g++ / gcc")
    d = tmp_path_factory.mktemp("onepass_dump")
    exe = str(d / "onepass_emu_dump")
    cmd = [gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", EMU, "-I", CSRC,
           os.path.join(EMU, "onepass_emu.cpp"), "-o", exe, "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe, rs.load_fma(str(d)), d


def _case_data(dt, m, n):
    rng = np.random.default_rng(1000 * m + n)
    A = (rng.random((m, n)) - 0.5).astype(dt)
    x = (rng.random(n) - 0.5).astype(dt)
    return A, x


def _emulate(dumper, dt, m, n, grid, variant, A, x):
    exe, _, d = dumper
    tag = f"{np.dtype(dt).itemsize}_{variant}_{m}_{n}_{grid}"
    inp, out = d / f"in_{tag}.bin", d / f"out_{tag}.bin"
    with open(inp, "wb") as f:
        f.write(np.array([np.dtype(dt).itemsize, variant], dtype=np.int32).tobytes())
        f.write(np.array([m], dtype=np.int64).tobytes())
        f.write(np.array([n, grid], dtype=np.int32).tobytes())
        f.write(np.asfortranarray(rs.padded(A, rs.ld_of(m))).tobytes(order="F"))
        f.write(x.tobytes())
    res = subprocess.run([exe, "dump", str(inp), str(out)], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    raw = out.read_bytes()
    sizes = [(dt, m), (np.float64, grid * n), (np.float64, n), (dt, n)]
    assert len(raw) == sum(np.dtype(t).itemsize * k for t, k in sizes)
    got, o = [], 0
    for t, k in sizes:
        got.append(np.frombuffer(raw, dtype=t, count=k, offset=o))
        o += np.dtype(t).itemsize * k
    got[1] = got[1].reshape(grid, n)
    return got


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    u = {4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(u), b.view(u))


@pytest.mark.parametrize("case", DUMP_CASES, ids=_case_id)
def test_restatement_equals_the_kernel_source(dumper, case):
    dt, m, n, grid, variant = case
    A, x = _case_data(dt, m, n)
    got = _emulate(dumper, dt, m, n, grid, variant, A, x)
    want = rs.apply_normal_gram(A, x, variant, grid, dumper[1])
    for name, g, w in zip(("y", "zpart", "dres", "z"), got, want):
        assert bits_equal(g, w), (name, np.flatnonzero(np.asarray(g).ravel() != np.asarray(w).ravel())[:10])


@pytest.mark.parametrize("control", ["butterfly", "grouped"])
def test_restatement_tells_the_orders_apart(dumper, control):
    """a restatement with the warp classes summed in sequence, or the partials summed in CTA order, misses the kernel
    source on at least one of the shapes: the comparison above pins the order, not just the value"""
    differs = []
    for dt, m, n, grid, variant in DUMP_CASES:
        A, x = _case_data(dt, m, n)
        got = _emulate(dumper, dt, m, n, grid, variant, A, x)
        want = rs.apply_normal_gram(A, x, variant, grid, dumper[1], **{control: False})
        differs.append(not all(bits_equal(g, w) for g, w in zip(got, want)))
    assert any(differs), control
