"""CPU-only: the C-ABI library loads and exports every symbol include/lhb200.h declares; compute entry
points fail loudly (ENODEV) without a GPU instead of falling back to a CPU path."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "lhb200.h")).read()
    return sorted(set(re.findall(r"LHB200_API[^;(]*?\b(lhb200_[a-z0-9_]+)\s*\(", hdr)))


def test_header_symbols_exported():
    so = os.path.join(ROOT, "lighthouse_b200", "liblhb200.so")
    assert os.path.exists(so), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(so)
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in lhb200.h but not exported"


def test_python_binding_covers_the_header():
    """Every entry point of include/lhb200.h has a typed ctypes signature in lighthouse_b200/_ffi.py (the binding the
    parity tests call through), and every new compute entry point refuses to run without a device."""
    from lighthouse_b200 import _ffi
    for s in declared_symbols():
        f = getattr(_ffi.lib, s)
        assert f.argtypes is not None, f"{s} has no ctypes signature in _ffi.py"
    import torch
    if not torch.cuda.is_available():
        out = ctypes.create_string_buffer(64)
        offs = (ctypes.c_uint64 * 2)(0, 84)
        assert _ffi.lib.lhb200_beacon_block_roots_deneb(b"\0" * 84, ctypes.cast(offs, ctypes.c_void_p), 1, out, None) == _ffi.ENODEV
        arr = (ctypes.c_uint64 * 4)(0, 1, 2, 3)
        assert _ffi.lib.lhb200_shuffle_list(ctypes.cast(arr, ctypes.c_void_p), 4, 90, b"\0" * 32, 0,
                                            ctypes.cast(arr, ctypes.c_void_p)) == _ffi.ENODEV


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lighthouse_b200 import _ffi
    assert _ffi.lib.lhb200_init(0) == _ffi.ENODEV
    out = ctypes.create_string_buffer(32)
    assert _ffi.lib.lhb200_merkleize(b"\0" * 64, 2, 1, out) == _ffi.ENODEV
    assert b"no CPU fallback" in _ffi.lib.lhb200_last_error()


def test_product_does_not_touch_oracle():
    """Nothing under lighthouse_b200/ may import, link or execute oracle/."""
    pkg = os.path.join(ROOT, "lighthouse_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")) or f == "Makefile":
                txt = open(os.path.join(dp, f), errors="replace").read()
                assert "liboracle" not in txt and "oracle_lib" not in txt and "from oracle" not in txt and \
                    "import oracle" not in txt and "oracle/" not in txt.replace("routing through oracle/", ""), \
                    f"{f} references the oracle"


def test_cpp_host_layer_builds_and_fails_loudly_without_gpu():
    """include/lhb200.hpp compiles and links against the C ABI; without a device the program reports ENODEV
    (exit code 2) instead of computing anything on the CPU."""
    import subprocess
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp"), "-s"])
    exe = os.path.join(ROOT, "tests", "cpp", "host_mirror_test")
    assert os.path.exists(exe)
    if not torch.cuda.is_available():
        r = subprocess.run([exe, "/dev/null"], capture_output=True, text=True)
        assert r.returncode == 2 and "no device" in r.stderr


def test_blinding_scalars_come_from_a_csprng_stream():
    """blst.rs:46-68: nonzero 64-bit scalars from a CSPRNG.  The library draws them from a getrandom(2)-keyed ChaCha20
    stream; two draws must differ, no value may be zero, and the bits must be balanced (a broken generator that
    repeats a block or returns a counter fails this)."""
    import ctypes as C
    import numpy as np
    from lighthouse_b200 import _ffi
    n = 1 << 16
    a = np.zeros(n, dtype=np.uint64)
    b = np.zeros(n, dtype=np.uint64)
    assert _ffi.lib.lhb200_debug_rand_scalars(C.c_void_p(a.ctypes.data), n) == 0
    assert _ffi.lib.lhb200_debug_rand_scalars(C.c_void_p(b.ctypes.data), n) == 0
    assert (a != 0).all() and (b != 0).all()
    assert len(np.unique(np.concatenate([a, b]))) == 2 * n
    bits = np.unpackbits(a.view(np.uint8))
    assert abs(bits.mean() - 0.5) < 0.005
    per_bit = np.unpackbits(a.view(np.uint8).reshape(n, 8), axis=1).mean(axis=0)
    assert (abs(per_bit - 0.5) < 0.02).all()


def test_plan_layout_matches_header():
    """Batch.plan() names the words of lhb200_bls_batch_plan in the order of the LHB200_PLAN_* indices and maps the
    LHB200_K_* kernel ids to the right names."""
    from lighthouse_b200 import bls
    hdr = open(os.path.join(ROOT, "include", "lhb200.h")).read()
    words = dict(re.findall(r"#define LHB200_PLAN_([A-Z0-9_]+) (\d+)", hdr))
    n_words = int(words.pop("WORDS"))
    assert n_words == len(bls.PLAN_FIELDS)
    assert sorted(int(v) for v in words.values()) == list(range(n_words))
    for name, v in words.items():
        assert bls.PLAN_FIELDS[int(v)] == name.lower(), name
    kernels = dict(re.findall(r"#define LHB200_K_([A-Z0-9_]+) (\d+)", hdr))
    assert len(kernels) == len(bls.PLAN_KERNELS) - 1
    for name, v in kernels.items():
        assert bls.PLAN_KERNELS[int(v)].replace("+k_pk_", "_").upper() == "K_" + name, name
