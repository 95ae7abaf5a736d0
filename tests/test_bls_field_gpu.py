"""GPU: the base-field arithmetic run alone on the device, one thread per case (lhb200_debug_fp_batch over
bls/fp_probe.cuh), against Python integers and against the host build of the same source.

On the device every carry chain is a run of separate `asm volatile` statements that relies on ptxas keeping the carry
flag intact between them; the host build emulates the flag with a variable.  So each case must give device == host ==
big integers: where only the device disagrees, the fault is in code generation or carry handling, not in the limb
algorithm.  The corpora (tests/bls_field_spec.py) put the crafted carry and borrow edges first, then ~10^5 random
cases per op.
"""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

from tests import bls_field_spec as F
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu

HS = os.path.join(O.ROOT, "tests", "hostsim")
HOST_RANDOM = 1000       # random cases per op that the host build also runs (it is ~10^4 times slower)


def n_random(name):
    if name in F.COSTLY:
        return 20000
    if name.startswith("sop") and int(name[3:]) >= 4:
        return 30000
    return 100000


@pytest.fixture(scope="module")
def host():
    subprocess.check_call(["make", "-C", HS, "-s"])
    return C.CDLL(os.path.join(HS, "libhostsim.so"))


def device_probe(name, inp):
    from lighthouse_b200 import _ffi
    out = np.zeros((inp.shape[0], F.OUT_WORDS), dtype=np.uint32)
    _ffi.check(_ffi.lib.lhb200_debug_fp_batch(F.OPS[name], inp.ctypes.data, inp.shape[1], inp.shape[0],
                                              out.ctypes.data, F.OUT_WORDS), "lhb200_debug_fp_batch")
    return out


def test_probe_rejects_a_wrong_layout(gpu):
    from lighthouse_b200 import _ffi
    inp = np.zeros((4, 24), dtype=np.uint32)
    out = np.zeros((4, F.OUT_WORDS), dtype=np.uint32)
    assert _ffi.lib.lhb200_debug_fp_batch(F.OPS["neg"], inp.ctypes.data, 24, 4, out.ctypes.data, F.OUT_WORDS) == _ffi.EINVAL
    assert _ffi.lib.lhb200_debug_fp_batch(99, inp.ctypes.data, 24, 4, out.ctypes.data, F.OUT_WORDS) == _ffi.EINVAL


@pytest.mark.parametrize("name", list(F.OPS))
def test_device_field_op_matches_host_and_big_integers(gpu, host, name):
    t0 = time.perf_counter()
    cases = F.corpus(name, n_random(name))
    inp = F.pack(cases)
    dev = device_probe(name, inp)
    n_edge = len(cases) - n_random(name)
    n_host = n_edge + HOST_RANDOM
    hs = np.zeros((n_host, F.OUT_WORDS), dtype=np.uint32)
    assert host.hs_fp_batch(F.OPS[name], C.c_void_p(inp.ctypes.data), n_host, C.c_void_p(hs.ctypes.data)) == 0
    diff = np.nonzero((dev[:n_host] != hs).any(axis=1))[0]
    assert not len(diff), (f"{name}: device != host build at {len(diff)} cases, first "
                           f"{[hex(v) for v in cases[diff[0]][:4]]}: the device's carry handling or code generation")
    bad = F.mismatches(name, cases, dev)
    assert not bad, "\n".join(bad)
    print(f"{name}: {len(cases)} cases ({n_edge} crafted), {n_host} also on the host, {time.perf_counter() - t0:.1f} s")
