"""CPU-only: the batched field probe (bls/fp_probe.cuh) compiled for the host (tests/hostsim, PTX carries emulated in C)
against Python integers on the crafted corpora of tests/bls_field_spec.py.  This pins the limb algorithms; the same
corpora run on the device in tests/test_bls_field_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import bls_field_spec as F
from tests import oracle_lib as O

HS = os.path.join(O.ROOT, "tests", "hostsim")
N_RANDOM = 300          # per op, after the crafted cases (the device run takes ~10^5)


@pytest.fixture(scope="module")
def L():
    subprocess.check_call(["make", "-C", HS, "-s"])
    return C.CDLL(os.path.join(HS, "libhostsim.so"))


def host_probe(L, name, cases):
    """hs_fp_batch over the cases -> uint32[n, 37]"""
    inp = F.pack(cases)
    out = np.zeros((len(cases), F.OUT_WORDS), dtype=np.uint32)
    assert L.hs_fp_batch(F.OPS[name], C.c_void_p(inp.ctypes.data), len(cases), C.c_void_p(out.ctypes.data)) == 0
    return out


def n_random(name):
    return N_RANDOM // 10 if name in F.COSTLY else N_RANDOM


@pytest.mark.parametrize("name", list(F.OPS))
def test_host_field_probe_matches_big_integers(L, name):
    cases = F.corpus(name, n_random(name))
    out = host_probe(L, name, cases)
    bad = F.mismatches(name, cases, out)
    assert not bad, "\n".join(bad)
    print(f"{name}: {len(cases)} cases")


def test_corpus_reaches_the_edges():
    """the crafted cases contain what they claim: every quotient-word pattern, operands at each op's bound, inputs on
    both sides of p and of (p - 1) / 2"""
    import random
    rnd = random.Random(1)
    for a, b in F.quotient_edge_pairs(rnd):
        assert a < F.P and b < F.P and (a * b) % F.R in (0, F.P)
    assert {(a * b) % F.R for a, b in F.quotient_edge_pairs(rnd)} == {0, F.P}
    lt = [x for (x,) in F.edge_corpus("lt_p", rnd)]
    assert {F.P - 1, F.P, F.P + 1, F.R - 1} <= set(lt)
    gt = [x for (x,) in F.edge_corpus("gt_half", rnd)]
    assert {F.HALF, F.HALF + 1} <= set(gt)
    split = F.edge_corpus("mul_split", rnd)
    assert max(a * b for a, b in split) > F.P * F.R * 0.99 and max(max(c) for c in split) == F.R - 1
    assert max(x for (x,) in F.edge_corpus("sqr_dedicated", rnd)) == F.SQR_MAX
    for k in F.SOP_KS:
        cases = F.sop_edge_corpus(k, rnd)
        for xmax, ymax in F.SOP_BOUNDS[k]:
            assert k * xmax <= 8 * F.P + k and k * xmax * ymax <= 9 * F.P * F.P + k * xmax
            assert any(c[:k] == (xmax - 1,) * k and c[k:2 * k] == (ymax - 1,) * k for c in cases), (k, xmax, ymax)
