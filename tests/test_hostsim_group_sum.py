"""CPU-only: the per-message key sum of grouped batches (bls/group_sum.cuh, k_g1_group_sum) compiled for the host
(tests/hostsim/group_sum_sim.cpp, built into a temporary directory) and run position by position, level by level,
against G1 sums of oracle/bls_ref.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import bls_ref as B
from tests import oracle_lib as O

SRC = os.path.join(O.ROOT, "tests", "hostsim", "group_sum_sim.cpp")


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("group_sum_sim") / "libgroupsum.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-shared",
                           "-o", so, SRC])
    return C.CDLL(so)


def group_sum(L, points, status, groups):
    """points: affine G1 tuples per set; groups: lists of set indices -> (levels, [(sum or None, skip)])"""
    n, ng = len(points), len(groups)
    p96 = b"".join(B.g1_uncompressed(p) for p in points)
    members = np.array([i for g in groups for i in g], dtype=np.uint32)
    offsets = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.uint32)
    st = np.array(status, dtype=np.uint8)
    out = C.create_string_buffer(96 * ng)
    skip = np.zeros(ng, dtype=np.uint8)
    levels = L.hs_group_sum(p96, C.c_void_p(st.ctypes.data), C.c_void_p(members.ctypes.data),
                            C.c_void_p(offsets.ctypes.data), n, ng, out, C.c_void_p(skip.ctypes.data))
    assert levels > 0
    res = []
    for g in range(ng):
        b = out.raw[96 * g:96 * g + 96]
        res.append((None if skip[g] else (int.from_bytes(b[:48], "big"), int.from_bytes(b[48:], "big")), int(skip[g])))
    return levels, res


def oracle_sum(points, status, group):
    acc = None
    for i in group:
        if status[i] == 0:
            acc = B.g1_add(acc, points[i])
    return acc


def check(L, points, status, groups):
    levels, res = group_sum(L, points, status, groups)
    for g, (got, skip) in zip(groups, res):
        want = oracle_sum(points, status, g)
        assert skip == (want is None), g
        assert got == want, g
    return levels, res


def pts(*sks):
    return [B.sk_to_pk(s) for s in sks]


def test_special_cases(L):
    P, Q, R = pts(3, 5, 7)
    points = [P, Q, P, P, B.g1_neg(P), P, Q, B.g1_neg(B.g1_add(P, Q)), P, Q, R, R, Q]
    status = [0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 0, 2, 6]
    groups = [[0, 1],            # P + Q
              [2, 3],            # P + P (the doubling branch)
              [4, 5],            # P + (-P) = O: skipped
              [6, 7, 8] + [],    # Q + (-(P + Q)) + P = O: skipped
              [9, 10],           # Q skipped by its status: R alone
              [11, 12]]          # every member skipped
    _, res = check(L, points, status, groups)
    assert [s for _, s in res] == [0, 0, 1, 1, 0, 1]
    assert res[0][0] == B.g1_add(P, Q) and res[1][0] == B.g1_add(P, P) and res[4][0] == R


def test_tree_levels(L):
    """groups of 1, 8, 9, 64, 65 and 70 members interleaved in set order, random skips: 1 to 3 tree levels, sums equal
    the oracle's; the level count follows the largest group"""
    rnd = random.Random(5)
    sizes = [1, 8, 9, 64, 65, 70]
    n = sum(sizes)
    base = pts(*range(11, 11 + 24))
    points = [base[rnd.randrange(len(base))] for _ in range(n)]
    status = [rnd.choice([0, 0, 0, 0, 1, 5]) for _ in range(n)]
    order = list(range(n))
    rnd.shuffle(order)
    groups, k = [], 0
    for s in sizes:
        groups.append(sorted(order[k:k + s]))
        k += s
    levels, _ = check(L, points, status, groups)
    assert levels == 3
    levels, _ = check(L, points, status, groups[:3])
    assert levels == 2
    levels, _ = check(L, points, status, groups[:2])
    assert levels == 1
