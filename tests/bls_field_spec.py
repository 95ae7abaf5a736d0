"""Big-integer reference and seeded corpora for the batched base-field probe (bls/fp_probe.cuh): the device runs it
through lhb200_debug_fp_batch, the host build through hs_fp_batch, and tests compare both with what this module
computes from Python integers.

Every operand and result is a raw 12-limb value (little-endian 32-bit words), in Montgomery form where the operation
assumes it: `mul` of raw a, b is a b / R mod p, `sqrt` of raw a is the Montgomery form of (a / R)^((p + 1) / 4).  The
corpora aim at the values where carry and borrow chains go wrong, which random operands almost never reach: powers of
two and their neighbours at every bit, p - 2^i, p +- small values, all-ones and alternating limbs, operands whose
Montgomery quotient words are all 0 or all 0xffffffff, and the largest operands each operation's bounds allow.
"""
import math
import random

import numpy as np

from oracle import bls_ref as B

P = B.P
R = 1 << 384
RINV = pow(R, -1, P)
HALF = (P - 1) // 2
M32 = 0xFFFFFFFF
NL = 12
OUT_WORDS = 3 * NL + 1
FLAG = 3 * NL
SEED = 0xF1E1D

OPS = {
    "add": 0, "sub": 1, "neg": 2, "mul": 3, "sqr": 4, "to_mont": 5, "from_mont": 6, "inv": 7, "inv_vartime": 8,
    "sqrt": 9, "lt_p": 10, "gt_half": 11, "mul_split": 12, "sqr_dedicated": 13,
    "fp2_mul": 14, "fp2_sqr": 15, "fp2_inv": 16, "fp2_sqrt": 17, "fp2_sgn0": 18,
}
SOP_KS = (1, 2, 4, 6, 8)
for _k in SOP_KS:
    OPS[f"sop{_k}"] = 32 + _k
ARITY = {"neg": 1, "sqr": 1, "to_mont": 1, "from_mont": 1, "inv": 1, "inv_vartime": 1, "sqrt": 1, "lt_p": 1,
         "gt_half": 1, "sqr_dedicated": 1, "add": 2, "sub": 2, "mul": 2, "mul_split": 2, "fp2_sqr": 2, "fp2_inv": 2,
         "fp2_sqrt": 2, "fp2_sgn0": 2, "fp2_mul": 4}
for _k in SOP_KS:
    ARITY[f"sop{_k}"] = 4 * _k
# ops whose corpus is costly to evaluate per case (exponentiation chains): fewer random cases
COSTLY = {"inv", "inv_vartime", "sqrt", "fp2_inv", "fp2_sqrt"}

# (K, x bound, y bound) of the fused sums of products: the call sites' (K = 2, X = 1 + 1/p, Y = 1) and (K, X = 2, Y = 1)
# and the header's general limits K X <= 8, K X Y <= 9 (sop.cuh)
SOP_BOUNDS = {1: [(2 * P, P), (8 * P, 9 * P // 8)], 2: [(P + 1, P), (2 * P, P), (4 * P, 9 * P // 8)],
              4: [(2 * P, P), (2 * P, 9 * P // 8)], 6: [(P + 1, P), (4 * P // 3, 9 * P // 8)],
              8: [(P + 1, P), (P + 1, 9 * P // 8)]}
SQR_MAX = math.isqrt(P * R - 1)           # fp_sqr_inl needs a a < p R


def mont(x): return x * R % P
def unmont(x): return x * RINV % P


# ------------------------------------------------------------------------------------------------ expected values
def expected(name, ops):
    """-> (r0, r1, r2, flag) for one case; None where the result is checked by `check` instead (square roots)."""
    a = ops[0]
    b = ops[1] if len(ops) > 1 else 0
    if name == "add": return (a + b) % P, 0, 0, 0
    if name == "sub": return (a - b) % P, 0, 0, 0
    if name == "neg": return -a % P, 0, 0, 0
    if name in ("mul", "mul_split"): return a * b * RINV % P, 0, 0, 0
    if name in ("sqr", "sqr_dedicated"): return a * a * RINV % P, 0, 0, 0
    if name == "to_mont": return a * R % P, 0, 0, 0
    if name == "from_mont": return a * RINV % P, 0, 0, 0
    if name in ("inv", "inv_vartime"):
        return (mont(pow(unmont(a), -1, P)) if a % P else 0), 0, 0, 0
    if name == "sqrt":
        r = pow(unmont(a), (P + 1) // 4, P)
        return mont(r), 0, 0, int(r * r % P == unmont(a))
    if name == "lt_p": return 0, 0, 0, int(a < P)
    if name == "gt_half": return 0, 0, 0, int(a > HALF)
    if name in ("fp2_mul", "fp2_sqr"):
        x = (a, b)
        y = (ops[2], ops[3]) if name == "fp2_mul" else x
        return (x[0] * y[0] - x[1] * y[1]) * RINV % P, (x[0] * y[1] + x[1] * y[0]) * RINV % P, 0, 0
    if name == "fp2_inv":
        x = (unmont(a), unmont(b))
        if x == (0, 0):
            return 0, 0, 0, 0
        r = B.f2_inv(x)
        return mont(r[0]), mont(r[1]), 0, 0
    if name == "fp2_sqrt":
        return None
    if name == "fp2_sgn0": return 0, 0, 0, B.f2_sgn0((unmont(a), unmont(b)))
    if name.startswith("sop"):
        k = int(name[3:])
        xa, ya, xb, yb = ops[:k], ops[k:2 * k], ops[2 * k:3 * k], ops[3 * k:]
        ra = sum(x * y for x, y in zip(xa, ya)) * RINV % P
        rb = sum(x * y for x, y in zip(xb, yb)) * RINV % P
        return ra, rb, ra, 0
    raise KeyError(name)


def fp2_is_square(x):
    """Fp2 = Fp[i], i^2 = -1, p = 3 mod 4: x is a square iff its norm x0^2 + x1^2 is a square in Fp"""
    n = (x[0] * x[0] + x[1] * x[1]) % P
    return n == 0 or pow(n, (P - 1) // 2, P) == 1


def check(name, ops, got):
    """got = (r0, r1, r2, flag) of one case -> None, or a description of the mismatch"""
    if name == "fp2_sqrt":
        x = (unmont(ops[0]), unmont(ops[1]))
        want = int(fp2_is_square(x))
        if got[3] != want:
            return f"flag {got[3]} != {want}"
        if want and B.f2_sqr((unmont(got[0]), unmont(got[1]))) != x:
            return "root squared != input"
        if got[0] >= P or got[1] >= P:
            return "root not canonical"
        return None
    want = expected(name, ops)
    if tuple(got) != tuple(want):
        return "got " + ", ".join(hex(v) for v in got) + " want " + ", ".join(hex(v) for v in want)
    return None


# ------------------------------------------------------------------------------------------------ corpora
def _bit_edges(lim):
    """2^i, 2^i - 1, p - 2^i, p + 2^i for every i < 384, kept below `lim`"""
    out = []
    for i in range(384):
        out += [1 << i, (1 << i) - 1, P - (1 << i), P + (1 << i)]
    return [v for v in out if 0 <= v < lim]


def _limb_patterns():
    return [R - 1, int("aaaaaaaa" * 12, 16), int("55555555" * 12, 16), int("ffffffff00000000" * 6, 16),
            int("00000000ffffffff" * 6, 16), int("80000000" * 12, 16), int("00000001" * 12, 16)]


def canonical_edges():
    """the host tests' edge values, the bit edges reduced mod p, p - small, limb patterns mod p; sorted, distinct"""
    v = [0, 1, 2, P - 1, P - 2, HALF, HALF + 1, (1 << 380) % P, 2 ** 32 - 1, 2 ** 64 - 1, 2 ** 352]
    v += list(range(9)) + [P - k for k in range(1, 9)] + [HALF - 1, HALF + 2]
    v += [x % P for x in _bit_edges(R)]
    v += [x % P for x in _limb_patterns()]
    v += [P - x % P for x in _limb_patterns()]
    v += [(P & ~M32) | w for w in (0, 1, M32)]                   # p with its low limb replaced
    v += [P - (1 << (32 * k)) for k in range(12)] + [(P + (1 << (32 * k))) % P for k in range(12)]
    return sorted(set(x % P for x in v))


def any_edges():
    """384-bit values around p, (p - 1) / 2 and the limb boundaries (the comparisons take any 384-bit input)"""
    v = _bit_edges(R) + _limb_patterns() + [0, P - 1, P, P + 1, HALF - 1, HALF, HALF + 1, HALF + 2, 2 * P, R - P]
    v += [P + d for d in range(-8, 9)] + [HALF + d for d in range(-8, 9)]
    for k in range(12):
        v += [P - (1 << (32 * k)), P + (1 << (32 * k)), HALF - (1 << (32 * k)), HALF + (1 << (32 * k))]
    v += [(P | ((1 << (32 * k)) - 1)) for k in range(1, 12)]      # p with its low limbs all ones
    return sorted(set(x for x in v if 0 <= x < R))


def quotient_edge_pairs(rnd, n=48):
    """canonical (a, b) with a b = 0 mod R (every Montgomery quotient word 0) and with a b = p mod R (every quotient word
    0xffffffff)"""
    out = [(1 << i, 1 << (384 - i)) for i in range(4, 381)]
    while len(out) < 377 + n:
        b = rnd.randrange(1, P) | 1
        a = P * pow(b, -1, R) % R
        if a < P:
            out.append((a, b))
    return out


def _pairs(edges, rnd, lim):
    out = []
    for e in edges:
        out += [(e, e), (e, P - 1), (P - 1, e), (e, 1), (e, rnd.randrange(lim)), (rnd.randrange(lim), e)]
    return out


def edge_corpus(name, rnd):
    """the crafted cases of one op: a list of operand tuples"""
    ce = canonical_edges()
    if name in ("lt_p", "gt_half"):
        return [(x,) for x in any_edges()]
    if name == "sqr_dedicated":
        v = [x for x in _bit_edges(SQR_MAX + 1) + _limb_patterns() if x <= SQR_MAX] + ce
        v += [SQR_MAX, SQR_MAX - 1, 2 * P - 1, 3 * P - 1, 3 * P, (1 << 382) - 1, 1 << 192, (1 << 192) - 1]
        return [(x,) for x in sorted(set(v))]
    if name == "mul_split":
        out = [(a, b) for a, b in _pairs(ce, rnd, P)] + quotient_edge_pairs(rnd)
        out += [(R - 1, 0), (R - 1, 1), (R - 1, 2), (R - 1, P - 1), (P, 1), (1, P), (2 * P - 1, 2 * P - 1),
                (SQR_MAX, SQR_MAX), (P, R - 1 - (R - 1) % 1)]
        for k in range(1, 12):                                   # a = k p - 1 with the largest b allowed
            a = k * P - 1
            out += [(a, (P * R - 1) // a), (a, P - 1), ((P * R - 1) // a, a)]
        for e in _bit_edges(R):
            if e:
                out.append((e, min(R - 1, (P * R - 1) // e)))
        return [(a, b) for a, b in out if a < R and b < R and a * b < P * R]
    if name.startswith("sop"):
        return sop_edge_corpus(int(name[3:]), rnd)
    ar = ARITY[name]
    if ar == 1:
        v = ce + [a for a, _ in quotient_edge_pairs(rnd, 16)]
        return [(x,) for x in v]
    if ar == 2 and not name.startswith("fp2"):
        return _pairs(ce, rnd, P) + quotient_edge_pairs(rnd)
    if name == "fp2_mul":
        out = [(a, b, c, d) for (a, b), (c, d) in zip(_pairs(ce, rnd, P), _pairs(ce[::-1], rnd, P))]
        out += [(a, 0, b, 0) for a, b in quotient_edge_pairs(rnd)] + [(0, a, 0, b) for a, b in quotient_edge_pairs(rnd)]
        return out
    # unary Fp2 ops take (c0, c1)
    out = _pairs(ce, rnd, P) + [(x, 0) for x in ce] + [(0, x) for x in ce]
    if name == "fp2_sqrt":                                       # squares, so the root branch runs for edge values too
        out += [(mont(s[0]), mont(s[1])) for s in (B.f2_sqr((unmont(a), unmont(b))) for a, b in out[:400])]
    return out


def sop_edge_corpus(k, rnd):
    out = []
    for xmax, ymax in SOP_BOUNDS[k]:
        top_x, top_y = xmax - 1, ymax - 1
        out += [([top_x] * k, [top_y] * k, [top_x] * k, [top_y] * k),
                ([top_x] * k, [0] * k, [0] * k, [top_y] * k),
                ([0] * k, [0] * k, [1] * k, [1] * k),
                ([P] * k, [top_y] * k, [P - 1] * k, [P - 1] * k),
                ([top_x] * k, [P - 1] * k, [P] * k, [top_y] * k)]
        for e in _bit_edges(min(xmax, ymax)) + _limb_patterns():
            if e < min(xmax, ymax):
                out.append(([e] * k, [top_y] * k, [top_x] * k, [e] * k))
        for a, b in quotient_edge_pairs(rnd, 8)[::16]:           # quotient words 0 / all ones in the first product
            out.append(([a] + [0] * (k - 1), [b] + [0] * (k - 1), [b] * k, [a] * k))
    return [tuple(xa + ya + xb + yb) for xa, ya, xb, yb in out]


def random_corpus(name, rnd, n):
    if name in ("lt_p", "gt_half"):   # half of them close to p or (p - 1) / 2
        return [(rnd.randrange(R) if i % 2 else rnd.choice((P, HALF)) + rnd.randrange(-(1 << 64), 1 << 64),)
                for i in range(n)]
    if name == "sqr_dedicated":
        return [(rnd.randrange(SQR_MAX + 1),) for _ in range(n)]
    if name == "mul_split":
        out = []
        for _ in range(n):
            a = rnd.randrange(1, R)
            out.append((a, rnd.randrange((P * R - 1) // a + 1 if a * (R - 1) >= P * R else R)))
        return out
    if name.startswith("sop"):
        k = int(name[3:])
        out = []
        for i in range(n):
            xmax, ymax = SOP_BOUNDS[k][i % len(SOP_BOUNDS[k])]
            out.append(tuple([rnd.randrange(xmax) for _ in range(k)] + [rnd.randrange(ymax) for _ in range(k)] +
                             [rnd.randrange(xmax) for _ in range(k)] + [rnd.randrange(ymax) for _ in range(k)]))
        return out
    return [tuple(rnd.randrange(P) for _ in range(ARITY[name])) for _ in range(n)]


def corpus(name, n_random):
    """edge cases then n_random random cases of one op (seeded: the same list on every run)"""
    rnd = random.Random(SEED * 1000 + OPS[name])
    return edge_corpus(name, rnd) + random_corpus(name, rnd, n_random)


# ------------------------------------------------------------------------------------------------ limb packing
def pack(cases):
    """operand tuples -> uint32[n, 12 * arity] of little-endian limbs"""
    w = len(cases[0])
    b = b"".join(v.to_bytes(48, "little") for c in cases for v in c)
    return np.frombuffer(b, dtype="<u4").reshape(len(cases), NL * w).copy()


def unpack(out):
    """uint32[n, 37] probe results -> list of (r0, r1, r2, flag)"""
    raw = np.ascontiguousarray(out, dtype="<u4").tobytes()
    res = []
    for i in range(out.shape[0]):
        row = raw[4 * OUT_WORDS * i:4 * OUT_WORDS * (i + 1)]
        res.append((int.from_bytes(row[0:48], "little"), int.from_bytes(row[48:96], "little"),
                    int.from_bytes(row[96:144], "little"), int.from_bytes(row[144:148], "little")))
    return res


def mismatches(name, cases, out, limit=5):
    """-> the first `limit` failing cases as strings (empty when every case matches the reference)"""
    bad = []
    for ops, got in zip(cases, unpack(out)):
        msg = check(name, ops, got)
        if msg:
            bad.append(f"{name}({', '.join(hex(v) for v in ops[:4])}{', ...' if len(ops) > 4 else ''}): {msg}")
            if len(bad) >= limit:
                break
    return bad
