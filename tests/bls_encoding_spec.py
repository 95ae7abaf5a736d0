"""Reference decoder for BLS12-381 point encodings: the ZCash serialisation rules as blst applies them behind Lighthouse
(crypto/bls/src/impls/blst.rs), the status each library entry point must report, and a seeded corpus of encodings at
the edges of those rules.

blst entry points and what they accept:
  * 48-byte keys, `PublicKey::deserialize` -> key_validate: compressed only (c flag set), x < p, on the curve, not
    infinity, in the r-order subgroup.
  * 96-byte keys, `deserialize_uncompressed` -> blst P1 deserialize through the Rust wrapper: the c flag must be clear;
    an infinity encoding (0x40 then zeros) is the point at infinity; the s flag is not allowed; x < p, y < p, on the
    curve.  No subgroup check.
  * 96-byte signatures, `Signature::from_bytes`: compressed only, x.c1 < p and x.c0 < p, on the curve, no subgroup
    check (verification checks the subgroup).  Lighthouse maps all-zero bytes to the "empty" signature first.

A compressed infinity encoding must be 0xc0 followed by zeros: the s flag or any other bit makes it malformed.
"""
import functools
import random

from oracle import bls_ref as B

P = B.P
SEED = 0xE1C0DE

# blst outcomes (BLST_ERROR names), plus the point at infinity and Lighthouse's empty signature
OK, INFINITY, BAD_ENCODING, NOT_ON_CURVE, NOT_IN_GROUP, EMPTY = (
    "ok", "infinity", "bad_encoding", "not_on_curve", "not_in_group", "empty")


def _be(x, n=48): return x.to_bytes(n, "big")


# ------------------------------------------------------------------------------------------------ decoders
def decode_g1_compressed(b):
    """48 bytes -> (outcome, point); outcome in OK, INFINITY, BAD_ENCODING, NOT_ON_CURVE"""
    assert len(b) == 48
    c, inf, s = b[0] >> 7 & 1, b[0] >> 6 & 1, b[0] >> 5 & 1
    if not c:
        return BAD_ENCODING, None
    if inf:
        return (INFINITY if b[0] == 0xC0 and not any(b[1:]) else BAD_ENCODING), None
    x = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:], "big")
    if x >= P:
        return BAD_ENCODING, None
    y = B.fp_sqrt((x ** 3 + B.B1) % P)
    if y is None:
        return NOT_ON_CURVE, None
    if (y > (P - 1) // 2) != bool(s):
        y = P - y
    return OK, (x, y)


def decode_g1_uncompressed(b):
    """96 bytes -> (outcome, point); outcome in OK, INFINITY, BAD_ENCODING, NOT_ON_CURVE"""
    assert len(b) == 96
    if b[0] & 0x80:
        return BAD_ENCODING, None
    if b[0] & 0x40:
        return (INFINITY if b[0] == 0x40 and not any(b[1:]) else BAD_ENCODING), None
    if b[0] & 0x20:
        return BAD_ENCODING, None
    x, y = int.from_bytes(b[:48], "big"), int.from_bytes(b[48:], "big")
    if x >= P or y >= P:
        return BAD_ENCODING, None
    if (y * y - x ** 3 - B.B1) % P:
        return NOT_ON_CURVE, None
    return OK, (x, y)


def decode_g2_compressed(b):
    """96 bytes (x.c1 || x.c0) -> (outcome, point); outcome in OK, INFINITY, BAD_ENCODING, NOT_ON_CURVE"""
    assert len(b) == 96
    c, inf, s = b[0] >> 7 & 1, b[0] >> 6 & 1, b[0] >> 5 & 1
    if not c:
        return BAD_ENCODING, None
    if inf:
        return (INFINITY if b[0] == 0xC0 and not any(b[1:]) else BAD_ENCODING), None
    x1 = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:48], "big")
    x0 = int.from_bytes(b[48:], "big")
    if x0 >= P or x1 >= P:
        return BAD_ENCODING, None
    x = (x0, x1)
    y = B.f2_sqrt(B.f2_add(B.f2_mul(B.f2_sqr(x), x), B.B2))
    if y is None:
        return NOT_ON_CURVE, None
    big = (y[1] > (P - 1) // 2) if y[1] else (y[0] > (P - 1) // 2)
    if big != bool(s):
        y = B.f2_neg(y)
    return OK, (x, y)


@functools.lru_cache(maxsize=None)
def _g1_in_group(x): return B.g1_in_subgroup((x, B.fp_sqrt((x ** 3 + B.B1) % P)))


@functools.lru_cache(maxsize=None)
def _g2_in_group(x): return B.g2_in_subgroup((x, B.f2_sqrt(B.f2_add(B.f2_mul(B.f2_sqr(x), x), B.B2))))


# ------------------------------------------------------------------------------------------------ per-API statuses
def key_validate(b48):
    """PublicKey::deserialize of 48 bytes: OK, INFINITY, BAD_ENCODING, NOT_ON_CURVE or NOT_IN_GROUP"""
    out, pt = decode_g1_compressed(b48)
    if out == OK and not _g1_in_group(pt[0]):
        return NOT_IN_GROUP
    return out


def signature_outcome(b96):
    """Signature::from_bytes plus the subgroup check verification applies: EMPTY, OK, INFINITY, BAD_ENCODING,
    NOT_ON_CURVE or NOT_IN_GROUP"""
    if not any(b96):
        return EMPTY
    out, pt = decode_g2_compressed(b96)
    if out == OK and not _g2_in_group(pt[0]):
        return NOT_IN_GROUP
    return out


# the device statuses each entry point reports for an outcome
G1_DECOMPRESS_VALIDATE = {OK: 0, INFINITY: 1, BAD_ENCODING: 2, NOT_ON_CURVE: 2, NOT_IN_GROUP: 3}   # lhb200_g1_decompress_validate
G1_DESERIALIZE_UNCOMPRESSED = {OK: 0, INFINITY: 1, BAD_ENCODING: 2, NOT_ON_CURVE: 2}            # lhb200_g1_deserialize_uncompressed
G2_DECOMPRESS = {OK: 0, NOT_IN_GROUP: 0, INFINITY: 1, BAD_ENCODING: 2, NOT_ON_CURVE: 2, EMPTY: 2}  # lhb200_g2_decompress rc
# SET_* of a batch set whose keys are valid (bls/kernels.cuh): the signature's status
SET_SIG = {EMPTY: 1, BAD_ENCODING: 2, NOT_ON_CURVE: 2, NOT_IN_GROUP: 3, OK: 0, INFINITY: 0}
SET_PK_DECODE, SET_APK_INFINITY = 6, 5


def table_append_refused(b96):
    """PubkeyTable.append refuses the whole call unless every key is a finite point on the curve"""
    return decode_g1_uncompressed(b96)[0] != OK


def g1_aggregate_refused(b96):
    """lhb200_g1_aggregate fails (EDECODE) on a malformed or off-curve key; infinity is the identity"""
    return decode_g1_uncompressed(b96)[0] in (BAD_ENCODING, NOT_ON_CURVE)


def g2_aggregate_refused(b96):
    """lhb200_g2_aggregate fails (EDECODE) on a malformed or off-curve signature (all-zero bytes included: the empty
    signature is filtered by the caller, generic_aggregate_signature.rs:124-136)"""
    return G2_DECOMPRESS[signature_outcome(b96)] == 2


def batch_key_outcome(b96):
    """the batch key kernels take keys a PublicKey already validated: they apply the encoding rules only (flags,
    infinity, x < p, y < p), not the curve equation.  -> OK, INFINITY or BAD_ENCODING"""
    out, _ = decode_g1_uncompressed(b96)
    return OK if out == NOT_ON_CURVE else out


def batch_key_set_status(keys96):
    """SET_* of a set with a valid signature and these keys (in order)"""
    outs = [batch_key_outcome(k) for k in keys96]
    if not outs:
        return 4
    if BAD_ENCODING in outs:
        return SET_PK_DECODE
    if all(o == INFINITY for o in outs):
        return SET_APK_INFINITY
    return 0


# ------------------------------------------------------------------------------------------------ corpus
def _set_flags(b, flags):
    return bytes([(b[0] & 0x1F) | flags]) + b[1:]


def _with_coord(b, off, v):
    """replace the 381-bit coordinate at byte offset `off` (keeping byte 0's flag bits when off == 0)"""
    raw = bytearray(b)
    raw[off:off + 48] = _be(v)
    if off == 0:
        raw[0] = (raw[0] & 0x1F) | (b[0] & 0xE0)
    return bytes(raw)


def _stray_bits(inf, n):
    """the canonical infinity encoding with one extra bit at each byte position"""
    out = []
    for k in range(n):
        raw = bytearray(inf)
        raw[k] |= (0x01 << (k % 5)) if k else 0x10
        out.append((f"inf_stray_byte{k}", bytes(raw)))
    return out


def _g1_bases(rnd):
    """subgroup points, curve points outside the subgroup, x values off the curve"""
    sub = [B.sk_to_pk(k) for k in (1, 2, rnd.randrange(1, B.R))]
    off_group, off_curve = [], []
    x = rnd.randrange(P)
    while len(off_group) < 2 or len(off_curve) < 2:
        y = B.fp_sqrt((x ** 3 + B.B1) % P)
        if y is None and len(off_curve) < 2:
            off_curve.append(x)
        elif y is not None and len(off_group) < 2 and not B.g1_in_subgroup((x, y)):
            off_group.append((x, y))
        x += 1
    return sub, off_group, off_curve


def _edge_xs():
    """canonical coordinates with carry-heavy limbs and non-canonical ones at p"""
    return [("x_p_minus_1", P - 1), ("x_all_ones_380", (1 << 380) - 1), ("x_limbs_ffffffff", int("ffffffff" * 11, 16)),
            ("x_eq_p", P), ("x_p_plus_1", P + 1), ("x_2^381-1", (1 << 381) - 1), ("x_zero", 0)]


def g1_compressed_corpus(seed=SEED):
    """[(name, 48 bytes)]"""
    rnd = random.Random(seed)
    sub, off_group, off_curve = _g1_bases(rnd)
    out = []
    bases = [(f"sub{i}", B.g1_compress(p)) for i, p in enumerate(sub)]
    bases += [(f"nosub{i}", B.g1_compress(p)) for i, p in enumerate(off_group)]
    bases += [(f"offcurve{i}", bytes([0x80 | _be(x)[0]]) + _be(x)[1:]) for i, x in enumerate(off_curve)]
    for name, b in bases:
        out += [(f"{name}_flags{f:03b}", _set_flags(b, f << 5)) for f in range(8)]
        x = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:], "big")
        if x + P < 1 << 381:
            out.append((f"{name}_x_plus_p", _with_coord(b, 0, x + P)))
    for name, x in _edge_xs():
        for s in (0x80, 0xA0):
            out.append((f"{name}_s{s >> 5 & 1}", _set_flags(_be(x), s)))
    inf = bytes([0xC0]) + bytes(47)
    out += [("inf", inf), ("inf_with_s", bytes([0xE0]) + bytes(47)), ("inf_without_c", bytes([0x40]) + bytes(47)),
            ("all_zero", bytes(48))]
    out += _stray_bits(inf, 48)
    return out


def g1_uncompressed_corpus(seed=SEED):
    """[(name, 96 bytes)]"""
    rnd = random.Random(seed + 1)
    sub, off_group, off_curve = _g1_bases(rnd)
    out = []
    pts = [(f"sub{i}", p) for i, p in enumerate(sub)] + [(f"nosub{i}", p) for i, p in enumerate(off_group)]
    pts += [(f"offcurve{i}", (x, rnd.randrange(P))) for i, x in enumerate(off_curve)]
    for name, (x, y) in pts:
        b = _be(x) + _be(y)
        out += [(f"{name}_flags{f:03b}", _set_flags(b, f << 5)) for f in range(8)]
        out += [(f"{name}_neg", _be(x) + _be((P - y) % P)), (f"{name}_y_plus_p", _be(x) + _be(y + P)),
                (f"{name}_y_plus_1", _be(x) + _be((y + 1) % P)), (f"{name}_y_minus_1", _be(x) + _be((y - 1) % P))]
        if x + P < 1 << 381:
            out.append((f"{name}_x_plus_p", _be(x + P) + _be(y)))
        out += [(f"{name}_y_eq_p", _be(x) + _be(P)), (f"{name}_y_2^384-1", _be(x) + _be((1 << 384) - 1))]
    for name, x in _edge_xs():
        if x < P:   # on-curve points at carry-heavy x where they exist, else the x with y = 0
            y = B.fp_sqrt((x ** 3 + B.B1) % P)
            out.append((name + "_point", _be(x) + _be(y or 0)))
        else:
            out.append((name, _be(x) + _be(sub[0][1])))
    inf = bytes([0x40]) + bytes(95)
    out += [("inf", inf), ("inf_with_s", bytes([0x60]) + bytes(95)), ("inf_with_c", bytes([0xC0]) + bytes(95)),
            ("all_zero", bytes(96))]
    out += _stray_bits(inf, 96)
    return out


def g2_compressed_corpus(seed=SEED):
    """[(name, 96 bytes)]: subgroup signatures (the golden deposit signatures), curve points outside the subgroup,
    x off the curve, and their flag / alias / infinity variants"""
    import json
    import os
    rnd = random.Random(seed + 2)
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "deposit_data.json")))
    sub = [bytes.fromhex(d["signature"].removeprefix("0x")) for d in gold[:2]]
    off_group, off_curve = [], []
    x = (rnd.randrange(P), rnd.randrange(P))
    while len(off_group) < 2 or len(off_curve) < 2:
        y = B.f2_sqrt(B.f2_add(B.f2_mul(B.f2_sqr(x), x), B.B2))
        if y is None and len(off_curve) < 2:
            off_curve.append(x)
        elif y is not None and len(off_group) < 2 and not B.g2_in_subgroup((x, y)):
            off_group.append((x, y))
        x = (x[0] + 1, x[1])
    bases = [(f"sub{i}", b) for i, b in enumerate(sub)]
    bases += [(f"nosub{i}", B.g2_compress(p)) for i, p in enumerate(off_group)]
    bases += [(f"offcurve{i}", _set_flags(_be(x[1]) + _be(x[0]), 0x80)) for i, x in enumerate(off_curve)]
    out = []
    for name, b in bases:
        out += [(f"{name}_flags{f:03b}", _set_flags(b, f << 5)) for f in range(8)]
        x1 = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:48], "big")
        x0 = int.from_bytes(b[48:], "big")
        if x1 + P < 1 << 381:
            out.append((f"{name}_c1_plus_p", _with_coord(b, 0, x1 + P)))
        out += [(f"{name}_c0_plus_p", _with_coord(b, 48, x0 + P)), (f"{name}_c0_eq_p", _with_coord(b, 48, P)),
                (f"{name}_c1_eq_p", _with_coord(b, 0, P)), (f"{name}_c0_p_plus_1", _with_coord(b, 48, P + 1)),
                (f"{name}_c1_2^381-1", _with_coord(b, 0, (1 << 381) - 1)),
                (f"{name}_c0_2^381-1", _with_coord(b, 48, (1 << 381) - 1))]
    for name, v in _edge_xs():
        for s in (0x80, 0xA0):
            out.append((f"c1_{name}_s{s >> 5 & 1}", _set_flags(_be(v) + bytes(48), s)))
            out.append((f"c0_{name}_s{s >> 5 & 1}", _set_flags(bytes(47) + b"\x01" + _be(v), s)))
    inf = bytes([0xC0]) + bytes(95)
    out += [("inf", inf), ("inf_with_s", bytes([0xE0]) + bytes(95)), ("inf_without_c", bytes([0x40]) + bytes(95)),
            ("all_zero", bytes(96))]
    out += _stray_bits(inf, 96)
    return out


@functools.lru_cache(maxsize=None)
def corpora():
    """{"g1c": [(name, bytes, outcome)], "g1u": ..., "g2c": ...} with key_validate / the 96-byte key decoder /
    signature_outcome as the outcome"""
    return {
        "g1c": [(n, b, key_validate(b)) for n, b in g1_compressed_corpus()],
        "g1u": [(n, b, decode_g1_uncompressed(b)[0]) for n, b in g1_uncompressed_corpus()],
        "g2c": [(n, b, signature_outcome(b)) for n, b in g2_compressed_corpus()],
    }


def class_sizes():
    """{kind: {outcome: count}}"""
    out = {}
    for kind, items in corpora().items():
        d = {}
        for _, _, o in items:
            d[o] = d.get(o, 0) + 1
        out[kind] = d
    return out
