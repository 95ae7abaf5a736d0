"""CPU-only: the encoding reference (tests/bls_encoding_spec.py) on golden data, and its corpus through the host build
of the device decoders (tests/hostsim): g1_decompress, g1_from_uncompressed + the on-curve check, g2_decompress."""
import ctypes as C
import json
import os
import subprocess

import pytest

from oracle import bls_ref as B
from tests import bls_encoding_spec as S
from tests import oracle_lib as O

HS = os.path.join(O.ROOT, "tests", "hostsim")
DEC = {S.OK: 0, S.NOT_IN_GROUP: 0, S.INFINITY: 1, S.BAD_ENCODING: 2, S.NOT_ON_CURVE: 2, S.EMPTY: 2}   # DecodeStatus


@pytest.fixture(scope="module")
def L():
    subprocess.check_call(["make", "-C", HS, "-s"])
    return C.CDLL(os.path.join(HS, "libhostsim.so"))


def _hex(s): return bytes.fromhex(s.removeprefix("0x"))


def test_reference_accepts_golden_keys_and_signatures():
    keys = [_hex(k["pubkey"]) for k in json.load(open(os.path.join(O.GOLDEN, "interop_keypairs.json")))]
    deposits = json.load(open(os.path.join(O.GOLDEN, "deposit_data.json")))
    keys += [_hex(d["pubkey"]) for d in deposits]
    for k in keys:
        assert S.key_validate(k) == S.OK, k.hex()
        out, pt = S.decode_g1_compressed(k)
        assert B.g1_compress(pt) == k
        assert S.decode_g1_uncompressed(B.g1_uncompressed(pt)) == (S.OK, pt)
    for d in deposits:
        sig = _hex(d["signature"])
        assert S.signature_outcome(sig) == S.OK
        assert B.g2_compress(S.decode_g2_compressed(sig)[1]) == sig


def test_reference_round_trips_and_agrees_with_the_oracle_decoders():
    """every accepted corpus encoding re-encodes to itself; bls_ref's decoders accept exactly what the reference
    accepts"""
    c = S.corpora()
    for name, b, out in c["g1c"]:
        ok, pt = S.decode_g1_compressed(b)
        try:
            ref = B.g1_decompress(b)
            accepted = True
        except ValueError:
            accepted = False
        assert accepted == (ok in (S.OK, S.INFINITY)), name
        if accepted:
            assert ref == pt and B.g1_compress(pt) == b, name
    for name, b, out in c["g1u"]:
        ok, pt = S.decode_g1_uncompressed(b)
        if ok in (S.OK, S.INFINITY):
            assert B.g1_uncompressed(pt) == b, name
    for name, b, out in c["g2c"]:
        ok, pt = S.decode_g2_compressed(b)
        try:
            ref = B.g2_decompress(b)
            accepted = True
        except ValueError:
            accepted = False
        assert accepted == (ok in (S.OK, S.INFINITY)), name
        if accepted:
            assert ref == pt and B.g2_compress(pt) == b, name


def test_corpus_covers_every_status_class():
    sizes = S.class_sizes()
    print("corpus sizes by outcome:", json.dumps(sizes, sort_keys=True))
    assert set(sizes["g1c"]) == {S.OK, S.INFINITY, S.BAD_ENCODING, S.NOT_ON_CURVE, S.NOT_IN_GROUP}
    assert set(sizes["g1u"]) == {S.OK, S.INFINITY, S.BAD_ENCODING, S.NOT_ON_CURVE}
    assert set(sizes["g2c"]) == {S.EMPTY, S.OK, S.INFINITY, S.BAD_ENCODING, S.NOT_ON_CURVE, S.NOT_IN_GROUP}
    assert [n for n, _ in S.g2_compressed_corpus()] == [n for n, _, _ in S.corpora()["g2c"]]   # seeded
    for kind in ("g1c", "g1u", "g2c"):
        names = [n for n, _, _ in S.corpora()[kind]]
        assert len(names) == len(set(names)), kind
    by_name = {n: o for n, _, o in S.corpora()["g2c"]}
    # the named edges the decoders must hold: non-canonical c1 or c0 alone, infinity with the s flag
    assert by_name["sub0_c1_plus_p"] == by_name["sub0_c0_plus_p"] == S.BAD_ENCODING
    assert by_name["inf_with_s"] == S.BAD_ENCODING and by_name["all_zero"] == S.EMPTY


def test_host_decoders_match_the_reference(L):
    c = S.corpora()
    o96 = C.create_string_buffer(96)
    for name, b, out in c["g1c"]:
        rc = L.hs_g1_decompress(b, o96)
        assert rc == DEC[out], (name, rc, out)
        if rc == 0:
            assert o96.raw == B.g1_uncompressed(S.decode_g1_compressed(b)[1]), name
            assert L.hs_g1_subgroup(b) == (out == S.OK), name
    for name, b, out in c["g1u"]:
        rc = L.hs_g1_from_uncompressed(b, o96)
        assert rc == DEC[out], (name, rc, out)
        if rc != 2:
            assert o96.raw == b, name
    for name, b, out in c["g2c"]:
        rc = L.hs_g2_roundtrip(b, o96)
        assert rc == DEC[out], (name, rc, out)
        if rc != 2:
            assert o96.raw == b, name
