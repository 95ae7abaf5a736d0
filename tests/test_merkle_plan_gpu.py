"""GPU tests of tree-hash entry points no other test reaches: lhb200_dev_merkleize (device in, device out, caller's
stream) against the oracle and lhb200_merkleize, and a patch batch refused as a whole because one edit is not
resident."""
import ctypes as C
import struct

import numpy as np
import pytest

from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


# n = 0 (the zero hash of depth), n = 1 at depth 0, the small tree (2..8), reduce passes (> 8), and depths above
# ceil_log2(n) (the zero ladder) for each
@pytest.mark.parametrize("n,depth", [(0, 0), (0, 9), (1, 0), (1, 6), (2, 1), (3, 2), (5, 3), (8, 3), (7, 33),
                                     (9, 4), (9, 12), (1000, 10), (4097, 13), (100_003, 17), (100_003, 40)])
def test_dev_merkleize_vs_oracle(gpu, n, depth):
    import torch
    from lighthouse_b200 import _ffi, tree_hash as T
    chunks = np.random.default_rng(n * 131 + depth).integers(0, 256, 32 * n, dtype=np.uint8).tobytes()
    d_in = torch.frombuffer(bytearray(chunks), dtype=torch.uint8).cuda() if n else None
    d_out = torch.full((32,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    _ffi.check(_ffi.lib.lhb200_dev_merkleize(d_in.data_ptr() if n else None, n, depth, d_out.data_ptr(),
                                             C.c_void_p(stream.cuda_stream)), "lhb200_dev_merkleize")
    got = bytes(d_out.cpu().numpy())
    assert got == O.merkleize(chunks, depth)
    assert got == T.merkleize_chunks(chunks, depth)
    if n == 0:
        assert got == O.zero_hash(depth)


@pytest.mark.parametrize("incremental", [False, True])
def test_patch_batch_with_one_nonresident_edit_is_refused(gpu, incremental):
    """Valid edits around one edit of the validators offset (not resident: part of the offset table): the whole batch
    is refused before anything is modified, so the next root is still the unpatched state's."""
    from lighthouse_b200 import tree_hash as T, Lhb200Error
    from lighthouse_b200.synthetic import beacon_state_deneb_ssz
    ssz = beacon_state_deneb_ssz(3000, seed=21)
    want = O.beacon_state_root_deneb(ssz)[0]
    o_val, o_bal = struct.unpack_from("<II", ssz, 524552)
    st = T.ResidentState(ssz)
    if incremental:
        st.enable_incremental()
    assert st.root() == want
    edits = [(o_val + 121 * 17 + 80, struct.pack("<Q", 31_000_000_000)),   # a validator's effective balance
             (o_bal + 8 * 5, struct.pack("<Q", 123)),                      # a balance
             (40, struct.pack("<Q", 777)),                                 # slot (a literal chunk)
             (524552, b"\0\0\0\0"),                                        # validators offset: not resident
             (524560 + 32 * 3, bytes(range(32)))]                          # a randao mix
    with pytest.raises(Lhb200Error, match="not resident"):
        st.patch_batch(edits)
    assert st.root() == want
    st.release()
