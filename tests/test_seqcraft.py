"""CPU checks of the crafted sequence sets (tests/seqcraft.py) the GPU tests decode: every case agrees three ways -- the plain
LZ77 reference, the oracle (whose trace must hold exactly the requested sequences) and, for spec-valid cases, libzstd -- and
error cases fail in the oracle.  The Compressed blocks then go through the bit-level model of k_exec_cta
(tests/emul_exec_cta.py) at 128-byte aligned frame addresses, the alignment the GPU tests use."""
import os

import pytest

import datagen
import emul_exec_cta as E
import seqcraft as S

pytestmark = pytest.mark.skipif(not os.path.exists(S.NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def crafted():
    return {g: S.cases(g) for g in S.GROUPS}


@pytest.mark.parametrize("group", list(S.GROUPS))
def test_three_way_agreement(oracle, crafted, group):
    for c in crafted[group]:
        got, err = S.oracle_decode(oracle, c.frame, c.blocks, c.ov)
        if c.valid:
            assert err is None and got == c.expected, (c, err)
            assert datagen.decompress(c.frame, len(c.expected)) == c.expected, c
        else:
            assert err is not None, (c, "the oracle decoded an invalid case")


@pytest.mark.parametrize("group", list(S.GROUPS))
def test_exec_cta_model(oracle, crafted, group):
    nblk = 0
    for c in crafted[group]:
        if c.valid:
            nblk += E.run_frame(oracle, c.frame, base=0, strict=True)[0]
    assert nblk >= sum(1 for c in crafted[group] if c.valid)


def test_groups_cover_their_constants(crafted):
    """The cases sit where their groups say: sequence counts around the batch constants, every overlap length at every
    residue mod 32 and in every quarter of a 128-byte row, the wide sequences' extra bits around the fast path's limit."""
    counts = {len(c.blocks[0][2]) for c in crafted["geometry"]}
    for k in (S.EXEC_BATCH, S.FSE_PUBLISH, S.XC_BATCH):
        assert {k - 1, k, k + 1} <= counts
    assert {c.xbits for c in crafted["fse"] if c.valid} == {32, 33, S.FSE_FAST_XBITS, S.FSE_FAST_XBITS + 1}
    for c in crafted["overlap"]:
        pos, res32, res128 = 0, set(), set()
        for ll, ml, _ in c.blocks[0][2]:
            res32.add((ml, (pos + ll) % 32))
            res128.add((ml, (pos + ll) % 128 // 32))
            pos += ll + ml
        assert res32 == {(ml, r) for ml in S.OVERLAP_LENGTHS for r in range(32)}, c
        assert res128 == {(ml, q) for ml in S.OVERLAP_LENGTHS for q in range(4)}, c
    assert any("of=window" in c.id for c in crafted["earlier"])
    short = [c for c in crafted["earlier"] if c.id.endswith("-inside-window")]
    assert len(short) == 2 and all(c.cap <= 1 << c.window_log for c in short)
    assert sum(not c.valid for g in crafted.values() for c in g) >= 6


def test_reference_repeat_offsets():
    """The reference's repeat-offset rules on their own: ll > 0 keeps / swaps, ll == 0 shifts by one, rep0 - 1 saturates."""
    h = [17, 9, 13]
    assert S.offset_history(1, 5, h) == 17 and h == [17, 9, 13]
    assert S.offset_history(2, 5, h) == 9 and h == [9, 17, 13]
    assert S.offset_history(3, 5, h) == 13 and h == [13, 9, 17]
    assert S.offset_history(1, 0, h) == 9 and h == [9, 13, 17]
    assert S.offset_history(2, 0, h) == 17 and h == [17, 9, 13]
    assert S.offset_history(3, 0, h) == 16 and h == [16, 17, 9]
    h = [1, 4, 8]
    assert S.offset_history(3, 0, h) == 0 and h == [0, 1, 4]
    assert S.offset_history(3, 0, h) == 0 and h == [0, 0, 1]
    assert S.offset_history(7, 0, h) == 4 and h == [4, 0, 0]
