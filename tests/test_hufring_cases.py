"""CPU checks of the crafted literal sections at the edges of k_huf's bit-reader ring (tests/hufring.py): every case decodes to
the requested literals in the oracle and in libzstd, and the streams have the sizes and end residues their ids claim."""
import os

import pytest

import datagen
import entcraft as E
import hufring as H

pytestmark = pytest.mark.skipif(not os.path.exists(E.S.NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def crafted():
    return H.cases()


def test_three_way_agreement(oracle, crafted):
    for c in crafted:
        got, err = E.oracle_decode(oracle, c)
        assert c.valid and err is None and got == c.expected, (c, err)
        assert datagen.decompress(c.frame, len(c.expected)) == c.expected, c


def test_cases_sit_on_the_ring_edges(crafted):
    for c in crafted:
        n = int(c.id.rsplit("bytes", 1)[1])
        assert H.stream_sizes(c) == [n] * 4, c
    ends = {(H.stream_offsets(c)[0] + H.stream_sizes(c)[0]) % 8 for c in crafted if "stream-end" in c.id}
    assert ends == set(range(8))   # where stream 0 ends, with the frame 16-byte aligned
    assert {n for c in crafted for n in H.stream_sizes(c)} >= set(H.RING_BYTES)
