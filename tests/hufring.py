"""Crafted literal sections at the edges of k_huf's narrow bit-reader ring (HufRingNarrow in csrc/kernels.cu): 8 groups of 8 bytes per
stream, filled 7 groups ahead, with an 8-byte mirror of the top group below slot 0.  Four equal streams of flat 7-bit codes
(k symbols make a stream of ceil((7k + 1) / 8) bytes) whose length is a whole ring or one byte off it, a ring plus its mirror
or one byte more, and streams whose last byte sits at every residue mod 8 of the group that holds it."""
import random

import entcraft as E

FLAT = E.Huf({s: 7 for s in range(128)})
RING_BYTES = (63, 64, 65, 72, 73)
END_RESIDUE_BYTES = tuple(range(200, 208))   # with a fixed stream start, eight lengths in a row end at every residue mod 8


def symbols_for(nbytes):
    """Symbols per stream that make a stream of exactly `nbytes` bytes of 7-bit codes."""
    return (8 * nbytes - 1) // 7


def _block(rng, nbytes):
    return E.Blk(bytes(rng.randrange(128) for _ in range(4 * symbols_for(nbytes))), huf=FLAT)


def cases():
    rng = random.Random(0x8A6)
    out = [E.Case("huf-ring", f"stream-bytes{n}", [_block(rng, n)]) for n in RING_BYTES]
    out += [E.Case("huf-ring", f"stream-end-bytes{n}", [_block(rng, n)]) for n in END_RESIDUE_BYTES]
    return out


def stream_sizes(c):
    """Byte sizes of the four streams of case `c`'s literal section."""
    pay = E.lit_payload(FLAT.table, c.blocks[0].lits, 4)
    sizes = list(E.struct.unpack("<3H", pay[:6]))
    return sizes + [len(pay) - 6 - sum(sizes)]


def stream_offsets(c):
    """Offsets of the four streams in case `c`'s frame (the frame itself starts 16-byte aligned in the GPU tests' input)."""
    pay = E.lit_payload(FLAT.table, c.blocks[0].lits, 4)
    start = c.frame.index(pay) + 6
    sizes = stream_sizes(c)
    return [start + sum(sizes[:j]) for j in range(4)]
