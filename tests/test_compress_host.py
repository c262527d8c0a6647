"""CPU checks of the compressor's format layer: zstd-rs_b200/csrc/encode.cuh (the code k_cenc runs on the GPU) compiled for the
host encodes crafted literal and sequence sets into Compressed blocks (tests/seqcraft.py); each is wrapped in a frame and must decode to the
expected bytes with the oracle (ruzstd's decode semantics) and with libzstd, and must be tests/cenc.py's block byte for byte.
Also: compress_bound and the layout of the new C-ABI structs."""
import os
import random
import subprocess

import pytest

import cenc
import datagen
import seqcraft
from conftest import ROOT

pytestmark = pytest.mark.skipif(not os.path.exists(seqcraft.NVCC), reason="nvcc not available")

LL_BASE = [*range(16), 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, *[1 << k for k in range(7, 17)]]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = [*range(3, 35), 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]


def roundtrip(oracle, lits, seqs, history=b""):
    lits = bytes(lits)
    blocks = [("raw", history[i:i + 131072]) for i in range(0, len(history), 131072)] + [("cmp", lits, seqs)]
    expect = seqcraft.execute(blocks)
    assert expect is not seqcraft.ERROR and len(expect) - len(history) <= 131072
    fr, [(huf, modes)] = seqcraft.frame(blocks)
    assert cenc.encode_block(lits, seqs) == tuple(seqcraft.encode(lits, seqs)), "the host build is not the plain model"
    assert oracle.decode_frame(fr)[0] == expect
    assert datagen.decompress(fr, len(expect)) == expect
    return huf, modes


def skewed(rng, n, alphabet):
    return bytes(rng.choice(alphabet) for _ in range(n))


def test_literals_distinct_counts(oracle):
    rng = random.Random(1)
    assert roundtrip(oracle, b"a" * 3000, [])[0] == 0          # one symbol: no Huffman table exists
    assert roundtrip(oracle, b"a" * 700, [])[0] == 0           # <= 1024 literals: Raw
    assert roundtrip(oracle, skewed(rng, 5000, b"ab"), [])[0] == 1
    lits = bytes(rng.choice(range(256)) if rng.random() < 0.3 else rng.choice(b"etaoin ") for _ in range(30000))
    assert len(set(lits)) == 256
    assert roundtrip(oracle, lits, [])[0] == 1
    assert roundtrip(oracle, os.urandom(20000), [])[0] == 0   # Huffman does not pay


def test_literals_rare_symbol_and_length_limit(oracle):
    fib = [1, 1]
    while len(fib) < 21:
        fib.append(fib[-1] + fib[-2])
    lits = bytearray()
    for s, c in enumerate(fib):   # Fibonacci counts: an unlimited Huffman code would be 20 bits deep
        lits += bytes([65 + s]) * c
    random.Random(2).shuffle(lits)
    assert roundtrip(oracle, lits, [])[0] == 1
    lits = bytearray(b"e" * 50000 + b"t" * 30000 + b"\x07")
    random.Random(3).shuffle(lits)
    assert roundtrip(oracle, lits, [])[0] == 1


def test_literals_fse_compressed_weights(oracle):
    rng = random.Random(4)
    lits = bytes(min(255, int(rng.expovariate(1 / 40))) for _ in range(60000))   # symbols up to 255: > 128 weights
    assert max(lits) > 128
    assert roundtrip(oracle, lits, [])[0] == 1


@pytest.mark.parametrize("nseq", [1, 127, 128, 0x7EFF, 0x7F00, 0x7FFF, 0x8000, 40000])
def test_sequence_counts(oracle, nseq):
    rng = random.Random(nseq)
    history = skewed(rng, 1000, b"abcdefgh")
    seqs = [(rng.choice([0, 0, 1]) if nseq < 40000 else 0, 3, rng.randint(1, 1000)) for _ in range(nseq)]
    lits = skewed(rng, sum(q[0] for q in seqs) + 5, b"xyz")
    roundtrip(oracle, lits, seqs, history)


def _values(bases, bits):
    vals = []
    for b, n in zip(bases, bits):
        vals += [b, b + (1 << n) - 1]
    return sorted(set(vals))


def test_every_ll_code_boundary(oracle):
    rng = random.Random(5)
    vals = _values(LL_BASE, LL_BITS)
    groups, cur = [], []
    for v in vals:   # as many values per block as fit
        if sum(cur) + v + 5 * (len(cur) + 1) > 131072:
            groups.append(cur)
            cur = []
        cur.append(v)
    groups.append(cur)
    for g in groups:
        if sum(g) + 4 * len(g) > 131072:
            g = [131072 - 4]
        seqs = [(v, 4, rng.randint(1, 50)) for v in g]
        lits = skewed(rng, sum(g), b"0123456789")
        roundtrip(oracle, lits, seqs, history=b"h" * 64)


def test_every_ml_code_boundary(oracle):
    rng = random.Random(6)
    vals = _values(ML_BASE, ML_BITS)
    groups, cur = [], []
    for v in vals:
        if sum(cur) + v + len(cur) + 1 > 131072:
            groups.append(cur)
            cur = []
        cur.append(v)
    groups.append(cur)
    for g in groups:
        g = [min(v, 131072 - 1) for v in g]
        seqs = [(1, v, rng.randint(1, 64)) for v in g]
        roundtrip(oracle, skewed(rng, len(g), b"xy"), seqs, history=bytes(range(64)))


def test_offsets_up_to_window(oracle):
    rng = random.Random(7)
    history = os.urandom(131072)
    offs = [131072, 131071, 131000, 100000, 65536, 65535, 1 << 15, 4096, 5, 1]
    seqs = [(1, 6, o) for o in offs] + [(2, 5, rng.randint(1, 131072)) for _ in range(500)]
    roundtrip(oracle, skewed(rng, 1600, b"pq"), seqs, history)


def test_single_code_tables_are_rle(oracle):
    seqs = [(0, 4, 5)] * 300
    huf, modes = roundtrip(oracle, b"abcdefgh", seqs, history=b"12345678")
    assert modes == [1, 1, 1]
    seqs = [(0, 4, 5), (3, 40, 900)] * 200
    rng = random.Random(8)
    huf, modes = roundtrip(oracle, skewed(rng, 600, b"abc"), seqs, history=bytes(1000))
    assert modes == [2, 2, 2]


def test_compress_bound_formula(pkg):
    for n in [0, 1, 5, 131071, 131072, 131073, 1 << 20, (1 << 30) + 7]:
        assert pkg.compress_bound(n) == n + 14 + 3 * max(1, -(-n // 131072)) + 4


def test_compress_struct_layouts_match_the_binding(pkg, tmp_path):
    B = pkg.binding
    pairs = {"b200z_compress_io": B.COMPRESS_IO_DTYPE, "b200z_compress_result": B.COMPRESS_RESULT_DTYPE}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200zstd.h"', 'int main(void) {']
    for s, dt in pairs.items():
        lines.append(f'  printf("{s} * %zu 0\\n", sizeof({s}));')
        for f in dt.names:
            lines.append(f'  printf("{s} {f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s} *)0)->{f}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    seen = 0
    for ln in subprocess.check_output([str(exe)]).decode().split("\n"):
        if not ln:
            continue
        s, f, a, b = ln.split()
        dt = pairs[s]
        if f == "*":
            assert dt.itemsize == int(a), s
        else:
            assert dt.fields[f][1] == int(a) and dt.fields[f][0].itemsize == int(b), (s, f)
            seen += 1
    assert seen == sum(len(dt.names) for dt in pairs.values())

