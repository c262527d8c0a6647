"""encode_block with a formatted dictionary's tables, on the host (tests/host/encode_dict_test.cpp, no GPU): crafted literal and
sequence sets against a crafted dictionary, each block wrapped in a frame that carries the dictionary's ID, must decode to the
plain LZ77 result (seqcraft.execute) with the oracle and with libzstd, and be tests/cenc.py's block byte for byte.  Covered: the
three literal choices (Raw, own Huffman, Treeless with 1 and 4 streams), a literal byte the dictionary's Huffman table lacks, and
each sequence table as Repeat / Compressed / RLE, including a code the dictionary's FSE table lacks."""
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import cenc
import datagen
import entcraft
import seqcraft

pytestmark = pytest.mark.skipif(not os.path.exists(seqcraft.NVCC), reason="nvcc not available")

DICT_ID = 4242
# Huffman codes for 8 letters only (Kraft-complete); LL codes 0-15 only; OF codes 0-7, mostly 2-7; ML codes 0-31
LENGTHS = {ord("e"): 2, ord("t"): 2, ord("a"): 3, ord("o"): 3, ord("i"): 4, ord("n"): 4, ord("s"): 4, ord("r"): 4}
LL_NORM = (6, [4] * 16)
OF_NORM = (5, [1, 1] + [5] * 6)
ML_NORM = (6, [2] * 32)


@pytest.fixture(scope="module")
def tool():
    d = tempfile.mkdtemp(prefix="encdict")
    exe = os.path.join(d, "encode_dict_test")
    subprocess.check_call([seqcraft.NVCC, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe,
                           os.path.join(seqcraft.HERE, "host", "encode_dict_test.cpp")])
    content = datagen.gen_text(5000, 0xD1).tobytes()
    raw, _ = entcraft.dictionary(DICT_ID, entcraft.Huf(LENGTHS), OF_NORM, ML_NORM, LL_NORM, (1, 4, 8), content)
    path = os.path.join(d, "dict")
    open(path, "wb").write(raw)
    yield exe, path, raw, d
    shutil.rmtree(d, True)


def encode(tool, lits, seqs):
    exe, dpath, _, d = tool
    src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<I", len(lits)) + bytes(lits) + struct.pack("<I", len(seqs)) +
                b"".join(struct.pack("<3I", ll, ml, of) for ll, ml, of in seqs))
    out = subprocess.run([exe, dpath, src, dst], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr
    f = out.stdout.split()
    return open(dst, "rb").read(), int(f[2]), [int(x) for x in f[3:6]]


def round_trip(oracle, tool, lits, seqs):
    """Encodes one first block, frames it with the dictionary's ID, and checks both decoders; returns (literals mode, modes)."""
    content, lit_mode, modes = encode(tool, lits, seqs)
    assert cenc.encode_block(lits, seqs, cenc.Tables(tool[2])) == (content, lit_mode, modes), "the host build is not the plain model"
    plain = seqcraft.execute([("cmp", bytes(lits), seqs)])
    assert plain is not seqcraft.ERROR
    hdr = struct.pack("<IBBII", 0xFD2FB528, (2 << 6) | 3, (17 - 10) << 3, DICT_ID, len(plain))
    frame = hdr + struct.pack("<I", 1 | (2 << 1) | (len(content) << 3))[:3] + content
    raw = tool[2]
    d = oracle.FrameDecoder()
    d.add_dict(raw)
    r = d.reset(frame)
    d.decode_blocks(r)
    assert d.collect() == plain
    assert datagen.decompress(frame, len(plain), raw_dict=raw) == plain
    return lit_mode, modes


def letters(rng, n, weights):
    syms, w = zip(*weights.items())
    return bytes(rng.choices(syms, w, k=n))


DICT_DIST = {s: 2.0 ** -n for s, n in LENGTHS.items()}


def seqs_for(rng, nlit, n, ll=range(16), ml=range(3, 35), ofk=range(2, 8)):
    """Up to n sequences over nlit literals: literal lengths from `ll`, match lengths from `ml`, OF codes from `ofk` (as far as the
    output so far allows)."""
    out, pos, used = [], 0, 0
    for _ in range(n):
        a = rng.choice(list(ll)) or (0 if out else 1)
        if used + a > nlit:
            break
        pos += a
        used += a
        k = rng.choice([k for k in ofk if (1 << k) - 3 <= pos])
        o = rng.randint((1 << k) - 3, min((2 << k) - 4, pos))
        m = rng.choice(list(ml))
        out.append((a, m, o))
        pos += m
    return out


def test_treeless_one_stream(oracle, tool):
    rng = random.Random(1)
    assert round_trip(oracle, tool, letters(rng, 600, DICT_DIST), []) == (3, [0, 0, 0])


def test_missing_literal_byte_falls_back(oracle, tool):
    rng = random.Random(2)
    lits = letters(rng, 600, DICT_DIST) + b"z"            # 'z' has no code in the dictionary's table
    assert round_trip(oracle, tool, lits, [])[0] == 0      # Raw: below 1024 literals there is no own Huffman table
    lits = letters(rng, 5000, DICT_DIST) + b"z"
    assert round_trip(oracle, tool, lits, [])[0] == 1      # own Huffman


def test_treeless_four_streams(oracle, tool):
    rng = random.Random(3)
    assert round_trip(oracle, tool, letters(rng, 5000, DICT_DIST), [])[0] == 3
    assert round_trip(oracle, tool, letters(rng, 70000, DICT_DIST), [])[0] == 3   # 5-byte header


def test_own_huffman_beats_the_dictionary(oracle, tool):
    rng = random.Random(4)
    lits = letters(rng, 5000, {ord("a"): 1, ord("o"): 1, ord("e"): 1, ord("t"): 1})   # 2 bits each alone, 2.5 with the dictionary
    assert round_trip(oracle, tool, lits, [])[0] == 1


def test_repeat_for_every_table(oracle, tool):
    rng = random.Random(5)
    lits = letters(rng, 4000, DICT_DIST)
    seqs = seqs_for(rng, len(lits), 120)   # few enough that the tables' own descriptions weigh
    assert len(seqs) == 120
    lit_mode, modes = round_trip(oracle, tool, lits, seqs)
    assert modes == [3, 3, 3], modes


def test_missing_code_falls_back_to_the_blocks_table(oracle, tool):
    rng = random.Random(6)
    lits = letters(rng, 4000, DICT_DIST)
    seqs = seqs_for(rng, len(lits), 300)
    a, m, o = seqs[5]
    seqs[5] = (a, m + 200, o)                               # ML code above 31: not in the dictionary's table
    lit_mode, modes = round_trip(oracle, tool, lits, seqs)
    assert modes[2] == 2 and modes[0] == 3, modes
    seqs2 = [(a + (40 if i == 7 else 0), m, o) for i, (a, m, o) in enumerate(seqs_for(rng, len(lits) - 100, 300))]   # an LL code above 15
    lit_mode, modes = round_trip(oracle, tool, lits, seqs2)
    assert modes[0] == 2, modes


def test_rle_stays_rle(oracle, tool):
    rng = random.Random(7)
    lits = letters(rng, 3000, DICT_DIST)
    seqs = seqs_for(rng, len(lits), 200, ml=[20])
    lit_mode, modes = round_trip(oracle, tool, lits, seqs)
    assert modes[2] == 1 and modes[0] == 3, modes


def test_dictionary_as_the_encoder_sees_it(tool):
    exe, dpath, _, _ = tool
    out = subprocess.run([exe, dpath], capture_output=True, text=True, timeout=60).stdout.split()
    assert out[0] == "tables"
    assert [int(x) for x in out[1].split(",")] == [s for s in range(256) if s not in LENGTHS]
    assert out[2] == ",".join(str(c) for c in range(16, 36))
    assert out[3] == ",".join(str(c) for c in range(8, 32))
    assert out[4] == ",".join(str(c) for c in range(32, 53))
