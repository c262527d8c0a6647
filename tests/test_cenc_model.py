"""The plain model of the compressor's entropy stage (tests/cenc.py) on the CPU.

- It equals the host build of encode.cuh (tests/host/encode_test.cpp, encode_dict_test.cpp) byte for byte, with the same literal and
  table modes, on crafted sets that sit on each decision edge (each set asserts its edge), and on every block the Fastest, LAZY and
  OPT parse models give for their crafted cases, forced long-distance pieces included.
- Its Huffman code is checked against references that share none of its decisions: a plain heap code (equal cost when that code
  is at most 11 deep), the package-merge optimum for the 11-bit limit (never below it; the gap above it is pinned), Kraft sum 1.
  Normalized FSE counts sum to 2^log and are nonzero exactly for the codes present.
- Its blocks decode with the oracle and libzstd to seqcraft.execute's bytes.
- Its dictionary writer equals b200z_debug_dict_from_counts."""
import heapq
import os
import random
import shutil
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import cenc
import clazy
import cldm
import copt
import cparse
import datagen
import entcraft as E
import seqcraft
import test_dict_format_host as DF
from test_cldm_model import planted

needs_nvcc = pytest.mark.skipif(not os.path.exists(seqcraft.NVCC), reason="nvcc not available")
M32 = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------------------------
# the host build
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dict_tool():
    d = tempfile.mkdtemp(prefix="cenc")
    exe = os.path.join(d, "encode_dict_test")
    subprocess.check_call([seqcraft.NVCC, "-x", "cu", "-std=c++17", "-O2", "-w", "-o", exe,
                           os.path.join(seqcraft.HERE, "host", "encode_dict_test.cpp")])
    yield exe, d
    shutil.rmtree(d, True)


def host(lits, recs, formatted=None, tool=None):
    """(content, literal mode, [LL, OF, ML] modes) from the host build; recs are (ll, ml, Offset_Value - 3 mod 2^32)."""
    if formatted is None:
        return seqcraft.encode(lits, recs)
    exe, d = tool
    dpath, src, dst = os.path.join(d, "dict"), os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    open(dpath, "wb").write(formatted)
    with open(src, "wb") as f:
        f.write(struct.pack("<I", len(lits)) + bytes(lits) + struct.pack("<I", len(recs)) +
                b"".join(struct.pack("<3I", ll, ml, of & M32) for ll, ml, of in recs))
    out = subprocess.run([exe, dpath, src, dst], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr
    f = out.stdout.split()
    return open(dst, "rb").read(), int(f[2]), [int(x) for x in f[3:6]]


def same_as_host(lits, recs, formatted=None, tool=None):
    """The model's (content, literal mode, modes), after checking them against the host build."""
    want = host(lits, recs, formatted, tool)
    got = cenc.encode_block(lits, recs, cenc.Tables(formatted) if formatted is not None else None)
    assert got[1:] == want[1:], f"modes: model {got[1:]}, host {want[1:]}"
    if got[0] != want[0]:
        j = next((j for j, (a, b) in enumerate(zip(got[0], want[0])) if a != b), min(len(got[0]), len(want[0])))
        pytest.fail(f"content differs at byte {j} (model {len(got[0])} bytes, host {len(want[0])})")
    return got


# ---------------------------------------------------------------------------------------------------------------------------
# crafted sets on the decision edges
# ---------------------------------------------------------------------------------------------------------------------------
def skewed(rng, n, alphabet=b"eeeetttaaoinshrdlu"):
    return bytes(rng.choice(alphabet) for _ in range(n))


def own_margin(lits):
    """hsize + csize - (n + 3) of the block's own Huffman literals (negative: Huffman pays)."""
    n = len(lits)
    lengths = cenc.huf_lengths(np.bincount(np.frombuffer(lits, dtype=np.uint8), minlength=256))
    desc = cenc.huf_description(lengths)
    csize = len(desc) + len(E.lit_payload(E.huf_table(E.huf_weights(lengths)), lits, 4))
    return (4 if n < 16384 and csize < 16384 else 5) + csize - (n + 3)


def fib_literals(k, seed):
    fib = [1, 1]
    while len(fib) < k:
        fib.append(fib[-1] + fib[-2])
    scale = -(-(cenc.RAW_LITERALS_MAX + 1) // sum(fib))    # past the Raw cap; scaling keeps every merge's order
    lits = bytearray()
    for s, c in enumerate(fib):
        lits += bytes([65 + s]) * (c * scale)
    random.Random(seed).shuffle(lits)
    return bytes(lits)


def fix_ups(lits):
    steps = []
    cenc.huf_lengths(np.bincount(np.frombuffer(lits, dtype=np.uint8), minlength=256), steps)
    return {k for k, _ in steps}


def recs_for(rng, n, ll=(0, 1, 2), ml=range(3, 12), of_max=1000):
    return [(rng.choice(ll), rng.choice(ml), rng.randint(1, of_max)) for _ in range(n)]


def lits_for(rng, recs, tail=5):
    return skewed(rng, sum(q[0] for q in recs) + tail, b"xyzw")


def seq_header(content, lits):
    """(count, the bytes after it) of a block without a dictionary."""
    p = len(cenc.literals_section(lits)[0])
    b = content[p]
    if b < 128:
        return b, content[p + 1:]
    if b < 255:
        return ((b - 128) << 8) + content[p + 1], content[p + 2:]
    return content[p + 1] + (content[p + 2] << 8) + 0x7F00, content[p + 3:]


class Set:
    """One crafted literal and record set.  edge(lits, recs, (content, lit mode, modes)) asserts the edge it sits on.  history:
    bytes of Raw blocks before it, for decoding (None: its offsets are not decodable)."""

    def __init__(self, name, lits, recs, edge, history=b"", formatted=None):
        self.id, self.lits, self.recs, self.edge, self.history, self.formatted = name, bytes(lits), list(recs), edge, history, formatted

    def __repr__(self):
        return self.id


def literal_sets():
    rng = random.Random(0xCE01)
    out = []
    text = skewed(rng, 20000)
    for n, mode in ((1024, cenc.RAW), (1025, cenc.HUF)):
        out.append(Set(f"n{n}", text[:n], [], lambda l, r, g, m=mode: g[1] == m))
    rnd = bytes(rng.randrange(256) for _ in range(5000))
    for n, h in ((31, 1), (32, 2), (4095, 2), (4096, 3)):
        out.append(Set(f"raw-n{n}-header{h}", rnd[:n], [], lambda l, r, g, h=h: g[1] == cenc.RAW and len(g[0]) == h + len(l) + 1))
    for n, h in ((16383, 4), (16384, 5)):
        out.append(Set(f"huf-n{n}-header{h}", text[:n], [], lambda l, r, g, h=h: g[1] == cenc.HUF and (g[0][0] >> 2) & 3 == h - 2))
    # Huffman does not pay when hsize + csize >= n + 3: a prefix of a nearly random buffer on each side
    rng2 = random.Random(11)
    buf = bytes(97 if rng2.random() < 0.05 else rng2.randrange(256) for _ in range(2600))
    out.append(Set("hsize+csize=n+3-raw", buf[:2524], [], lambda l, r, g: own_margin(l) == 0 and g[1] == cenc.RAW))
    out.append(Set("hsize+csize=n+2-huf", buf[:2525], [], lambda l, r, g: own_margin(l) == -1 and g[1] == cenc.HUF))
    # the largest literal byte sets the number of weights: 127 and 128 direct, 129 FSE-compressed
    for top in (127, 128, 129):
        lits = bytearray(skewed(rng, 3000, b"ab"))
        lits[1234] = top
        direct = top <= 128
        out.append(Set(f"largest-byte{top}-{'direct' if direct else 'fse'}-weights", lits, [],
                       lambda l, r, g, top=top, d=direct: g[1] == cenc.HUF and (g[0][4] == 127 + top if d else g[0][4] < 128)))
    # Fibonacci counts: clamping to 11 bits overflows the Kraft sum; k = 14, 17, 24 also shorten after lengthening
    for k in (13, 14, 17, 20, 24):
        want = {"grow", "shrink"} if k in (14, 17, 24) else {"grow"}
        out.append(Set(f"fibonacci{k}-fix-ups-{'+'.join(sorted(want))}", fib_literals(k, k), [],
                       lambda l, r, g, w=want: g[1] == cenc.HUF and fix_ups(l) == w))
    out.append(Set("one-distinct-byte", b"q" * 3000, [], lambda l, r, g: g[1] == cenc.RAW))
    out.append(Set("random-does-not-pay", rnd, [], lambda l, r, g: g[1] == cenc.RAW and own_margin(l) >= 0))
    many = bytes(rng.randrange(256) if rng.random() < 0.3 else rng.choice(b"etaoin ") for _ in range(30000))
    out.append(Set("all-256-bytes", many, [], lambda l, r, g: g[1] == cenc.HUF and len(set(l)) == 256))
    return out


def sequence_sets():
    rng = random.Random(0xCE02)
    hist = bytes(rng.randrange(256) for _ in range(1000))
    out = []
    for n, nb in ((0, 1), (1, 1), (127, 1), (128, 2), (0x7EFF, 2), (0x7F00, 3), (0x8000, 3)):
        recs = recs_for(rng, n, ll=(0, 0, 1), ml=(3, 4), of_max=1000)
        out.append(Set(f"nseq{n}-count{nb}bytes", lits_for(rng, recs), recs,
                       lambda l, r, g, nb=nb: seq_header(g[0], l)[0] == len(r) and
                       len(seq_header(g[0], l)[1]) == len(g[0]) - len(cenc.literals_section(l)[0]) - nb, hist))
    recs = [(0, 4, 5)] * 300
    out.append(Set("single-code-per-table-rle", b"abcdefgh", recs, lambda l, r, g: g[2] == [1, 1, 1], hist))
    far = bytes(rng.randrange(256) for _ in range(64))
    top = [(65536, 5, 10), (3, 7, 12), (50000, 9, 4)]
    out.append(Set("ll-code35", bytes(rng.randrange(256) for _ in range(65536 + 50000 + 3 + 4)), top,
                   lambda l, r, g: 35 in cenc.codes(r)[0].tolist(), far))
    top = [(3, 65539 + 77, 12), (2, 9, 4), (0, 30000, 30)]
    out.append(Set("ml-code52", b"abcdefg", top, lambda l, r, g: 52 in cenc.codes(r)[2].tolist(), far))
    recs = [(1, 5 + c % 7, ((1 << c) - 3 + rng.randrange(1 << c)) & M32) for c in range(2, 28) for _ in range(3)]
    recs += [(ll, 6, (ov - 3) & M32) for ov in (1, 2, 3) for ll in (0, 2)]          # Offset_Values 1-3: OF codes 0 and 1
    rng.shuffle(recs)
    out.append(Set("of-codes0-27", lits_for(rng, recs), recs, lambda l, r, g: set(cenc.codes(r)[1].tolist()) == set(range(28)), None))
    # ML codes {0, 4, 29, 30} over many sequences: zero runs of 3 and 24 in the ML description (LL and OF are RLE)
    recs = [(1, 3 + rng.choice((0, 4, 29, 30)), 40) for _ in range(400)]
    out.append(Set("zero-runs-3-and-24", lits_for(rng, recs), recs, lambda l, r, g: g[2] == [1, 1, 2] and _ml_runs(g[0], l) >= {3, 24}, hist))
    recs = [(rng.choice((0, 1, 3)), rng.randint(3, 30), (rng.choice((1, 2, 3)) - 3) & M32 if rng.random() < 0.4 else rng.randint(1, 900))
            for _ in range(500)]
    out.append(Set("repeat-offset-values", lits_for(rng, recs), recs, lambda l, r, g: {0, 1} <= set(cenc.codes(r)[1].tolist()), None))
    for k in range(3):
        recs = recs_for(rng, rng.randint(200, 1500), ll=range(0, 40), ml=range(3, 60), of_max=100000)
        out.append(Set(f"mixed-{k}", skewed(rng, sum(q[0] for q in recs) + 9), recs, lambda l, r, g: g[2] == [2, 2, 2],
                       bytes(rng.randrange(256) for _ in range(100000))))
    return out


def _ml_runs(content, lits):
    _, rest = seq_header(content, lits)
    _, norm, _ = E.read_ncount(rest[3:])                   # modes byte, LL and OF RLE bytes, then ML's description
    runs, z = set(), 0
    for p in norm + [1]:
        if p == 0:
            z += 1
        elif z:
            runs.add(z)
            z = 0
    return runs


NEAR_FLAT = {s: 7 if s == 0 else 9 if s >= 254 else 8 for s in range(256)}


def dictionary(ll_norm, dict_id=0x5151):
    """A formatted dictionary whose Huffman code is NEAR_FLAT and whose LL table is ll_norm = (log, norm)."""
    rng = random.Random(dict_id)
    huf = E.fse_weights(rng, NEAR_FLAT, 6)
    of = (5, [2] * 16)
    ml = (6, [2] * 32)
    return E.dictionary(dict_id, huf, of, ml, ll_norm, (1, 4, 8), bytes(rng.randrange(256) for _ in range(3000)))[0]


def dictionary_sets():
    out = []
    d = dictionary((6, [4] * 16))
    # 1-stream Treeless against Raw (601 literals): a zeros (7 bits) and b 0xFE (9 bits); a - b = 9 ties, a - b = 17 is one smaller
    for a, b, mode in ((305, 296, cenc.RAW), (309, 292, cenc.TREELESS)):
        lits = bytes([0] * a + [0xFE] * b)
        tie = 3 + len(E.huf_stream(cenc.Tables(d).huf, lits)) - (2 + len(lits))
        out.append(Set(f"treeless-{'tie-refused' if mode == cenc.RAW else 'one-smaller-taken'}", lits, [],
                       lambda l, r, g, m=mode, t=tie: g[1] == m and t == (0 if m == cenc.RAW else -1), None, d))
    rng = random.Random(0xCE03)
    out.append(Set("treeless-4-streams", bytes(rng.choice((0, 0, 0, 1, 2, 254)) for _ in range(5000)), [],
                   lambda l, r, g: g[1] in (cenc.TREELESS, cenc.HUF), None, d))
    out.append(Set("treeless-byte-without-code-never", b"", [], lambda l, r, g: g[1] == cenc.RAW, None, d))
    # Repeat for LL against its own table: LL codes 0 (c0 times) and 1, OF and ML single codes.  The dictionary's LL norm [a, 64 - a]
    # makes its cost exactly desc * 2^11 + own cost (taken) or one more (refused)
    for n, c0, a, mode in ((24, 7, 48, cenc.REPEAT_MODE), (15, 1, 41, cenc.FSE_MODE)):
        recs = [(0, 4, 7)] * c0 + [(1, 4, 7)] * (n - c0)
        random.Random(n).shuffle(recs)
        dd = dictionary((6, [a, 64 - a]), 0x6000 + a)
        out.append(Set(f"repeat-{'tie-taken' if mode == cenc.REPEAT_MODE else 'one-over-refused'}", b"x" * (n - c0 + 3), recs,
                       lambda l, r, g, m=mode, c0=c0, a=a: g[2] == [m, 1, 1] and _repeat_margin(r, a) == (0 if m == cenc.REPEAT_MODE else 1),
                       b"h" * 64, dd))
    recs = recs_for(rng, 300, ll=range(16), ml=range(3, 35), of_max=28)
    out.append(Set("repeat-missing-code-own-table", b"x" * 3000, recs + [(40, 4, 7)], lambda l, r, g: g[2][0] == cenc.FSE_MODE, b"h" * 64, d))
    return out


def _repeat_margin(recs, a):
    """cost(dictionary) - (desc * 2^11 + cost(own)) of the LL table of recs against the LL norm [a, 64 - a] at log 6."""
    c = np.bincount(cenc.codes(recs)[0], minlength=2).tolist()
    n = len(recs)
    log = cenc.fse_pick_log(n, 1, 2, 9)
    norm = cenc.fse_normalize(c, n, log)
    return cenc.fse_cost_q8(c, [a, 64 - a], 6) - (len(E.write_ncount(norm, log)) << 11) - cenc.fse_cost_q8(c, norm, log)


SETS = literal_sets() + sequence_sets() + dictionary_sets()


@needs_nvcc
@pytest.mark.parametrize("s", SETS, ids=repr)
def test_model_is_the_host_build_on_the_edges(dict_tool, s):
    got = same_as_host(s.lits, s.recs, s.formatted, dict_tool)
    assert s.edge(s.lits, s.recs, got), f"{s.id}: the set is not on its edge ({got[1:]})"


def test_model_blocks_decode(oracle):
    """Every crafted set with decodable offsets, framed after its history, decodes with the oracle and libzstd."""
    n = 0
    for s in SETS:
        if s.history is None:
            continue
        hist = [("raw", s.history[i:i + cparse.BLOCK]) for i in range(0, len(s.history), cparse.BLOCK)]
        ovs = [(ll, ml, (of + 3) & M32) for ll, ml, of in s.recs]
        expect = seqcraft.execute(hist + [("cmp", s.lits, ovs)], ov=True)
        assert expect is not seqcraft.ERROR, s.id
        content = cenc.encode_block(s.lits, s.recs, cenc.Tables(s.formatted) if s.formatted else None)[0]
        frame = struct.pack("<IBB", 0xFD2FB528, (2 << 6) | (3 if s.formatted else 0), (17 - 10) << 3)
        frame += (struct.unpack_from("<I", s.formatted, 4)[0].to_bytes(4, "little") if s.formatted else b"") + struct.pack("<I", len(expect))
        for i, (_, h) in enumerate(hist):
            frame += struct.pack("<I", len(h) << 3)[:3] + h
        frame += struct.pack("<I", 1 | (2 << 1) | (len(content) << 3))[:3] + content
        if s.formatted:
            dec = oracle.FrameDecoder()
            dec.add_dict(s.formatted)
            dec.decode_blocks(dec.reset(frame))
            assert dec.collect() == expect, s.id
        else:
            assert oracle.decode_frame(frame)[0] == expect, s.id
        assert datagen.decompress(frame, len(expect), raw_dict=s.formatted) == expect, s.id
        n += 1
    assert n >= 30


# ---------------------------------------------------------------------------------------------------------------------------
# every block of the parse models
# ---------------------------------------------------------------------------------------------------------------------------
PARSES = {"fastest": (cparse.FASTEST, cparse.cases), "lazy": (clazy.LAZY, clazy.cases), "opt": (copt.OPT, copt.cases)}


def parse_blocks(level, cases):
    for c in cases():
        for f, blocks in zip(c.frames, cparse.parse(c.frames, c.content, level)):
            for b in blocks:
                if b[0] != "rle" and (b[0] or b[1]):
                    yield c.id, b[0], level.records(b[1])


@needs_nvcc
@pytest.mark.parametrize("name", list(PARSES))
def test_model_is_the_host_build_on_every_parse_block(name):
    level, cases = PARSES[name]
    n = 0
    for cid, lits, recs in parse_blocks(level, cases):
        want = seqcraft.encode(lits, recs)
        got = cenc.encode_block(lits, recs)
        assert got == (want[0], want[1], want[2]), f"{cid}: a block of {len(recs)} sequences differs"
        n += 1
    assert n >= 40


@needs_nvcc
@pytest.mark.parametrize("level", [cparse.FASTEST, clazy.LAZY], ids=["fastest", "lazy"])
def test_model_is_the_host_build_with_forced_pieces(level):
    data = planted(600000, [(400000, 100, 150000), (520000, 30000, 20000)], 5)
    blocks = cldm.parse([data], 20, level=level)[0]
    assert max(cldm.offsets(blocks)) > cldm.WINDOW
    for b in blocks:
        if b[0] != "rle":
            recs = level.records(b[1])
            assert cenc.encode_block(b[0], recs) == tuple(seqcraft.encode(b[0], recs)), "a block with long matches differs"


# ---------------------------------------------------------------------------------------------------------------------------
# Huffman and FSE against exact references
# ---------------------------------------------------------------------------------------------------------------------------
def heap_code(w):
    """(cost, depth) of a plain Huffman code over the positive weights w (a heap of subtrees, each a list of leaves)."""
    h = [(c, i, [i]) for i, c in enumerate(w)]
    heapq.heapify(h)
    depth, cost, tick = [0] * len(w), 0, len(w)
    while len(h) > 1:
        a, _, la = heapq.heappop(h)
        b, _, lb = heapq.heappop(h)
        for i in la + lb:
            depth[i] += 1
        cost += a + b
        heapq.heappush(h, (a + b, tick, la + lb))
        tick += 1
    return cost, max(depth)


def package_merge(w, limit):
    """Cost of the optimal prefix code over w with lengths <= limit (package-merge)."""
    n = len(w)
    leaves = sorted(((c, np.eye(1, n, i, dtype=np.int64)[0]) for i, c in enumerate(w)), key=lambda x: x[0])
    cur = leaves
    for _ in range(limit - 1):
        pk = [(cur[k][0] + cur[k + 1][0], cur[k][1] + cur[k + 1][1]) for k in range(0, len(cur) - 1, 2)]
        cur = sorted(leaves + pk, key=lambda x: x[0])
    lengths = sum(v for _, v in cur[:2 * n - 2])
    return int(np.dot(lengths, w))


def histograms():
    """(name, counts[256]) of Fibonacci sets and of the literals of the suite's texts."""
    out = []
    for k in range(12, 32):
        c = np.zeros(256, dtype=np.int64)
        fib = [1, 1]
        while len(fib) < k:
            fib.append(fib[-1] + fib[-2])
        c[65:65 + k] = fib
        out.append((f"fibonacci{k}", c))
    texts = {"gen_text": datagen.gen_text(4 * cparse.BLOCK, 0xC9A1).tobytes(),
             "gen_silesia_mix": datagen.gen_silesia_mix(2 * cparse.BLOCK, 0xC9A2).tobytes(),
             "gen_binary_records": datagen.gen_binary_records(2 * cparse.BLOCK, 0xC9A3).tobytes()}
    for name, t in texts.items():
        for k, b in enumerate(cparse.parse_frame(t)):
            if b[0] != "rle" and len(b[0]) > cenc.RAW_LITERALS_MAX:
                out.append((f"{name}-block{k}", np.bincount(np.frombuffer(b[0], dtype=np.uint8), minlength=256)))
    rng = np.random.default_rng(9)
    for k in range(20):
        out.append((f"random{k}", np.bincount(np.minimum(255, rng.geometric(rng.uniform(0.01, 0.5), 5000)), minlength=256)))
    return out


HIST = histograms()
# bits above the package-merge optimum, measured: where the 11-bit limit binds (Fibonacci sets from 15 symbols), and on the texts
# from the encoder's tie order and fix-up choices (0.14-0.18 % on gen_text, 1.6 % on the first gen_silesia_mix block)
GAP = {"fibonacci15": 5, "fibonacci16": 26, "fibonacci17": 26, "fibonacci18": 60, "fibonacci19": 149, "fibonacci20": 382,
       "fibonacci21": 759, "fibonacci22": 1602, "fibonacci23": 3571, "fibonacci24": 4304, "fibonacci25": 7087, "fibonacci26": 11789,
       "fibonacci27": 19918, "fibonacci28": 34668, "fibonacci29": 62715, "fibonacci30": 118809, "fibonacci31": 237618,
       "gen_text-block0": 262, "gen_text-block1": 244, "gen_text-block2": 282, "gen_text-block3": 322, "gen_silesia_mix-block0": 2895}
RANDOM_GAP_MAX = 0.002     # relative, on the random geometric sets (measured 0.18 %)


def test_huffman_against_heap_and_package_merge():
    gaps = {}
    for name, c in HIST:
        ln = cenc.huf_lengths(c)
        w = [int(x) for x in c if x]
        cost = sum(int(c[s]) * l for s, l in ln.items())
        assert sum(1 << (11 - l) for l in ln.values()) == 1 << 11, name            # Kraft sum exactly 1
        assert set(ln) == set(np.flatnonzero(c).tolist()) and max(ln.values()) <= 11, name
        hcost, hdepth = heap_code(w)
        if hdepth <= 11:
            assert cost == hcost, f"{name}: {cost} bits, a plain Huffman code within 11 bits takes {hcost}"
        opt = package_merge(w, 11)
        assert cost >= opt, name
        if name.startswith("random"):
            assert cost - opt <= RANDOM_GAP_MAX * opt, name
        elif cost > opt:
            gaps[name] = cost - opt
    assert gaps == GAP, gaps


def test_fse_normalization_properties():
    rng = random.Random(0xCE04)
    for _ in range(3000):
        t = rng.randrange(3)
        k = rng.randint(2, cenc.MAX_SYM[t] + 1)
        cnt = [0 if rng.random() < 0.3 else int(rng.paretovariate(0.7)) for _ in range(k)]
        cnt[-1] = cnt[-1] or 1
        cnt[0] = cnt[0] or 1
        n = sum(cnt)
        present = [s for s, x in enumerate(cnt) if x]
        log = cenc.fse_pick_log(n, k - 1, len(present), cenc.MAX_LOG[t])
        assert 5 <= log <= cenc.MAX_LOG[t] and (1 << log) >= len(present)
        norm = cenc.fse_normalize(cnt, n, log)
        assert sum(abs(p) for p in norm) == 1 << log
        assert [p != 0 for p in norm] == [x != 0 for x in cnt]
        desc = E.write_ncount(norm, log)
        assert E.read_ncount(desc + b"\0\0") == (log, norm, len(desc))


def test_log2_q8_against_floats():
    for p in list(range(1, 1200)) + [1 << k for k in range(31)] + [(1 << 31) - 1]:
        assert abs(cenc.log2_q8(p) - np.log2(p) * 256) < 1.0, p


# ---------------------------------------------------------------------------------------------------------------------------
# the dictionary writer
# ---------------------------------------------------------------------------------------------------------------------------
def test_dictionary_writer_is_the_librarys(pkg):
    content = datagen.gen_text(30000, 0xD1C7).tobytes()
    for name, counts in DF.crafted(len(content)):
        assert cenc.dict_from_counts(counts, content) == pkg.dict_from_counts(counts, content), name
        assert cenc.dict_from_counts(counts, content, 77, 2000) == pkg.dict_from_counts(counts, content, dict_id=77, dict_cap=2000), name
    fs = datagen.config_c5(nframes=300, cache=False)
    plain = fs.plain.tobytes()
    samples = [plain[int(o):int(o + n)] for o, n in zip(fs.out_off, fs.out_size)]
    raw = fs.raw_dict.tobytes()
    counts = cparse.counts(samples, raw)
    assert cenc.dict_from_counts(counts, raw) == pkg.dict_from_counts(counts, raw), "C5 counts"
