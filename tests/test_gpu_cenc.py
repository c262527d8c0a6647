"""k_cenc on the GPU against the plain model of the entropy stage (tests/cenc.py), which shares no code with encode.cuh.

- Edges through the parse: single-block frames whose parse (the level's model, used as the search oracle) gives exactly 1024 /
  1025 and 16383 / 16384 literals, at Fastest, LAZY and OPT; the GPU frame is reference_frame's, now entirely Python.
- Without a parse model: every Compressed block of a GPU frame, re-encoded from the oracle's trace (its literals and Offset_Values),
  must be the block's bytes.  Checked on 64 MiB of C2b-shaped text as 512 frames and as one frame at every level, on a planted
  input at window_log 27 (LAZY and ULTRA) whose repeats lie more than 2^26 bytes back (OF codes 26 and 27 occur), and on one
  FrameCompressor frame.  Every block with a literal count within 2 of 1024, 4096 or 16384 or an OF code >= 24 is checked, with a
  seeded sample of 64 others: LL codes >= 25, ML codes >= 43 and repeat codes are in most blocks of text, and one block takes the
  model about 80 ms.  Every block follows the block-type rule."""
import functools
import random

import numpy as np
import pytest

import cenc
import clazy
import copt
import cparse
import datagen
import streamframe as SF
from test_gpu_compress_stream import Sink, Source
from test_gpu_cparse import compress

pytestmark = pytest.mark.gpu

B = cparse.BLOCK
MIB = 1 << 20
MODELS = {"fastest": cparse.FASTEST, "lazy": clazy.LAZY, "opt": copt.OPT}
SAMPLE = 64


# ---------------------------------------------------------------------------------------------------------------------------
# edges through the parse
# ---------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def edge_input(name, target):
    """A prefix of a 12-letter random text whose one-block parse at the level has exactly `target` literals: the prefix grows
    while the count is below the target; a text that overshoots is replaced by the next seed's."""
    for seed in range(64):
        rng = random.Random(target * 64 + seed)
        buf = bytes(rng.choice(b"etaoinshrdlu") for _ in range(2 * target + 8192))
        lo = target
        while lo <= len(buf):
            blk = cparse.parse_frame(buf[:lo], MODELS[name])[0]
            n = len(blk[0])
            if n == target:
                return buf[:lo], blk
            if n > target:
                break
            lo += max(1, (target - n) // 2)
    raise AssertionError("no prefix has that literal count")


@pytest.mark.parametrize("name", list(MODELS))
def test_literal_count_edges_through_the_parse(pkg, ctx, name):
    datas, blocks = [], []
    for target in (1024, 1025, 16383, 16384):
        d, blk = edge_input(name, target)
        assert len(blk[0]) == target
        mode = cenc.encode_block(blk[0], MODELS[name].records(blk[1]))[1]
        assert mode == (cenc.RAW if target == 1024 else cenc.HUF), (target, mode)
        datas.append(d)
        blocks.append(blk)
    frames, _ = compress(pkg, ctx, datas, level=getattr(pkg, name.upper()))
    for d, blk, f in zip(datas, blocks, frames):
        assert f == cparse.reference_frame(d, [blk], level=MODELS[name]), f"{len(blk[0])} literals"


# ---------------------------------------------------------------------------------------------------------------------------
# re-encoding traced blocks
# ---------------------------------------------------------------------------------------------------------------------------
def traced(oracle, frame):
    """Per block (every type): (block type, literals, [(ll, ml, Offset_Value)]) from the oracle's trace; also the decoded content."""
    d = oracle.FrameDecoder()
    d.set_max_window_size(1 << 27)
    d.trace_enable()
    d.decode_blocks(d.reset(frame))
    out = d.collect()
    blocks, lits, seqs = d.trace()
    res = []
    for b in blocks:
        lo, k = int(b["lit_offset"]), int(b["seq_offset"])
        s = [(int(ll), int(ml), int(ov)) for ll, ml, ov, _ in seqs[k:k + int(b["num_sequences"])].tolist()]
        res.append((int(b["block_type"]), lits[lo:lo + int(b["regenerated_size"])], s))
    return res, out


def rare(lits, ovs):
    """A literal count within 2 of 1024, 4096 or 16384, or an OF code >= 24."""
    n = len(lits)
    return any(abs(n - t) <= 2 for t in (1024, 4096, 16384)) or any(ov >= (1 << 24) for _, _, ov in ovs)


def check_frames(oracle, frames, datas, seed, stats=None):
    """Every block of the frames follows the block-type rule; Compressed blocks re-encode from their trace to their bytes: every one
    with a rare feature and a seeded sample of SAMPLE others.  Returns the number of blocks re-encoded."""
    cand = []
    for fi, (f, data) in enumerate(zip(frames, datas)):
        _, blocks, _ = SF.split_frame(f)
        tr, out = traced(oracle, f)
        assert out == data
        assert [t[0] for t in tr] == [b[1] for b in blocks]
        pos = 0
        for (last, btype, size, body), (_, lits, ovs) in zip(blocks, tr):
            n = min(B, len(data) - pos)
            raw = data[pos:pos + n]
            allsame = n > 0 and raw.count(raw[:1]) == n
            assert (btype == 1) == allsame, (fi, pos)
            if btype == 2:
                assert size < n
                cand.append((rare(lits, ovs), fi, pos, body, lits, ovs))
            elif btype == 0:
                assert size == n
            pos += n
    rng = random.Random(seed)
    rest = [c for c in cand if not c[0]]
    picked = [c for c in cand if c[0]] + rng.sample(rest, min(SAMPLE, len(rest)))
    for _, fi, pos, body, lits, ovs in picked:
        recs = [(ll, ml, (ov - 3) & 0xFFFFFFFF) for ll, ml, ov in ovs]
        got = cenc.encode_block(lits, recs)[0]
        assert got == body, f"frame {fi} block at {pos}: {len(ovs)} sequences, {len(lits)} literals"
        if stats is not None:
            stats.update(cenc.codes(recs)[1].tolist() if recs else [])
    return len(picked)


@functools.lru_cache(None)
def c2b_text():
    return datagen.c2_text_plain(64 * MIB).tobytes()


@pytest.mark.parametrize("level", ["fastest", "lazy", "opt", "ultra"])
@pytest.mark.parametrize("shape", ["512-frames", "one-frame"])
def test_c2b_blocks_reencode(pkg, ctx, oracle, level, shape):
    text = c2b_text()
    if shape == "512-frames":
        datas = [text[i:i + B] for i in range(0, len(text), B)]
        frames, _ = compress(pkg, ctx, datas, level=getattr(pkg, level.upper()))
    else:
        datas = [text]
        frames = [pkg.compress_to_vec(ctx, text, level=getattr(pkg, level.upper()), window_log=23 if level == "ultra" else 17)]
    assert check_frames(oracle, frames, datas, f"{level}-{shape}") >= SAMPLE


def far_planted():
    """2^27 + 1 MiB: random bytes and text, with 40 KiB pieces copied from 2^27 - 2 bytes back (OF code 27) and from 2^26 + 5000
    back (OF code 26)."""
    n = (1 << 27) + MIB
    rng = np.random.default_rng(27)
    buf = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    text = datagen.gen_text(8 * MIB, 27).tobytes()
    for k in range(8 * MIB, n - 8 * MIB, 32 * MIB):     # text only from 8 MiB on: the far pieces' sources stay unique
        buf[k:k + 4 * MIB] = text[:4 * MIB]
    for dst, off in ((n - 300000, (1 << 27) - 2), (n - 600000, (1 << 26) + 5000), ((1 << 26) + 900000, (1 << 26) + 5000)):
        buf[dst:dst + 40960] = buf[dst - off:dst - off + 40960]
    return bytes(buf)


@pytest.mark.parametrize("level", ["lazy", "ultra"])
def test_far_offsets_reencode(pkg, ctx, oracle, level):
    data = far_planted()
    frame = pkg.compress_to_vec(ctx, data, level=getattr(pkg, level.upper()), window_log=27)
    stats = set()
    check_frames(oracle, [frame], [data], 27, stats)
    assert {26, 27} <= stats, sorted(stats)


def test_frame_compressor_blocks_reencode(pkg, ctx, oracle):
    data = c2b_text()[:12 * MIB + 777]
    fc = pkg.FrameCompressor(ctx, pkg.LAZY)
    sink = Sink()
    fc.set_source(Source(data, "rand", seed=5))
    fc.set_drain(sink)
    assert fc.compress()["status"] == 0
    assert check_frames(oracle, [bytes(sink.buf)], [data], 5) >= SAMPLE
