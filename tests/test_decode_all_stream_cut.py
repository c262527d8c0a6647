"""How decode_all_stream cuts a source into submissions (b200z_debug_stream_cut, host only), checked against the plain model in
tests/streamcut.py on crafted streams: golden frames with skippable frames between them, long multi-block frames, truncations and
garbage tails.  No GPU needed."""
import pytest

import streamcut
from test_decode_all_chain import concat_with_skippables, corpus_frames, py_chain, raw_frame, skippable

CHUNKS = [4096, 131072, 1 << 20, 64 << 20]


def check(pkg, data, C):
    cuts, end = pkg.binding.stream_cut(data, C)
    got = [tuple(int(r[k]) for k in ("start", "end", "in_bytes", "out_bound", "nblocks", "nseq", "nframes", "flags")) for r in cuts]
    want, wend = streamcut.cut(data, C)
    assert got == want
    status = pkg.error_names().get(end["status"], "").replace("B200Z_ERR_", "") if end["status"] else None
    assert (end["error_offset"], status, end["error_frame"], end["skippable_frames"]) == \
        (wend["error_offset"], wend["status"], wend["error_frame"], wend["skippable_frames"])
    ends = streamcut.block_ends(data)
    prev_end = 0
    for i, r in enumerate(want):
        start, stop, inb, out, nb, nseq, nf, flags = r
        assert stop - start == inb
        assert start >= prev_end
        prev_end = stop
        # every cut followed by another submission lies at a block or frame end, and a frame continues exactly across the cuts
        # that fall inside it; the bounds hold, or the submission holds exactly one block
        if i + 1 < len(want):
            assert stop in ends, (r, C)
            assert bool(flags & 2) == bool(want[i + 1][7] & 1)
        assert nb == 1 or (inb <= C and out <= 4 * C and nb <= max(1, C // 16384) and nseq <= C // 4), (r, C)
    # the buffer never holds more than a chunk and a few blocks, whatever the skippable frames
    assert end["peak_buffered"] <= C + 2 * (18 + 3 + 131072 + 4)
    return want, end


@pytest.mark.parametrize("C", CHUNKS)
def test_corpus_with_skippables(pkg, manifest, C):
    buf, starts = concat_with_skippables(corpus_frames(manifest))
    subs, end = check(pkg, buf, C)
    assert end["status"] == 0 and end["error_offset"] == len(buf)
    assert end["skippable_frames"] == len(starts) // 2


@pytest.mark.parametrize("C", [4096, 131072, 1 << 20])
def test_long_frames_span_submissions(pkg, C):
    data = bytes((i * 131 + (i >> 9)) & 0xFF for i in range(5 << 20))
    buf = raw_frame(data) + raw_frame(data[:300000], checksum=True) + raw_frame(b"x" * 10)
    subs, end = check(pkg, buf, C)
    assert end["status"] == 0
    if C < (4 << 20):
        assert any(r[7] & 1 for r in subs) and any(r[7] & 2 for r in subs)


def test_skippable_larger_than_a_chunk_is_not_buffered(pkg, manifest):
    frames = corpus_frames(manifest)[:6]
    big = skippable(3 << 20)
    buf = frames[0] + big + frames[1] + big + big + b"".join(frames[2:])
    for C in (4096, 131072, 1 << 20):
        subs, end = check(pkg, buf, C)
        assert end["status"] == 0 and end["skippable_frames"] == 3
        assert end["peak_buffered"] < len(big)


def test_truncations_and_garbage_end_where_the_chain_does(pkg, manifest):
    buf, starts = concat_with_skippables(corpus_frames(manifest)[:20])
    pieces = set()
    for s in starts + [len(buf)]:
        for d in (-5, -4, -3, -1, 0, 1, 2, 3, 4, 5, 8, 9, 40):
            if 0 <= s + d <= len(buf):
                pieces.add(s + d)
    for C in (4096, 1 << 20):
        for n in sorted(pieces):
            _, end = check(pkg, buf[:n], C)
            chain = py_chain(buf[:n])
            if end["status"]:
                assert end["error_offset"] == chain[-1], (n, end)
            else:
                assert end["error_offset"] == n
        for tail in (b"\x00", b"\x28\xb5", b"garbage that is no frame", b"\x28\xb5\x2f\xfd", b"\x50\x2a\x4d\x18\x00\x00"):
            _, end = check(pkg, buf + tail, C)
            assert end["status"] and end["error_offset"] == len(buf) == py_chain(buf + tail)[-1]


def test_empty_and_only_skippable(pkg):
    for C in (4096, 1 << 20):
        assert check(pkg, b"", C)[0] == []
        subs, end = check(pkg, skippable(0) + skippable(3), C)
        assert subs == [] and end["status"] == 0 and end["skippable_frames"] == 2
