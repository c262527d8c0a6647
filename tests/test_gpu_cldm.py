"""Long-distance matching on the GPU (window_log > 17): the batch compressor's frames equal tests/cldm.py's byte for byte, window_log 17
and small frames are unchanged, the stream compressor's blocks equal the batch compressor's, every frame decodes everywhere within
its own window, the ratio follows the window, bad arguments are refused before any launch, and memory and output are stable."""
import functools
import gc
import io
import struct

import numpy as np
import pytest

import clazy
import cldm
import cparse
import datagen
import streamframe as SF
from test_gpu_compress_stream import Sink, Source, _chunk
from test_gpu_cparse import compress

pytestmark = pytest.mark.gpu

B = cldm.BLOCK
MIB = 1 << 20


def planted(n, seed, offsets):
    """Text and random stretches, with for every offset o a 20-60 KiB piece copied from o bytes back (repeats planted at several
    places, so that some of them overlap earlier copies)."""
    rng = np.random.default_rng(seed)
    text = datagen.gen_text(n, seed).tobytes()
    noise = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    buf = bytearray()
    while len(buf) < n:   # alternate 64 KiB of text and of noise, so the regular parse sees both
        k = len(buf)
        buf += (text if (k >> 16) & 1 else noise)[k:k + 65536]
    del buf[n:]
    at = 200000
    for i, o in enumerate(offsets * 3):
        at += int(rng.integers(150000, 400000))
        ln = int(rng.integers(20000, 60000))
        if at + ln > n:
            break
        if at >= o:
            buf[at:at + ln] = buf[at - o:at - o + ln]
    return bytes(buf)


OFFSETS = [131073, 140000, 600000, 2 * MIB + 3, 4 * MIB]


@functools.lru_cache(None)
def inputs():
    """(big, mid, plain): a 5 MiB frame with repeats up to 4 MiB back, a 700,000-byte one, and a submission of big, 100,000
    bytes, mid and one block of big."""
    big = planted(5 * MIB, 71, OFFSETS)
    mid = planted(700000, 72, [131073, 300000])
    return big, mid, [big, planted(100000, 73, []), mid, big[:B]]

_models = {}


def model(frames, wl, lazy, content=None):
    key = (tuple(map(len, frames)), hash(tuple(frames)), wl, lazy, content and hash(content))
    if key not in _models:
        _models[key] = cldm.parse(frames, wl, content, clazy.LAZY if lazy else cparse.FASTEST)
    return _models[key]


def reference(data, blocks, window_log, lazy, **kw):
    return cparse.reference_frame(data, blocks, level=clazy.LAZY if lazy else cparse.FASTEST, window_log=window_log, **kw)


def check_decodes(pkg, ctx, oracle, datas, frames, window_log):
    """libzstd, the oracle (through its trace: each frame's window is its descriptor's and every offset lies within it) and
    FrameDecoder."""
    dec = pkg.FrameDecoder(ctx)
    for d, f in zip(datas, frames):
        wl = cparse.frame_window_log(len(d), window_log)
        assert f[5] == (wl - 10) << 3
        o = oracle.FrameDecoder()
        o.set_max_window_size(1 << 27)
        o.trace_enable()
        o.decode_blocks(o.reset(f))
        assert o.collect() == d
        seqs = o.trace()[2]
        assert o.window_size() == 1 << wl and (len(seqs) == 0 or int(seqs[:, 3].max()) <= 1 << wl)
        assert datagen.decompress(f, len(d), window_log_max=27) == d
        assert dec.decode_all(f, len(d)) == d


@pytest.mark.parametrize("lazy", [False, True], ids=["fastest", "lazy"])
@pytest.mark.parametrize("window_log", [18, 23, 27])
def test_frames_equal_the_model(pkg, ctx, oracle, lazy, window_log):
    big, mid, plain = inputs()
    level = pkg.LAZY if lazy else pkg.FASTEST
    blocks = model(plain, window_log, lazy)
    before = ctx.kernel_launches()
    frames, res = compress(pkg, ctx, plain, level=level, window_log=window_log)
    assert ctx.kernel_launches() - before == 17 + 4   # the long-match kernels, then the four stages
    for i, (d, f) in enumerate(zip(plain, frames)):
        assert f == reference(d, blocks[i], window_log, lazy), f"frame {i}"
    far = [o for o in cldm.offsets(blocks[0]) if o > B]
    assert far and max(far) <= 1 << window_log
    if window_log >= 23:
        assert 4 * MIB in far
    frames2, _ = compress(pkg, ctx, plain[:1], level=level, window_log=window_log, checksum=False, device=True)
    assert frames2[0] == reference(big, blocks[0], window_log, lazy, checksum=False)
    if window_log == 23:
        check_decodes(pkg, ctx, oracle, plain, frames, window_log)


@pytest.mark.parametrize("lazy", [False, True], ids=["fastest", "lazy"])
def test_frames_with_dictionaries_equal_the_model(pkg, ctx, lazy):
    big, mid, plain = inputs()
    level = pkg.LAZY if lazy else pkg.FASTEST
    content = mid[:60000] + big[:50000]
    datas = [mid, big[:2 * MIB]]
    blocks = model(datas, 23, lazy, content)
    R = pkg.Dictionary.raw_content(ctx, 1, content)
    frames, _ = compress(pkg, ctx, datas, dict=R, level=level, window_log=23)
    for i, d in enumerate(datas):
        assert frames[i] == reference(d, blocks[i], 23, lazy), f"raw content frame {i}"
    fin = pkg.finalize_dict(ctx, content, [mid[i:i + 4096] for i in range(0, 400000, 4096)])
    F = pkg.Dictionary.decode_dict(ctx, fin)
    frames, _ = compress(pkg, ctx, datas, dict=F, dict_tables=True, level=level, window_log=23)
    for i, d in enumerate(datas):
        assert frames[i] == reference(d, blocks[i], 23, lazy, dict_id=F.id, dict_tables=fin), f"formatted frame {i}"


def test_window_17_is_the_dict_entry(pkg, ctx):
    big, mid, plain = inputs()
    L = pkg.lib()
    datas = plain
    for level in (pkg.UNCOMPRESSED, pkg.FASTEST, pkg.LAZY):
        frames, _ = compress(pkg, ctx, datas, level=level, window_log=17)
        io_ = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
        so = oo = 0
        for i, d in enumerate(datas):
            io_[i] = (so, len(d), oo, pkg.compress_bound(len(d)))
            so += len(d)
            oo += pkg.compress_bound(len(d))
        src = np.frombuffer(b"".join(datas), dtype=np.uint8)
        out = np.zeros(oo, dtype=np.uint8)
        res = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
        assert L.b200z_compress_frames_batch_dict(ctx.h, src.ctypes.data, src.size, 0, io_.ctypes.data, len(datas), level, 1, None,
                                                  out.ctypes.data, out.size, 0, res.ctypes.data) == 0
        assert [out[int(r["dst_off"]):int(r["dst_off"]) + int(x["dst_size"])].tobytes() for r, x in zip(io_, res)] == frames


def test_c2b_shaped_frames_are_unchanged_at_27(pkg, ctx):
    plain = datagen.c2_text_plain(8192 * B).tobytes()
    datas = [plain[i:i + B] for i in range(0, len(plain), B)]
    for level in (pkg.FASTEST, pkg.LAZY):
        a, _ = compress(pkg, ctx, datas, level=level, window_log=17)
        before = ctx.kernel_launches()
        b, _ = compress(pkg, ctx, datas, level=level, window_log=27)
        assert ctx.kernel_launches() - before == 4   # the four stages, no long-match kernel
        assert a == b
        assert all(f[5] == 0x38 for f in b[:16])


@pytest.mark.parametrize("chunk", [131072, MIB, 12 * MIB])
def test_stream_equals_the_batch_blocks(pkg, ctx, oracle, monkeypatch, chunk):
    _chunk(monkeypatch, chunk)
    data = planted(14 * MIB + 777, 74, OFFSETS + [9 * MIB])
    for level in (pkg.FASTEST, pkg.LAZY):
        fc = pkg.FrameCompressor(ctx, level, window_log=23)
        assert fc.window_log() == 23
        src, sink = Source(data, "rand", seed=chunk), Sink()
        fc.set_source(src)
        fc.set_drain(sink)
        r = fc.compress()
        frame = bytes(sink.buf)
        assert r["status"] == 0 and r["dst_size"] == len(frame)
        batch = pkg.compress_to_vec(ctx, data, level=level, window_log=23)
        hdr, blocks, tail = SF.split_frame(frame)
        bhdr, bblocks, btail = SF.split_frame(batch)
        assert hdr == struct.pack("<IBB", 0xFD2FB528, 4, (23 - 10) << 3) and tail == btail
        assert [b[1:] for b in blocks] == [b[1:] for b in bblocks]
        assert sum(b[1] == SF.COMPRESSED for b in blocks) > 0
        if chunk == MIB:
            assert datagen.decompress(frame, len(data), window_log_max=27) == data


def test_round_trips(pkg, ctx, oracle, tmp_path):
    big, mid, plain = inputs()
    frames, res = compress(pkg, ctx, plain, level=pkg.FASTEST, window_log=24)
    check_decodes(pkg, ctx, oracle, plain, frames, 24)
    whole = b"".join(frames)
    out = bytearray()
    pkg.decode_all_stream(ctx, io.BytesIO(whole), out)
    assert bytes(out) == b"".join(plain)
    got = np.zeros(sum(map(len, plain)) + 64, dtype=np.uint8)
    r = pkg.decode_all(ctx, np.frombuffer(whole, dtype=np.uint8), got)
    assert got[:sum(map(len, plain))].tobytes() == b"".join(plain), r
    for f, d in zip(frames, plain):
        assert pkg.StreamingDecoder(ctx, f).read_to_end() == d


def test_ratio_follows_the_window(pkg, ctx):
    base = np.random.default_rng(75).integers(0, 256, 8 * MIB, dtype=np.uint8).tobytes()
    data = base * 8
    f24 = pkg.compress_to_vec(ctx, data, window_log=24)
    f22 = pkg.compress_to_vec(ctx, data, window_log=22)
    assert len(f24) < 8.2 * MIB, len(f24)
    assert len(f22) > 63 * MIB, len(f22)
    out = np.zeros(len(data) + 64, dtype=np.uint8)
    pkg.decode_all(ctx, np.frombuffer(f24, dtype=np.uint8), out)
    assert out[:len(data)].tobytes() == data


def test_bad_arguments_are_refused_before_any_launch(pkg, ctx):
    big, mid, plain = inputs()
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}["B200Z_ERR_INVALID_ARGUMENT"]
    src = np.frombuffer(mid, dtype=np.uint8)
    cap = pkg.compress_bound(len(mid))
    out = np.zeros(cap, dtype=np.uint8)
    io_ = np.array([(0, len(mid), 0, cap)], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    res = np.zeros(1, dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
    other = pkg.Context(0)
    D = pkg.Dictionary.raw_content(other, 1, mid[:5000])
    before = ctx.kernel_launches()
    for level, wl, d in ((pkg.FASTEST, 16, None), (pkg.FASTEST, 28, None), (pkg.LAZY, 28, None), (pkg.UNCOMPRESSED, 18, None),
                         (pkg.FASTEST, 23, D)):
        assert L.b200z_compress_frames_batch_long(ctx.h, src.ctypes.data, src.size, 0, io_.ctypes.data, 1, level, 1, None if d is None else d.h, wl,
                                                  out.ctypes.data, out.size, 0, res.ctypes.data) == err
    fc = pkg.FrameCompressor(ctx)
    for wl in (16, 28):
        with pytest.raises(pkg.B200ZError):
            fc.set_window_log(wl)
    assert fc.window_log() == 17
    fc.set_compression_level(pkg.UNCOMPRESSED)
    fc.set_window_log(18)
    fc.set_source(mid)
    fc.set_drain(bytearray())
    with pytest.raises(pkg.B200ZError):
        fc.compress()
    assert ctx.kernel_launches() == before
    del D
    other.close()


def test_deterministic_across_runs_and_batch_shapes(pkg, ctx):
    big, mid, plain = inputs()
    a, _ = compress(pkg, ctx, plain, window_log=23)
    b, _ = compress(pkg, ctx, plain, window_log=23)
    c, _ = compress(pkg, ctx, plain[::-1], window_log=23)
    assert a == b == c[::-1]
    assert [compress(pkg, ctx, [d], window_log=23)[0][0] for d in plain] == a


class Repeat(io.RawIOBase):
    """`times` copies of `block`, read in pieces of at most the size asked for."""

    def __init__(self, block, times):
        self.block, self.left, self.at = block, times * len(block), 0

    def read(self, n):
        n = min(n, self.left)
        out = bytearray()
        while len(out) < n:
            k = self.at % len(self.block)
            take = min(n - len(out), len(self.block) - k)
            out += self.block[k:k + take]
            self.at += take
        self.left -= n
        return bytes(out)


class Count:
    def __init__(self):
        self.n = 0

    def write(self, b):
        self.n += len(b)
        return len(b)


def test_stream_memory_is_bounded(pkg, monkeypatch):
    """After a 1 GiB source the stream compressor holds what it held after a 64 MiB one (the header's formula sizes everything by
    the chunk and the window, not the source)."""
    monkeypatch.delenv("B200Z_PIPELINE_CHUNK_BYTES", raising=False)
    ctx = pkg.Context(0)
    plain = datagen.gen_text(64 << 20, 76).tobytes()
    fc = pkg.FrameCompressor(ctx, pkg.FASTEST, window_log=27)
    gc.collect()
    gc.disable()
    try:
        fc.set_source(Repeat(plain, 1))
        fc.set_drain(Count())
        r1 = fc.compress()
        dev1, pin1 = pkg.binding.held_bytes()
        fc.set_source(Repeat(plain, 16))
        fc.set_drain(Count())
        r2 = fc.compress()
        dev2, pin2 = pkg.binding.held_bytes()
    finally:
        gc.enable()
    assert r1["status"] == 0 and r2["status"] == 0
    assert dev2 == dev1 and pin2 == pin1, (dev1, dev2, pin1, pin2)
    assert r2["dst_size"] < 2 * r1["dst_size"]   # the 15 later copies lie within 2^27 of their source
    print(f"FrameCompressor at window_log 27 holds {dev1} device and {pin1} pinned bytes; 64 MiB -> {r1['dst_size']}, "
          f"1 GiB -> {r2['dst_size']}")
    del fc
    ctx.close()
