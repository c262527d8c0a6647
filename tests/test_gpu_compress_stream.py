"""The stream compressor (FrameCompressor / compress, b200z_frame_compressor) on the GPU.

Uncompressed must be the framing model of tests/streamframe.py byte for byte, with no kernel launched, whatever the reads return.
Fastest must frame its blocks as the model does, and every non-empty block must equal, type, size and body, the same block of
the batch compressor's frame of the same input (only the last-block bit may differ, where the stream adds an empty last block).
Every frame must decode with libzstd, the oracle (offsets within the 128 KiB window) and this library's decoders, and carry the
input's checksum.  Chunk sizes are set through B200Z_PIPELINE_CHUNK_BYTES, which a compressor reads when it is created."""
import io
import random
import struct

import numpy as np
import pytest

import datagen
import streamframe as SF
from test_compress import within_window

pytestmark = pytest.mark.gpu

B = SF.BLOCK
MIB = 1 << 20
CHUNKS = [131072, 262144, MIB, None]   # None: the default chunk (64 MiB)


class Source:
    """A reader that counts its calls: `all` returns what is asked for, `one` a byte per call, `rand` seeded random short reads;
    `fail_at` raises on that call."""

    def __init__(self, data, mode="all", seed=0, fail_at=None):
        self.b, self.mode, self.rng, self.fail_at, self.calls = io.BytesIO(data), mode, random.Random(seed), fail_at, 0

    def read(self, n):
        self.calls += 1
        if self.calls == self.fail_at:
            raise OSError("the source failed")
        if self.mode == "one":
            n = min(n, 1)
        elif self.mode == "rand" and n > 1:
            n = self.rng.randint(1, n)
        return self.b.read(n)


class Sink:
    """A writer that counts its calls; `zero_at` returns 0 (nothing written) on that call."""

    def __init__(self, zero_at=None):
        self.buf, self.calls, self.zero_at = bytearray(), 0, zero_at

    def write(self, b):
        self.calls += 1
        if self.calls == self.zero_at:
            return 0
        self.buf += b
        return len(b)


def _err(pkg, name):
    return {v: k for k, v in pkg.error_names().items()}["B200Z_ERR_" + name]


def _chunk(monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("B200Z_PIPELINE_CHUNK_BYTES", raising=False)
        return 64 * MIB
    monkeypatch.setenv("B200Z_PIPELINE_CHUNK_BYTES", str(chunk))
    return chunk


def run(fc, data, mode="all", seed=0):
    src, sink = Source(data, mode, seed), Sink()
    fc.set_source(src)
    fc.set_drain(sink)
    res = fc.compress()
    assert res["status"] == 0 and res["dst_size"] == len(sink.buf)
    return bytes(sink.buf), res


@pytest.fixture(scope="module")
def inputs():
    ins = {f"text{n}": bytes(datagen.gen_text(n, 31 + n)) if n else b"" for n in
           (0, 1, B - 1, B, B + 1, 2 * B, 3 * B, MIB - 1, MIB, MIB + 1, 2 * MIB + B)}
    ins["text9m5"] = bytes(datagen.gen_text(9 * MIB + 5, 32))
    ins["silesia"] = bytes(datagen.gen_silesia_mix(3 * MIB, 23))
    ins["rle300k"] = b"\x2a" * (300 << 10)
    ins["random1m"] = np.random.default_rng(3).integers(0, 256, MIB, dtype=np.uint8).tobytes()
    return ins


# ---------------------------------------------------------------------------------------------------- Uncompressed
@pytest.mark.parametrize("chunk", [131072, None])
def test_uncompressed_is_the_model(pkg, ctx, monkeypatch, chunk):
    _chunk(monkeypatch, chunk)
    rng = np.random.default_rng(5)
    for checksum in (True, False):
        fc = pkg.FrameCompressor(ctx, pkg.UNCOMPRESSED, checksum)
        for n in (0, 1, B - 1, B, B + 1, 3 * B, 5 * MIB + 3):
            data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            want = SF.uncompressed_frame(data, checksum, pkg.xxh64)
            for mode in ("all", "one", "rand"):
                if mode == "one" and n > 140 << 10:
                    continue
                before = ctx.kernel_launches()
                got, res = run(fc, data, mode, seed=n)
                assert ctx.kernel_launches() == before
                assert got == want, (n, checksum, mode)
                assert res["blocks"] == res["raw_blocks"] == len(SF.pieces(data)) and res["rle_blocks"] == 0
                assert res["has_checksum"] == int(checksum)
                if checksum:
                    assert res["checksum"] == pkg.xxh64(data) & 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------- Fastest
def check_fastest(pkg, data, frame, batch, checksum=True):
    """`frame` (the stream's) is framed as the model says and its non-empty blocks equal the batch frame's."""
    hdr, blocks, tail = SF.split_frame(frame)
    _, bblocks, btail = SF.split_frame(batch)
    model = SF.pieces(data)
    assert hdr == SF.header(checksum) and tail == SF.trailer(data, checksum, pkg.xxh64)
    assert len(blocks) == len(model)
    for (last, t, size, body), (piece, mlast) in zip(blocks, model):
        assert last == int(mlast)
        if t != SF.COMPRESSED:
            assert size == len(piece)
        assert body == (piece if t == SF.RAW else piece[:1] if t == SF.RLE else body)
    full = [b for b, (piece, _) in zip(blocks, model) if piece]
    assert [b[1:] for b in full] == [b[1:] for b in bblocks[:len(full)]]
    if not data:
        assert blocks == bblocks
    if checksum:
        assert tail == btail


@pytest.mark.parametrize("chunk", CHUNKS)
def test_fastest_equals_the_batch_compressor(pkg, ctx, inputs, monkeypatch, chunk):
    C = _chunk(monkeypatch, chunk)
    fc = pkg.FrameCompressor(ctx)
    for name in sorted(inputs):
        data = inputs[name]
        before = ctx.kernel_launches()
        frame, res = run(fc, data, "rand" if name == "silesia" else "all", seed=len(data))
        assert ctx.kernel_launches() - before == 3 * -(-len(data) // C), name
        check_fastest(pkg, data, frame, pkg.compress_to_vec(ctx, data))
        blocks = SF.split_frame(frame)[1]
        assert res["blocks"] == len(blocks)
        assert res["raw_blocks"] == sum(t == SF.RAW for _, t, _, _ in blocks) and res["rle_blocks"] == sum(t == SF.RLE for _, t, _, _ in blocks)
    if chunk == 131072:
        assert SF.split_frame(run(fc, inputs["rle300k"])[0])[1][0][1] == SF.RLE
        assert all(t == SF.RAW for _, t, _, _ in SF.split_frame(run(fc, inputs["random1m"])[0])[1])


@pytest.mark.parametrize("chunk", [131072, MIB])
def test_round_trip(pkg, ctx, oracle, inputs, monkeypatch, chunk):
    _chunk(monkeypatch, chunk)
    for level in (pkg.FASTEST, pkg.UNCOMPRESSED):
        fc = pkg.FrameCompressor(ctx, level)
        dec = pkg.FrameDecoder(ctx)
        for name in ("text0", "text1", f"text{B}", f"text{MIB + 1}", "text9m5", "silesia", "rle300k", "random1m"):
            data = inputs[name]
            frame, res = run(fc, data)
            want = pkg.xxh64(data) & 0xFFFFFFFF
            assert struct.unpack("<I", frame[-4:])[0] == want and res["checksum"] == want and res["has_checksum"] == 1
            assert datagen.decompress(frame, len(data)) == data, name
            assert within_window(oracle, frame) == data, name
            assert pkg.StreamingDecoder(ctx, frame).read_to_end() == data, name
            assert dec.decode_all(frame, len(data)) == data, name


def test_without_checksum(pkg, ctx, oracle, inputs, monkeypatch):
    _chunk(monkeypatch, 262144)
    fc = pkg.FrameCompressor(ctx, checksum=False)
    for name in ("text0", f"text{2 * B}", "text9m5"):
        data = inputs[name]
        frame, res = run(fc, data)
        assert res["has_checksum"] == 0
        check_fastest(pkg, data, frame, pkg.compress_to_vec(ctx, data, checksum=False), checksum=False)
        assert datagen.decompress(frame, len(data)) == data and oracle.decode_frame(frame)[0] == data


# ---------------------------------------------------------------------------------------------------- reuse, interface
def test_reuse_and_level_change(pkg, ctx, inputs, monkeypatch):
    _chunk(monkeypatch, 262144)
    data = inputs["silesia"]
    fc = pkg.FrameCompressor(ctx)
    a, _ = run(fc, data)
    b, _ = run(fc, data, "rand", seed=9)
    assert a == b
    fc0 = pkg.FrameCompressor(ctx, pkg.UNCOMPRESSED)
    assert fc0.compression_level() == pkg.UNCOMPRESSED
    assert run(fc0, data)[0] == SF.uncompressed_frame(data, True, pkg.xxh64)
    assert fc0.set_compression_level(pkg.FASTEST) == pkg.UNCOMPRESSED and fc0.compression_level() == pkg.FASTEST
    assert run(fc0, data)[0] == a


def test_sources_drains_and_compress(pkg, ctx, inputs):
    data = inputs[f"text{MIB + 1}"]
    want = run(pkg.FrameCompressor(ctx), data)[0]
    fc = pkg.FrameCompressor(ctx)
    assert fc.source() is None and fc.set_source(data) is None and fc.source() is data
    out = bytearray()
    assert fc.set_drain(out) is None and fc.drain() is out
    fc.compress()
    assert bytes(out) == want
    assert fc.take_source() is data and fc.source() is None and fc.take_drain() is out and fc.drain() is None
    with pytest.raises(pkg.B200ZError):
        fc.compress()
    f = io.BytesIO()
    res = pkg.compress(ctx, io.BytesIO(data), f)
    assert f.getvalue() == want and res["dst_size"] == len(want)
    ba = bytearray(b"prefix")
    pkg.compress(ctx, data, ba, level=pkg.UNCOMPRESSED, checksum=False)
    assert bytes(ba) == b"prefix" + SF.uncompressed_frame(data, False, pkg.xxh64)


# ---------------------------------------------------------------------------------------------------- rejections, failures
def test_rejections(pkg, ctx):
    L = pkg.lib()
    for level in (2, 3, 4):
        fc = pkg.FrameCompressor(ctx, level)
        src, sink = Source(b"abc" * 1000), Sink()
        fc.set_source(src)
        fc.set_drain(sink)
        before = ctx.kernel_launches()
        with pytest.raises(pkg.B200ZError) as e:
            fc.compress()
        assert e.value.code == _err(pkg, "REFERENCE_WOULD_PANIC")
        assert src.calls == 0 and sink.calls == 0 and ctx.kernel_launches() == before
    with pytest.raises(pkg.B200ZError) as e:
        pkg.FrameCompressor(ctx, 9)
    assert e.value.code == _err(pkg, "INVALID_ARGUMENT")
    fc = pkg.FrameCompressor(ctx)
    with pytest.raises(pkg.B200ZError) as e:
        fc.set_compression_level(-1)
    assert e.value.code == _err(pkg, "INVALID_ARGUMENT") and fc.compression_level() == pkg.FASTEST
    assert L.b200z_frame_compressor_compression_level(fc.h) == pkg.FASTEST


@pytest.mark.parametrize("level", [0, 1])
def test_failing_source_and_drain_leave_the_compressor_usable(pkg, ctx, inputs, monkeypatch, level):
    _chunk(monkeypatch, 131072)
    data = inputs["silesia"]
    want = run(pkg.FrameCompressor(ctx, level), data)[0]
    fc = pkg.FrameCompressor(ctx, level)
    # the Uncompressed level reads block by block, Fastest chunk by chunk: with 128 KiB chunks the third read is the third block
    src, sink = Source(data, fail_at=3), Sink()
    fc.set_source(src)
    fc.set_drain(sink)
    with pytest.raises(pkg.B200ZError) as e:
        fc.compress()
    assert e.value.code == _err(pkg, "REFERENCE_WOULD_PANIC") and isinstance(e.value.__cause__, OSError)
    assert want.startswith(bytes(sink.buf))
    assert run(fc, data)[0] == want
    src, sink = Source(data), Sink(zero_at=2)
    fc.set_source(src)
    fc.set_drain(sink)
    with pytest.raises(pkg.B200ZError) as e:
        fc.compress()
    assert e.value.code == _err(pkg, "REFERENCE_WOULD_PANIC")
    assert sink.calls == 2 and want.startswith(bytes(sink.buf)) and len(sink.buf) > 0
    assert run(fc, data)[0] == want
