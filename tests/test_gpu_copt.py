"""The OPT level on the GPU against its plain model (tests/copt.py): every frame is the model's reference_frame byte for byte -- in
one submission and one frame per submission, from host and device memory, against raw-content and formatted dictionaries with and
without their tables (as test_gpu_cparse.py checks Fastest and LAZY), and with the long-distance matches of tests/cldm.py forced
at window_log 18, 23 and 27.  The frames round-trip through libzstd, the oracle and this library's decoder in both execution
modes and FrameDecoder; the output does not depend on the run or the batch; the ratio on 64 frames of C2b-shaped text is at least
libzstd level 3's and above LAZY's; FrameCompressor and the seekable writers at OPT write the batch compressor's blocks; and
levels 6 and 8 are refused before any launch."""
import functools

import numpy as np
import pytest

import cldm
import copt
import cparse
import datagen
import test_gpu_cldm as G
from test_compress import batch_decode, check_frames
from test_gpu_compress_stream import _chunk, check_fastest, run
from test_gpu_cparse import compress

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def opt(pkg, ctx, datas, **kw):
    return compress(pkg, ctx, datas, level=pkg.OPT, **kw)


CASES = copt.cases()
_models, _refs = {}, {}


def model(c):
    """The parse of case c at OPT, computed once."""
    if c.id not in _models:
        _models[c.id] = cparse.parse(c.frames, c.content, copt.OPT)
    return _models[c.id]


def reference(c, i, **kw):
    """reference_frame of frame i of case c at OPT, cached per options."""
    key = (c.id, i, tuple(sorted((k, v if not isinstance(v, bytes) else hash(v)) for k, v in kw.items())))
    if key not in _refs:
        _refs[key] = cparse.reference_frame(c.frames[i], model(c)[i], level=copt.OPT, **kw)
    return _refs[key]


def test_frames_are_the_models(pkg, ctx):
    """Every case without a dictionary: in one submission, and one frame per submission from host and device memory."""
    plain = [c for c in CASES if c.content is None]
    frames, _ = opt(pkg, ctx, [f for c in plain for f in c.frames])
    at = 0
    for c in plain:
        for i in range(len(c.frames)):
            assert frames[at + i] == reference(c, i), f"{c.id} frame {i}"
        at += len(c.frames)
    for c in plain:
        for i, data in enumerate(c.frames):
            for device in (False, True):
                assert opt(pkg, ctx, [data], device=device)[0][0] == reference(c, i), f"{c.id} frame {i} device={device}"


def test_frames_with_dictionaries_are_the_models(pkg, ctx):
    """Every case with a dictionary: against its raw content from host and device memory, and against the finalized dictionary
    with and without its tables."""
    for c in [c for c in CASES if c.content is not None]:
        R = pkg.Dictionary.raw_content(ctx, 1, c.content)
        for device in (False, True):
            frames, _ = opt(pkg, ctx, c.frames, dict=R, device=device)
            for i, f in enumerate(frames):
                assert f == reference(c, i), f"{c.id} frame {i} raw content device={device}"
        if len(c.content) < 8:                                           # the finalizer's smallest content
            continue
        fin = pkg.finalize_dict(ctx, c.content, c.frames[:50])
        assert fin.endswith(c.content)
        F = pkg.Dictionary.decode_dict(ctx, fin)
        for tables in (False, True):
            frames, _ = opt(pkg, ctx, c.frames, dict=F, dict_tables=tables)
            for i, f in enumerate(frames):
                want = reference(c, i, dict_id=F.id, dict_tables=fin if tables else None)
                assert f == want, f"{c.id} frame {i} finalized dictionary tables={tables}"


@functools.lru_cache(None)
def long_inputs():
    """A 1.5 MiB frame with repeats 131073 and 600,000 bytes back, and one block of it."""
    big = G.planted(3 * MIB // 2, 75, [131073, 600000])
    return [big, big[:cparse.BLOCK]]


@pytest.mark.parametrize("window_log", [18, 23, 27])
def test_long_frames_are_the_models(pkg, ctx, window_log):
    plain = long_inputs()
    blocks = cldm.parse(plain, window_log, None, copt.OPT)
    before = ctx.kernel_launches()
    frames, _ = opt(pkg, ctx, plain, window_log=window_log)
    assert ctx.kernel_launches() - before == 17 + 4   # the long-match kernels, then the four stages
    for i, (d, f) in enumerate(zip(plain, frames)):
        assert f == cparse.reference_frame(d, blocks[i], level=copt.OPT, window_log=window_log), f"frame {i}"
    assert any(o > cparse.BLOCK for o in cldm.offsets(blocks[0]))


@pytest.fixture(scope="module")
def texts():
    return [bytes(datagen.gen_text(3 * MIB + 5, 41)), bytes(datagen.gen_silesia_mix(2 * MIB, 42)),
            bytes(datagen.gen_binary_records(MIB + 7, 43)), b"\x2a" * 300000, b"", b"abcde"]


def test_round_trips(pkg, ctx, oracle, texts, monkeypatch):
    frames, res = opt(pkg, ctx, texts)
    check_frames(pkg, ctx, oracle, texts, frames, res)                  # libzstd, the oracle within the window, FrameDecoder
    for mode in ("cta", "warp"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        batch_decode(pkg, ctx, texts, frames)
    assert pkg.compress_to_vec(ctx, texts[0], level=pkg.OPT) == frames[0]


def test_deterministic_across_runs_and_batch_shapes(pkg, ctx, texts):
    a, _ = opt(pkg, ctx, texts)
    b, _ = opt(pkg, ctx, texts)
    c, _ = opt(pkg, ctx, texts[::-1])
    assert a == b == c[::-1]
    assert [opt(pkg, ctx, [t])[0][0] for t in texts] == a
    many = [t[:200000] for t in texts] * 150                            # more blocks than the grid's CTAs: each CTA takes several
    d, _ = opt(pkg, ctx, many)
    assert d[:len(texts)] == [opt(pkg, ctx, [t[:200000]])[0][0] for t in texts] and d == d[:len(texts)] * 150


def test_ratio_on_c2b_shaped_frames(pkg, ctx, oracle):
    plain = datagen.c2_text_plain(64 * 131072).tobytes()
    datas = [plain[i:i + 131072] for i in range(0, len(plain), 131072)]
    frames, res = opt(pkg, ctx, datas)
    check_frames(pkg, ctx, oracle, datas[:4], frames[:4], res[:4])
    ratio = len(plain) / sum(map(len, frames))
    lazy = len(plain) / sum(map(len, compress(pkg, ctx, datas, level=pkg.LAZY)[0]))
    zstd3 = len(plain) / sum(len(datagen.compress(d, level=3, window_log=17)) for d in datas)
    print(f"OPT {ratio:.3f}, LAZY {lazy:.3f}, libzstd level 3 {zstd3:.3f}")
    assert ratio >= zstd3 and ratio > lazy


@pytest.mark.parametrize("chunk", [131072, MIB, 12 * MIB])
def test_frame_compressor_equals_the_batch_blocks(pkg, ctx, texts, monkeypatch, chunk):
    C = _chunk(monkeypatch, chunk)
    fc = pkg.FrameCompressor(ctx, pkg.OPT)
    assert fc.compression_level() == pkg.OPT
    for data in texts:
        before = ctx.kernel_launches()
        frame, _ = run(fc, data, "rand", seed=len(data))
        assert ctx.kernel_launches() - before == 3 * -(-len(data) // C)
        check_fastest(pkg, data, frame, pkg.compress_to_vec(ctx, data, level=pkg.OPT))
    fc2 = pkg.FrameCompressor(ctx)
    assert fc2.set_compression_level(pkg.OPT) == pkg.FASTEST
    check_fastest(pkg, texts[0], run(fc2, texts[0])[0], pkg.compress_to_vec(ctx, texts[0], level=pkg.OPT))


def test_seekable_archive_is_the_batch_frames(pkg, ctx, texts):
    plain = texts[0][:MIB + 4321]
    fs = 262144
    arch = pkg.compress_seekable(ctx, plain, frame_size=fs, level=pkg.OPT)
    pieces = [plain[i:i + fs] for i in range(0, len(plain), fs)]
    frames, _ = opt(pkg, ctx, pieces)
    assert arch.startswith(b"".join(frames))
    assert pkg.compress_seekable(ctx, plain, frame_size=fs, level=pkg.LAZY) != arch


def test_levels_6_and_8_are_refused_before_any_launch(pkg, ctx):
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}
    src = np.zeros(1000, dtype=np.uint8)
    out = np.zeros(4096, dtype=np.uint8)
    io = np.array([(0, 1000, 0, pkg.compress_bound(1000))], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    res = np.zeros(1, dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
    before = ctx.kernel_launches()
    for level in (6, 8):
        assert L.b200z_compress_frames_batch(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, 1, level, 1, out.ctypes.data, out.size, 0,
                                             res.ctypes.data) == err["B200Z_ERR_INVALID_ARGUMENT"]
        with pytest.raises(pkg.B200ZError):
            pkg.FrameCompressor(ctx, level)
    fc = pkg.FrameCompressor(ctx, pkg.OPT)
    with pytest.raises(pkg.B200ZError):
        fc.set_compression_level(8)
    assert fc.compression_level() == pkg.OPT
    assert ctx.kernel_launches() == before
