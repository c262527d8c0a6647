"""The LAZY level on the GPU against its plain model (tests/clazy.py): every frame is the model's reference_frame byte for byte --
in one submission and one frame per submission, from host and device memory, against raw-content and formatted dictionaries
with and without their tables, by the checks test_gpu_cparse.py runs at Fastest.  The frames round-trip through libzstd, the
oracle and this library's decoder in both execution modes and FrameDecoder; the output does not depend on the run or the batch;
the ratio on 64 frames of C2b-shaped text is at least libzstd level 1's and above Fastest's; FrameCompressor at LAZY writes the
batch compressor's blocks; and an unknown level is refused before any launch."""
import numpy as np
import pytest

import datagen
from test_compress import batch_decode, check_frames
from test_gpu_compress_stream import _chunk, check_fastest, run
from test_gpu_cparse import check_reference_frames, check_reference_frames_with_dictionaries, compress

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def lazy(pkg, ctx, datas, **kw):
    return compress(pkg, ctx, datas, level=pkg.LAZY, **kw)


def test_frames_are_the_models(pkg, ctx):
    check_reference_frames(pkg, ctx, "lazy")


def test_frames_with_dictionaries_are_the_models(pkg, ctx):
    check_reference_frames_with_dictionaries(pkg, ctx, "lazy")


@pytest.fixture(scope="module")
def texts():
    return [bytes(datagen.gen_text(3 * MIB + 5, 41)), bytes(datagen.gen_silesia_mix(2 * MIB, 42)),
            bytes(datagen.gen_binary_records(MIB + 7, 43)), b"\x2a" * 300000, b"", b"abcde"]


def test_round_trips(pkg, ctx, oracle, texts, monkeypatch):
    frames, res = lazy(pkg, ctx, texts)
    check_frames(pkg, ctx, oracle, texts, frames, res)                  # libzstd, the oracle within the window, FrameDecoder
    for mode in ("cta", "warp"):
        monkeypatch.setenv("B200Z_EXEC_MODE", mode)
        batch_decode(pkg, ctx, texts, frames)
    assert pkg.compress_to_vec(ctx, texts[0], level=pkg.LAZY) == frames[0]


def test_deterministic_across_runs_and_batch_shapes(pkg, ctx, texts):
    a, _ = lazy(pkg, ctx, texts)
    b, _ = lazy(pkg, ctx, texts)
    c, _ = lazy(pkg, ctx, texts[::-1])
    assert a == b == c[::-1]
    assert [lazy(pkg, ctx, [t])[0][0] for t in texts] == a


def test_ratio_on_c2b_shaped_frames(pkg, ctx, oracle):
    plain = datagen.c2_text_plain(64 * 131072).tobytes()
    datas = [plain[i:i + 131072] for i in range(0, len(plain), 131072)]
    frames, res = lazy(pkg, ctx, datas)
    check_frames(pkg, ctx, oracle, datas[:4], frames[:4], res[:4])
    ratio = len(plain) / sum(map(len, frames))
    fastest = len(plain) / sum(map(len, compress(pkg, ctx, datas, level=pkg.FASTEST)[0]))
    zstd1 = len(plain) / sum(len(datagen.compress(d, level=1, window_log=17)) for d in datas)
    print(f"LAZY {ratio:.3f}, Fastest {fastest:.3f}, libzstd level 1 {zstd1:.3f}")
    assert ratio >= zstd1 and ratio > fastest


@pytest.mark.parametrize("chunk", [131072, 262144, MIB])
def test_frame_compressor_equals_the_batch_blocks(pkg, ctx, texts, monkeypatch, chunk):
    C = _chunk(monkeypatch, chunk)
    fc = pkg.FrameCompressor(ctx, pkg.LAZY)
    assert fc.compression_level() == pkg.LAZY
    for data in texts:
        before = ctx.kernel_launches()
        frame, _ = run(fc, data, "rand", seed=len(data))
        assert ctx.kernel_launches() - before == 3 * -(-len(data) // C)
        check_fastest(pkg, data, frame, pkg.compress_to_vec(ctx, data, level=pkg.LAZY))
    fc2 = pkg.FrameCompressor(ctx)
    assert fc2.set_compression_level(pkg.LAZY) == pkg.FASTEST
    check_fastest(pkg, texts[0], run(fc2, texts[0])[0], pkg.compress_to_vec(ctx, texts[0], level=pkg.LAZY))


def test_unknown_level_is_refused_before_any_launch(pkg, ctx):
    L = pkg.lib()
    err = {v: k for k, v in pkg.error_names().items()}
    src = np.zeros(1000, dtype=np.uint8)
    out = np.zeros(4096, dtype=np.uint8)
    io = np.array([(0, 1000, 0, pkg.compress_bound(1000))], dtype=pkg.binding.COMPRESS_IO_DTYPE)
    res = np.zeros(1, dtype=pkg.binding.COMPRESS_RESULT_DTYPE)
    before = ctx.kernel_launches()
    for level, want in ((6, "B200Z_ERR_INVALID_ARGUMENT"), (2, "B200Z_ERR_REFERENCE_WOULD_PANIC"), (4, "B200Z_ERR_REFERENCE_WOULD_PANIC")):
        assert L.b200z_compress_frames_batch(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, 1, level, 1, out.ctypes.data, out.size, 0,
                                             res.ctypes.data) == err[want]
        assert L.b200z_compress_frames_batch_dict(ctx.h, src.ctypes.data, src.size, 0, io.ctypes.data, 1, level, 1, None, out.ctypes.data,
                                                  out.size, 0, res.ctypes.data) == err[want]
    with pytest.raises(pkg.B200ZError):
        pkg.FrameCompressor(ctx, 6)
    fc = pkg.FrameCompressor(ctx, pkg.LAZY)
    with pytest.raises(pkg.B200ZError):
        fc.set_compression_level(6)
    assert fc.compression_level() == pkg.LAZY
    assert ctx.kernel_launches() == before
