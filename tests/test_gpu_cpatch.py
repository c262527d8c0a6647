"""Long matches into a dictionary on the GPU (B200Z_FLAG_DICT_LONG): the batch compressor's frames equal tests/cpatch.py's byte for
byte at every level, with raw-content and formatted dictionaries, host and device memory, one and many frames and a dictionary
larger than 2^27 bytes; they decode everywhere; the flag changes nothing where it should not; the dictionary's anchors cost the
documented launches and memory once; submissions split differently write the same bytes; compress_patch_from is the model's frame."""
import functools
import gc
import io

import numpy as np
import pytest

import cldm
import cparse
import cpatch
import datagen
from test_cpatch_model import LEVELS, edited, level_of, positioned, rand

pytestmark = pytest.mark.gpu

MIB = 1 << 20
WL = 23


def compress(pkg, ctx, datas, dict=None, level=1, window_log=WL, dict_long=True, device=False, **kw):
    """compress_frames over datas laid out back to back; returns the frames."""
    fio = np.zeros(len(datas), dtype=pkg.binding.COMPRESS_IO_DTYPE)
    so = oo = 0
    for i, d in enumerate(datas):
        cap = pkg.compress_bound(len(d), dict)
        fio[i] = (so, len(d), oo, cap)
        so += len(d)
        oo += cap
    src = np.frombuffer(b"".join(datas), dtype=np.uint8)
    out = np.zeros(oo, dtype=np.uint8)
    if device:
        import torch
        src_t, out_t = torch.from_numpy(src.copy()).cuda(), torch.zeros(out.size, dtype=torch.uint8, device="cuda")
        res = pkg.compress_frames(ctx, src_t, fio, out_t, level, True, dict, window_log=window_log, dict_long=dict_long, **kw)
        out = out_t.cpu().numpy()
    else:
        res = pkg.compress_frames(ctx, src, fio, out, level, True, dict, window_log=window_log, dict_long=dict_long, **kw)
    assert (res["status"] == 0).all()
    return [out[fio[i]["dst_off"]:fio[i]["dst_off"] + res[i]["dst_size"]].tobytes() for i in range(len(datas))]


@functools.lru_cache(None)
def inputs():
    """(D, datas): 400,000 bytes of text; an edited copy of its last 200,000 bytes, one of its first 60,000, and 300,000 bytes of new
    text holding a third edited copy of 100,000 bytes of D."""
    D = datagen.gen_text(400000, 81).tobytes()
    new = datagen.gen_text(300000, 92).tobytes()
    return D, [edited(D[200000:], 82), edited(D[:60000], 83), new[:100000] + edited(D[150000:250000], 93) + new[200000:]]


_parses = {}


def parse(datas, name, D, window_log=WL):
    key = (hash(tuple(datas)), name, hash(D), window_log)
    if key not in _parses:
        _parses[key] = cpatch.parse(datas, window_log, D, level_of(name, window_log))
    return _parses[key]


def reference(datas, blocks, name, D, window_log=WL, **kw):
    lv = level_of(name, window_log)
    return [cpatch.reference_frame(d, b, window_log, len(D), level=lv, **kw) for d, b in zip(datas, blocks)]


LEVEL = {"fastest": 1, "lazy": 5, "opt": 7, "ultra": 10}


@functools.lru_cache(None)
def formatted(pkg, ctx):
    D, datas = inputs()
    return pkg.finalize_dict(ctx, D, [datas[2][i:i + 4096] for i in range(0, 300000, 4096)], dict_id=9)


@pytest.mark.parametrize("kind", ["raw", "formatted", "formatted-tables"])
@pytest.mark.parametrize("name", LEVELS)
def test_frames_equal_the_model(pkg, ctx, name, kind):
    D, datas = inputs()
    blocks = parse(datas, name, D)
    if kind == "raw":
        R, kw, ref = pkg.Dictionary.raw_content(ctx, 1, D), {}, {}
    else:
        fin = formatted(pkg, ctx)
        R = pkg.Dictionary.decode_dict(ctx, fin)
        tables = kind == "formatted-tables"
        kw, ref = {"dict_tables": tables}, {"dict_id": 9, "dict_tables": fin if tables else None}
    want = reference(datas, blocks, name, D, **ref)
    assert compress(pkg, ctx, datas, R, LEVEL[name], **kw) == want
    assert compress(pkg, ctx, datas[:1], R, LEVEL[name], device=True, **kw) == want[:1]
    assert 400000 in [o for p, o in positioned(blocks[1]) if o > p]


def test_dictionary_larger_than_2_27(pkg, ctx):
    D = rand((1 << 27) + MIB, 94)
    X = bytearray(rand(300000, 95))
    X[1000:11000] = D[len(D) - (1 << 27) + 2000:len(D) - (1 << 27) + 12000]   # offset 2^27 - 1000: taken
    X[50000:60000] = D[100000:110000]                                      # before D's last 2^27 bytes: not
    X[200000:230000] = D[-40000:-10000]
    X = bytes(X)
    blocks = cpatch.parse([X], 27, D)
    offs = cldm.offsets(blocks[0])
    assert (1 << 27) - 1000 in offs and 200000 + 40000 in offs
    assert all(o <= 1 << 27 for o in offs)
    R = pkg.Dictionary.raw_content(ctx, 0, D)
    got = compress(pkg, ctx, [X], R, window_log=27)
    assert got == [cpatch.reference_frame(X, blocks[0], 27, len(D))]
    assert got[0][5] == (27 - 10) << 3
    assert datagen.decompress(got[0], len(X), raw_dict=D, window_log_max=27) == X


def test_frames_decode_everywhere(pkg, ctx):
    D, datas = inputs()
    R = pkg.Dictionary.raw_content(ctx, 1, D)
    frames = compress(pkg, ctx, datas, R, window_log=24)
    whole = b"".join(frames)
    plain = b"".join(datas)
    for f, d in zip(frames, datas):
        assert datagen.decompress(f, len(d), raw_dict=D, window_log_max=27) == d
        dec = pkg.FrameDecoder(ctx)
        dec.set_max_window_size(1 << 27)
        dec.add_raw_content_dict(1, D)
        r = dec.reset(f)
        dec.force_dict(1)
        dec.decode_blocks(r)
        assert dec.collect() == d
    fio = np.zeros(len(frames), dtype=pkg.binding.FRAME_IO_DTYPE)
    so = oo = 0
    for i, (f, d) in enumerate(zip(frames, datas)):
        fio[i] = (so, len(f), oo, len(d))
        so += len(f)
        oo += len(d)
    out = np.zeros(oo, dtype=np.uint8)
    res = pkg.decode_frames(ctx, np.frombuffer(whole, dtype=np.uint8), fio, out, forced_dict=R, max_window_size=1 << 27)
    assert (res["status"] == 0).all() and out.tobytes() == plain
    out = np.zeros(len(plain) + 64, dtype=np.uint8)
    r, _ = pkg.decode_all(ctx, np.frombuffer(whole, dtype=np.uint8), out, forced_dict=R, max_window_size=1 << 27)
    assert r["status"] == 0 and out[:len(plain)].tobytes() == plain, r
    sink = bytearray()
    pkg.decode_all_stream(ctx, io.BytesIO(whole), sink, forced_dict=R, max_window_size=1 << 27)
    assert bytes(sink) == plain
    F = pkg.Dictionary.decode_dict(ctx, formatted(pkg, ctx))   # by the frames' dictionary ID
    fframes = compress(pkg, ctx, datas, F, window_log=24)
    out = np.zeros(len(plain) + 64, dtype=np.uint8)
    r, _ = pkg.decode_all(ctx, np.frombuffer(b"".join(fframes), dtype=np.uint8), out, dicts=[F], max_window_size=1 << 27)
    assert r["status"] == 0 and out[:len(plain)].tobytes() == plain, r


def test_the_flag_is_inert_where_it_should_be(pkg, ctx):
    D, datas = inputs()
    R = pkg.Dictionary.raw_content(ctx, 1, D)
    compress(pkg, ctx, datas, R, 1, 17, dict_long=False)   # builds the dictionary's match table first
    for level, wl, d in ((1, WL, None), (5, WL, None), (1, 17, R), (7, 17, R), (0, 17, R), (0, 17, None)):
        before = ctx.kernel_launches()
        a = compress(pkg, ctx, datas, d, level, wl, dict_long=False)
        mid = ctx.kernel_launches()
        b = compress(pkg, ctx, datas, d, level, wl, dict_long=True)
        assert a == b, (level, wl, d is None)
        assert ctx.kernel_launches() - mid == mid - before


def test_first_use_launches_and_memory(pkg, ctx):
    D, datas = inputs()
    n = len(cpatch.dict_anchors(D)[0])
    big = pkg.Dictionary.raw_content(ctx, 2, rand(2 * MIB, 96))   # grows the context's long-match scratch beyond D's needs
    compress(pkg, ctx, datas, big)
    del big
    gc.collect()
    dev0, _ = pkg.binding.held_bytes()
    R = pkg.Dictionary.raw_content(ctx, 1, D)
    compress(pkg, ctx, datas, R, dict_long=False)   # builds the dictionary's match table
    dev1, _ = pkg.binding.held_bytes()
    counts, held = [], []
    for _ in range(2):
        before = ctx.kernel_launches()
        compress(pkg, ctx, datas, R)
        counts.append(ctx.kernel_launches() - before)
        held.append(pkg.binding.held_bytes()[0])
    assert counts == [16 + 17 + 4, 17 + 4]      # the anchor build once; then the long-match kernels and the four stages
    assert held[0] - dev1 == 8 * n and held[1] == held[0], (dev1, held, n)
    del R
    gc.collect()
    assert pkg.binding.held_bytes()[0] == dev0


def test_deterministic_across_submissions(pkg, ctx):
    D, datas = inputs()
    R = pkg.Dictionary.raw_content(ctx, 1, D)
    for level in (1, 7):
        a = compress(pkg, ctx, datas, R, level)
        b = compress(pkg, ctx, datas[:1], R, level) + compress(pkg, ctx, datas[1:], R, level)
        c = compress(pkg, ctx, datas[::-1], R, level)[::-1]
        assert a == b == c


def test_compress_patch_from(pkg, ctx):
    base = datagen.gen_text(2 * MIB, 90).tobytes()
    copy = edited(base, 91)
    wl = pkg.patch_window_log(len(base), len(copy))
    assert wl == 22
    f = pkg.compress_patch_from(ctx, base, copy)
    blocks = cpatch.parse([copy], wl, base)
    assert f == cpatch.reference_frame(copy, blocks[0], wl, len(base))
    assert len(copy) / len(f) >= 20
    R = pkg.Dictionary.raw_content(ctx, 0, base)
    out = np.zeros(len(copy) + 64, dtype=np.uint8)
    r, _ = pkg.decode_all(ctx, np.frombuffer(f, dtype=np.uint8), out, forced_dict=R, max_window_size=1 << 27)
    assert r["status"] == 0 and out[:len(copy)].tobytes() == copy
    assert datagen.decompress(f, len(copy), raw_dict=base, window_log_max=27) == copy
