"""Long matches into a dictionary (B200Z_FLAG_DICT_LONG, tests/cpatch.py) on the CPU: the model's frames decode to their
input with libzstd and the oracle within their own Window_Descriptor at every level and window_log, the offset edges into the
dictionary, the nearest-anchor rule, small frames, the cases where the flag changes nothing, and the ratio on an edited copy."""
import functools

import numpy as np
import pytest

import clazy
import cldm
import copt
import cparse
import cpatch
import cultra
import datagen

B = cldm.BLOCK
MIB = 1 << 20
LEVELS = ["fastest", "lazy", "opt", "ultra"]


def level_of(name, window_log):
    return {"fastest": cparse.FASTEST, "lazy": clazy.LAZY, "opt": copt.OPT}[name] if name != "ultra" else cultra.level(window_log)


def model(frames, window_log, name, content, dict_long=True, **kw):
    """(blocks, frames) of the model: the parse with the flag, and the frames the compressor must write for it."""
    lv = level_of(name, window_log)
    blocks = cpatch.parse(frames, window_log, content, lv, dict_long)
    dl = cpatch.header_dict_len(content, window_log, dict_long)
    return blocks, [cpatch.reference_frame(f, b, window_log, dl, level=lv, **kw) for f, b in zip(frames, blocks)]


def positioned(blocks):
    """(frame position, offset) of every sequence of a frame's parse."""
    out = []
    for k, b in enumerate(blocks):
        if b[0] == "rle":
            continue
        pos = k * B
        for ll, ml, of in b[1]:
            out.append((pos + ll, of))
            pos += ll + ml
    return out


def edited(base, seed):
    """bench_compress_patch.py's copy of `base`: about 1 % of its bytes replaced by seeded random runs of 1-32 bytes."""
    rng = np.random.default_rng(seed)
    v = np.frombuffer(bytes(base), dtype=np.uint8).copy()
    n = len(v)
    runs = int(0.01 * n / 16.5)
    at = rng.integers(0, n - 32, runs)
    ln = rng.integers(1, 33, runs)
    for a, k in zip(at.tolist(), ln.tolist()):
        v[a:a + k] = rng.integers(0, 256, k, dtype=np.uint8)
    return v.tobytes()


def rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


@functools.lru_cache(None)
def versions():
    """(D, frames): 400,000 bytes of text as the dictionary; an edited copy of its last 200,000 bytes (offset 200,000 into D) and
    one of its first 60,000 (offset 400,000: beyond 2^18)."""
    D = datagen.gen_text(400000, 81).tobytes()
    return D, [edited(D[200000:], 82), edited(D[:60000], 83)]


def trace(oracle, frame, formatted):
    o = oracle.FrameDecoder()
    o.set_max_window_size(1 << 27)
    o.trace_enable()
    o.add_dict(formatted)
    r = o.reset(frame)
    o.decode_blocks(r)
    return o, o.collect(), o.trace()[2]


@pytest.mark.parametrize("window_log", [18, 23, 27])
@pytest.mark.parametrize("name", LEVELS)
def test_model_frames_decode_within_their_window(pkg, oracle, name, window_log):
    D, datas = versions()
    blocks, frames = model(datas, window_log, name, D)
    formatted = pkg.dict_from_counts(np.zeros(cparse.DS_BINS, dtype=np.uint64) + 3, D, dict_id=7)
    _, fframes = model(datas, window_log, name, D, dict_id=7)
    into = []
    for d, bl, f, ff in zip(datas, blocks, frames, fframes):
        wl = cpatch.frame_window_log(len(d), window_log, len(D))
        assert f[5] == (wl - 10) << 3
        assert datagen.decompress(f, len(d), raw_dict=D, window_log_max=27) == d
        o, out, seqs = trace(oracle, ff, formatted)
        assert out == d and o.window_size() == 1 << wl
        assert len(seqs) == 0 or int(seqs[:, 3].max()) <= 1 << wl
        for pos, of in positioned(bl):
            assert of <= min(pos + len(D), 1 << wl)
            if of > pos:
                into.append(of)
    assert 200000 in into                                   # the first copy's source, at every window_log
    assert (400000 in into) == (window_log > 18)            # the second's lies beyond 2^18


@pytest.mark.parametrize("name", LEVELS)
def test_offset_edges_into_the_dictionary(name):
    wl = 18
    D = rand(600000, 84)
    X = bytearray(rand(100000, 85))
    edges = {131072: 10000, 131073: 30000, 1 << wl: 50000, (1 << wl) + 1: 70000}
    for o, p in edges.items():
        X[p:p + 3000] = D[len(D) + p - o:len(D) + p - o + 3000]
    X = bytes(X)
    offs = set(cldm.offsets(cpatch.parse([X], wl, D, level_of(name, wl))[0]))
    assert {131072, 131073, 1 << wl} <= offs and (1 << wl) + 1 not in offs
    off = set(cldm.offsets(cldm.parse([X], wl, D, level_of(name, wl))[0]))
    assert 131072 in off and not ({131073, 1 << wl} & off)   # 131072 is the regular parse's reach into the dictionary


def test_the_nearest_anchor_is_the_frames():
    wl = 23
    D = rand(MIB, 86)
    R = D[500000:504000]
    X = bytearray(rand(400000, 87))
    X[10000:14000] = R         # taken from D; its copy 190,000 bytes later takes the frame's (a kept offset)
    X[200000:204000] = R
    X[250000:254000] = R       # 50,000 after that copy: the nearest is out of range, so no long match, and none from D
    offs = cldm.offsets(cpatch.parse([bytes(X)], wl, D)[0])
    into = lambda p: p + len(D) - 500000
    assert into(10000) in offs and 190000 in offs
    assert into(200000) not in offs and into(250000) not in offs
    cands = cpatch.candidates([bytes(X)], wl, D)[0]
    assert all(o == 190000 for p, o in cands if 200000 <= p < 204000)
    assert not [1 for p, o in cands if 250000 <= p < 254000]


def test_small_frames_reach_megabytes_back():
    wl = 23
    D = rand(3 * MIB, 88)
    X = bytearray(rand(100000, 89))
    X[20000:40000] = D[500000:520000]
    X = bytes(X)
    blocks, frames = model([X], wl, "fastest", D)
    assert 20000 + len(D) - 500000 in cldm.offsets(blocks[0])
    assert frames[0][5] == (22 - 10) << 3                 # ceil(log2(100000 + 3 MiB)) = 22
    assert len(frames[0]) < len(X) - 19000
    assert datagen.decompress(frames[0], len(X), raw_dict=D, window_log_max=27) == X
    assert cldm.parse([X], wl, D)[0] == cparse.parse([X], D)[0]   # without the flag: the window_log 17 parse


def test_the_flag_is_inert_where_it_should_be():
    D, datas = versions()
    for name in ("fastest", "lazy"):
        lv = level_of(name, 23)
        today = cldm.parse(datas, 23, D, lv)
        assert cpatch.parse(datas, 23, D, lv, False) == today
        assert cpatch.parse(datas, 23, None, lv, True) == cldm.parse(datas, 23, None, lv)
        assert cpatch.parse(datas, 17, D, lv, True) == cldm.parse(datas, 17, D, lv)
        for wl, content, flag in ((23, D, False), (23, None, True), (17, D, True)):
            _, frames = model(datas, wl, name, content, flag)
            want = [cparse.reference_frame(d, b, level=lv, window_log=wl) for d, b in zip(datas, cldm.parse(datas, wl, content, lv))]
            assert frames == want, (name, wl, content is None, flag)


def test_ratio_of_an_edited_copy():
    base = datagen.gen_text(2 * MIB, 90).tobytes()
    copy = edited(base, 91)
    _, (f,) = model([copy], 22, "fastest", base)
    _, (g,) = model([copy], 22, "fastest", base, False)
    assert datagen.decompress(f, len(copy), raw_dict=base, window_log_max=27) == copy
    print(f"2 MiB edited copy against its base: {len(copy) / len(f):.2f} with the flag, {len(copy) / len(g):.2f} without")
    assert len(copy) / len(f) >= 20
    assert len(copy) / len(g) < 3


@pytest.mark.parametrize("chunk", [1000, 4096, 65536])
def test_chunked_anchors_are_cldms(chunk):
    data = datagen.gen_text(300000, 97).tobytes() + b"\0" * 5000 + rand(100000, 98)
    a, b = cpatch.anchors(data, chunk), cldm.anchors(data)
    assert a[0].tolist() == b[0].tolist() and a[1].tolist() == b[1].tolist()
    assert len(b[0]) > 1000
