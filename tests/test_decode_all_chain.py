"""How decode_all finds the frames of a buffer of concatenated frames (b200z_decode_all_prepare), checked on the host: the host-input
walk from frame to frame and the device-input selection through every magic-number candidate (b200z_debug_decode_all_chain runs
the latter with its scan and walks on the host) must both visit exactly the frames a plain Python walker visits, built on
tests/refwalk.py's header parsing.  No GPU needed."""
import os
import subprocess

from conftest import ROOT, read_golden
import refwalk

ZSTD_MAGIC = b"\x28\xb5\x2f\xfd"


def skippable(n, magic_low=0):
    return (0x184D2A50 + magic_low).to_bytes(4, "little") + n.to_bytes(4, "little") + bytes((i * 7) & 0xFF for i in range(n))


def raw_frame(content, checksum=False):
    """A zstd frame of Raw blocks holding `content` (window 1 MiB, no content size)."""
    out = bytearray(ZSTD_MAGIC + bytes([0x04 if checksum else 0x00, 0x50]))
    pos = 0
    while True:
        piece = content[pos:pos + 131072]
        pos += len(piece)
        last = pos >= len(content)
        h = (len(piece) << 3) | (0 << 1) | (1 if last else 0)
        out += h.to_bytes(3, "little") + piece
        if last:
            break
    if checksum:
        out += b"\x01\x02\x03\x04"
    return bytes(out)


def py_chain(buf):
    """decode_all's walk (frame_decoder.rs:541-577) over whole frames: the offsets it visits, the one where it ends included."""
    at, pos, n = [], 0, len(buf)
    while pos < n:
        at.append(pos)
        if n - pos < 4:
            break
        magic = int.from_bytes(buf[pos:pos + 4], "little")
        if 0x184D2A50 <= magic <= 0x184D2A5F:
            if n - pos < 8:
                break
            nxt = pos + 8 + int.from_bytes(buf[pos + 4:pos + 8], "little")
            if nxt > n:
                break
            pos = nxt
            continue
        if magic != 0xFD2FB528 or n - pos < 5:
            break
        desc = buf[pos + 4]
        single = (desc >> 5) & 1
        hlen = 6 - single + [0, 1, 2, 4][desc & 3] + [single, 2, 4, 8][desc >> 6]
        if n - pos < hlen:
            break
        hl, _window, csum = refwalk.frame_header(buf[pos:pos + hlen])
        p, ended = pos + hl, False
        while n - p >= 3:
            h = int.from_bytes(buf[p:p + 3], "little")
            t, size = (h >> 1) & 3, h >> 3
            if t == 3 or size > 131072:
                break
            p += 3
            c = 1 if t == 1 else size
            if n - p < c:
                break
            p += c
            if h & 1:
                ended = True
                break
        if not ended:
            break
        nxt = p + (4 if csum else 0)
        if nxt > n:
            break
        pos = nxt
    return at


def corpus_frames(manifest):
    return [read_golden("decodecorpus", name) for name in sorted(manifest["corpus"])]


def concat_with_skippables(frames):
    """The frames with skippable frames of 0, 1 and 300 bytes between them, and the offset of every piece."""
    buf, starts, lens = bytearray(), [], [0, 1, 300]
    for i, f in enumerate(frames):
        starts.append(len(buf)); buf += f
        s = skippable(lens[i % 3], i % 16)
        starts.append(len(buf)); buf += s
    return bytes(buf), starts


def check(pkg, buf):
    want = py_chain(buf)
    assert pkg.binding.decode_all_chain(buf) == want
    assert pkg.binding.decode_all_chain(buf, by_candidates=True) == want
    return want


def test_corpus_concatenation(pkg, manifest):
    frames = corpus_frames(manifest)
    assert len(frames) == 101
    buf, starts = concat_with_skippables(frames)
    assert check(pkg, buf) == starts


def test_truncations_around_boundaries(pkg, manifest):
    buf, starts = concat_with_skippables(corpus_frames(manifest)[:24])
    cuts = set()
    for s in starts + [len(buf)]:
        for d in (-5, -4, -3, -1, 0, 1, 2, 3, 4, 5, 8, 9):
            if 0 <= s + d <= len(buf):
                cuts.add(s + d)
    for cut in sorted(cuts):
        at = check(pkg, buf[:cut])
        assert at == [s for s in starts if s < cut][:len(at)]


def test_trailing_garbage_and_bytes(pkg, manifest):
    buf, starts = concat_with_skippables(corpus_frames(manifest)[:10])
    for tail in (b"\x00", b"\x28\xb5", b"\x28\xb5\x2f", b"garbage that is no frame", ZSTD_MAGIC, ZSTD_MAGIC + b"\x00",
                 b"\x50\x2a\x4d\x18\x00\x00"):
        at = check(pkg, buf + tail)
        assert at == starts + [len(buf)]


def test_overrunning_skippable_frame(pkg, manifest):
    frames = corpus_frames(manifest)[:3]
    buf = b"".join(frames)
    s = skippable(100)
    for cut in (8, 9, 50, 107):
        at = check(pkg, buf + s[:cut])
        assert at[-1] == len(buf)
    assert check(pkg, buf + s)[-1] == len(buf)


def test_false_candidates_inside_raw_blocks(pkg, manifest):
    frames = corpus_frames(manifest)
    inner = b"".join(frames[:12]) + skippable(5)
    wrapped = raw_frame(inner)
    wrapped_ck = raw_frame(inner[:200000], checksum=True)
    assert inner.count(ZSTD_MAGIC) >= 12
    buf = frames[0] + wrapped + frames[1] + skippable(1) + wrapped_ck + frames[2]
    at = check(pkg, buf)
    l0, lw, l1 = len(frames[0]), len(wrapped), len(frames[1])
    assert at == [0, l0, l0 + lw, l0 + lw + l1, l0 + lw + l1 + 9, l0 + lw + l1 + 9 + len(wrapped_ck)]
    # cut inside the wrapping frame: the chain ends there, whatever the candidates inside it
    for cut in (l0 + 100, l0 + lw // 2, l0 + lw - 1):
        assert check(pkg, buf[:cut]) == [0, l0]


def test_empty_and_tiny_inputs(pkg):
    for buf in (b"", b"\x00", b"\x28", ZSTD_MAGIC, skippable(0), skippable(0) + skippable(3)):
        check(pkg, buf)
    assert check(pkg, b"") == []
    assert check(pkg, skippable(0) + skippable(3)) == [0, 8]


def test_all_result_layout(pkg, tmp_path):
    """b200z_all_result as gcc lays it out == the numpy dtype the binding fills, field by field."""
    dt = pkg.binding.ALL_RESULT_DTYPE
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200zstd.h"', 'int main(void) {',
             '  printf("* %zu 0\\n", sizeof(b200z_all_result));']
    for f in dt.names:
        lines.append(f'  printf("{f} %zu %zu\\n", offsetof(b200z_all_result, {f}), sizeof(((b200z_all_result *)0)->{f}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    seen = 0
    for ln in subprocess.check_output([str(exe)]).decode().split("\n"):
        if not ln:
            continue
        f, a, b = ln.split()
        if f == "*":
            assert dt.itemsize == int(a)
        else:
            assert dt.fields[f][1] == int(a) and dt.fields[f][0].itemsize == int(b), f
            seen += 1
    assert seen == len(dt.names)
