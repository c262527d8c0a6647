"""The stream compressor's framing model (tests/streamframe.py) against hand-written frames: ruzstd's FrameCompressor at
CompressionLevel::Uncompressed -- header, block cut, last-block bit, trailing empty block and checksum.  CPU only."""
import struct

import cparse
import streamframe as SF

HDR = bytes.fromhex("28b52ffd0438")
HDR_NOSUM = bytes.fromhex("28b52ffd0038")


def _sum(data):
    return struct.pack("<I", cparse.xxh64(data) & 0xFFFFFFFF)


def test_plain_xxh64_agrees_with_the_library(pkg):
    for d in (b"", b"A", bytes(range(256)) * 600):
        assert cparse.xxh64(d) == pkg.xxh64(d)


def test_empty_frame():
    assert SF.uncompressed_frame(b"", True, cparse.xxh64) == bytes.fromhex("28b52ffd0438 010000 99e9d851")
    assert SF.uncompressed_frame(b"", False, cparse.xxh64) == bytes.fromhex("28b52ffd0038010000")


def test_one_byte():
    # one Raw block of 1 byte, last: 1 | 0 << 1 | 1 << 3 = 0x09
    assert SF.uncompressed_frame(b"A", True, cparse.xxh64) == HDR + bytes.fromhex("090000") + b"A" + _sum(b"A")
    assert SF.uncompressed_frame(b"A", False, cparse.xxh64) == HDR_NOSUM + bytes.fromhex("090000") + b"A"


def test_one_full_block_is_followed_by_an_empty_last_block():
    d = bytes(range(256)) * 512   # 131072 bytes
    # 131072 << 3 = 0x100000, not last: 00 00 10; then the empty last Raw block 01 00 00
    want = HDR + bytes.fromhex("000010") + d + bytes.fromhex("010000") + _sum(d)
    assert SF.uncompressed_frame(d, True, cparse.xxh64) == want
    assert SF.uncompressed_frame(d, False, cparse.xxh64) == HDR_NOSUM + bytes.fromhex("000010") + d + bytes.fromhex("010000")


def test_block_cut():
    B = SF.BLOCK
    for n, want in ((0, [(0, True)]), (1, [(1, True)]), (B - 1, [(B - 1, True)]), (B, [(B, False), (0, True)]),
                    (B + 1, [(B, False), (1, True)]), (3 * B, [(B, False)] * 3 + [(0, True)]), (5 * B + 7, [(B, False)] * 5 + [(7, True)])):
        assert [(len(b), last) for b, last in SF.pieces(b"x" * n)] == want, n


def test_split_frame_takes_the_model_apart():
    d = b"0123456789" * 30000   # 300000 bytes: 128 KiB, 128 KiB, 37856
    hdr, blocks, tail = SF.split_frame(SF.uncompressed_frame(d, True, cparse.xxh64))
    assert hdr == HDR and tail == _sum(d)
    assert [(last, t, size) for last, t, size, _ in blocks] == [(0, 0, SF.BLOCK), (0, 0, SF.BLOCK), (1, 0, 300000 - 2 * SF.BLOCK)]
    assert b"".join(body for *_, body in blocks) == d
