"""The stream compressor's framing written out plainly: ruzstd's FrameCompressor::compress (frame_compressor.rs:131-224).

  header    magic, FHD 0x04 with the checksum (0x00 without), Window_Descriptor 0x38 (128 KiB); no Frame_Content_Size, no
            Single_Segment, no dictionary ID.
  blocks    the source is cut into 128 KiB blocks; a block is last only when the source ended before it filled.  When the length is
            a multiple of 128 KiB (0 included) every data block is non-last and an empty last Raw block (01 00 00) follows.
  checksum  the low 32 bits of XXH64 (seed 0) of the whole input, little-endian, when the header says so.

At the Uncompressed level every block is Raw, so `uncompressed_frame` is the whole frame.  `split_frame` takes any zstd frame apart
into its header, its blocks and its checksum, so that frames of the stream and the batch compressor can be compared block by block.
Nothing here calls the library."""
import struct

BLOCK = 131072
MAGIC = struct.pack("<I", 0xFD2FB528)
RAW, RLE, COMPRESSED = 0, 1, 2


def header(checksum):
    return MAGIC + bytes([0x04 if checksum else 0x00, 0x38])


def block_header(last, btype, size):
    return struct.pack("<I", int(last) | (btype << 1) | (size << 3))[:3]


def pieces(data):
    """The reference's block cut: (bytes, last) per block, the trailing empty block included."""
    out, pos = [], 0
    while True:
        b = bytes(data[pos:pos + BLOCK])
        pos += len(b)
        if not b:
            out.append((b"", True))
            return out
        out.append((b, len(b) < BLOCK))
        if len(b) < BLOCK:
            return out


def trailer(data, checksum, xxh64):
    return struct.pack("<I", xxh64(data) & 0xFFFFFFFF) if checksum else b""


def uncompressed_frame(data, checksum, xxh64):
    """The whole frame FrameCompressor writes at CompressionLevel::Uncompressed."""
    out = bytearray(header(checksum))
    for b, last in pieces(data):
        out += block_header(last, RAW, len(b)) + b
    return bytes(out + trailer(data, checksum, xxh64))


def split_frame(frame):
    """(header bytes, [(last, type, size, body bytes)], checksum bytes) of one zstd frame; raises when the frame does not end
    exactly after its checksum."""
    f = bytes(frame)
    assert f[:4] == MAGIC
    fhd = f[4]
    single, has_sum, did = (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
    fcs = [1 if single else 0, 2, 4, 8][fhd >> 6]
    p = 5 + (0 if single else 1) + [0, 1, 2, 4][did] + fcs
    hdr, blocks = f[:p], []
    while True:
        h = int.from_bytes(f[p:p + 3], "little")
        last, btype, size = h & 1, (h >> 1) & 3, h >> 3
        n = 1 if btype == RLE else size
        blocks.append((last, btype, size, f[p + 3:p + 3 + n]))
        assert len(blocks[-1][3]) == n, "truncated block"
        p += 3 + n
        if last:
            break
    tail = f[p:p + 4] if has_sum else b""
    assert p + len(tail) == len(f) and len(tail) == (4 if has_sum else 0), "bytes after the frame's end"
    return hdr, blocks, tail
