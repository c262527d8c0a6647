"""A plain model of zstd's seekable format (contrib/seekable_format in the zstd repository) and of the read plan of
b200z_seekable_read_ranges.

An archive is zstd frames back to back and one skippable frame holding the seek table:

    Skippable_Magic_Number u32 LE 0x184D2A5E
    Frame_Size             u32 LE n * (8 or 12) + 9
    n entries              Compressed_Size u32, Decompressed_Size u32, [checksum u32: low 32 bits of XXH64(seed 0)]
    Number_Of_Frames       u32 LE n
    Seek_Table_Descriptor  u8     bit 7 Checksum_Flag, bits 6-2 reserved (0), bits 1-0 unused
    Seekable_Magic_Number  u32 LE 0x8F92EAB1

The read plan: every touched frame once; a frame wholly inside a range is decoded in place in the first such range's output slot,
every other touched frame into scratch (by ascending frame index, each at a multiple of 16); each range's other bytes are copy
pieces, per range in call order and per frame by ascending index, taken from scratch or from the slot of the range the frame is
in place for.  Plan rows are (frame, dst_off, range) and (dst_off, src_off, len, from_scratch, range).
"""
import bisect
import struct

SKIPPABLE_MAGIC = 0x184D2A5E
FOOTER_MAGIC = 0x8F92EAB1
ERR_INVALID_ARGUMENT = 220
ERR_SEEKABLE_TABLE = 240


class TableError(Exception):
    """A seek table that breaks a rule: .code is ERR_SEEKABLE_TABLE, the message names the rule."""
    code = ERR_SEEKABLE_TABLE


class RangeError(Exception):
    code = ERR_INVALID_ARGUMENT


def table(entries, checksum):
    """The seek table frame for entries [(compressed_size, decompressed_size, checksum)]."""
    body = b"".join(struct.pack("<II", c, d) + (struct.pack("<I", s & 0xFFFFFFFF) if checksum else b"") for c, d, s in entries)
    footer = struct.pack("<IBI", len(entries), 0x80 if checksum else 0, FOOTER_MAGIC)
    return struct.pack("<II", SKIPPABLE_MAGIC, len(body) + 9) + body + footer


def write(frames, sizes, checksums=None):
    """An archive of `frames` (bytes each) whose plaintexts have `sizes` bytes; with `checksums` the table carries them."""
    entries = [(len(f), d, checksums[i] if checksums is not None else 0) for i, (f, d) in enumerate(zip(frames, sizes))]
    return b"".join(frames) + table(entries, checksums is not None)


def parse(archive):
    """(entries [(c_off, c_size, d_off, d_size, checksum or None)], checksum flag); raises TableError."""
    n_len = len(archive)
    if n_len < 17:
        raise TableError("the archive is shorter than a seek table")
    n, desc, magic = struct.unpack_from("<IBI", archive, n_len - 9)
    if magic != FOOTER_MAGIC:
        raise TableError("Seekable_Magic_Number")
    if desc & 0x7C:
        raise TableError("reserved bits")
    ck = bool(desc & 0x80)
    esz = 12 if ck else 8
    tb = 17 + n * esz
    if tb > n_len:
        raise TableError("Number_Of_Frames gives a table larger than the archive")
    at = n_len - tb
    skm, fsize = struct.unpack_from("<II", archive, at)
    if skm != SKIPPABLE_MAGIC:
        raise TableError("Skippable_Magic_Number")
    if fsize != n * esz + 9:
        raise TableError("Frame_Size")
    out, co, do = [], 0, 0
    for i in range(n):
        c, d = struct.unpack_from("<II", archive, at + 8 + i * esz)
        s = struct.unpack_from("<I", archive, at + 16 + i * esz)[0] if ck else None
        out.append((co, c, do, d, s))
        co += c
        do += d
    if co != at:
        raise TableError("the frames' Compressed_Size do not add up to the table frame's offset")
    return out, ck


def plan(entries, ranges, output_cap=None):
    """The read plan for ranges [(offset, length, out_off)] over parse()'s entries: (frames, pieces, scratch bytes, touched per
    range); raises RangeError for a range past the content or the output, or for overlapping output slots."""
    content = entries[-1][2] + entries[-1][3] if entries else 0
    cap = (1 << 64) - 1 if output_cap is None else output_cap
    for off, ln, oo in ranges:
        if off + ln > content or oo + ln > cap:
            raise RangeError("range past the content or the output")
    slots = sorted((oo, ln) for _, ln, oo in ranges if ln)
    for (a, la), (b, _) in zip(slots, slots[1:]):
        if a + la > b:
            raise RangeError("ranges overlap in the output")
    starts = [e[2] for e in entries] + [content]
    in_place, touched = {}, []
    for r, (off, ln, oo) in enumerate(ranges):
        t = []
        if ln:
            f = bisect.bisect_right(starts, off) - 1
            while f < len(entries) and starts[f] < off + ln:
                if starts[f + 1] > starts[f]:
                    t.append(f)
                    whole = starts[f] >= off and starts[f + 1] <= off + ln
                    if f not in in_place:
                        in_place[f] = r if whole else -1
                    elif whole and in_place[f] < 0:
                        in_place[f] = r
                f += 1
        touched.append(t)
    frames, at, scratch = [], {}, 0
    for f in sorted(in_place):
        r = in_place[f]
        if r >= 0:
            dst = ranges[r][2] + starts[f] - ranges[r][0]
        else:
            dst = scratch
            scratch = (scratch + starts[f + 1] - starts[f] + 15) & ~15
        at[f] = dst
        frames.append((f, dst, r))
    pieces = []
    for r, (off, ln, oo) in enumerate(ranges):
        for f in touched[r]:
            owner = in_place[f]
            if owner == r:
                continue
            lo, hi = max(off, starts[f]), min(off + ln, starts[f + 1])
            pieces.append((oo + lo - off, at[f] + lo - starts[f], hi - lo, 1 if owner < 0 else 0, r))
    return frames, pieces, scratch, touched


def execute(plaintext, entries, ranges, out_len):
    """What the plan makes of the content: the output buffer, built only from frames' plaintexts and the plan's moves."""
    frames, pieces, scratch, _ = plan(entries, ranges)
    out = bytearray(out_len)
    scr = bytearray(scratch)
    for f, dst, r in frames:
        d0, ds = entries[f][2], entries[f][3]
        (out if r >= 0 else scr)[dst:dst + ds] = plaintext[d0:d0 + ds]
    for dst, src, ln, from_scratch, _ in pieces:
        out[dst:dst + ln] = (scr if from_scratch else out)[src:src + ln]
    return bytes(out)


def crafted_ranges(entries):
    """The crafted range sets: an empty range, one byte, a range on a frame boundary, the whole content, overlapping ranges, several
    ranges inside one frame, a frame wholly inside two ranges.  Output slots are laid out back to back with a 3-byte gap."""
    content = entries[-1][2] + entries[-1][3] if entries else 0
    sized = [e for e in entries if e[3]]
    sets = {"empty": [(content // 2, 0)], "whole": [(0, content)]}
    if content:
        sets["one_byte"] = [(content // 3, 1)]
    if len(sized) >= 2:
        b = sized[1][2]
        sets["boundary"] = [(b, sized[1][3]), (b - 1, 2), (sized[0][2], b - sized[0][2])]
        f = sized[1]
        sets["two_contain"] = [(f[2] - 5, f[3] + 10), (f[2] - 1, f[3] + 1), (f[2], f[3])]
        sets["overlap"] = [(f[2] - 100, 300), (f[2] - 50, 300), (max(0, f[2] - 1000), 2000)]
    if sized:
        f = sized[0]
        q = max(1, f[3] // 5)
        sets["inside_one"] = [(f[2] + q, q), (f[2], q), (f[2] + 3 * q, min(q, f[3] - 3 * q))]
    out = {}
    for k, rs in sets.items():
        rows, oo = [], 7
        for off, ln in rs:
            off = max(0, min(off, content))
            ln = max(0, min(ln, content - off))
            rows.append((off, ln, oo))
            oo += ln + 3
        out[k] = rows
    return out


def random_ranges(content, n, rng, lo=1, hi=65536):
    """n ranges of lo..hi bytes at random offsets, slots back to back with a 1-byte gap."""
    rows, oo = [], 1
    for _ in range(n):
        ln = int(rng.integers(lo, hi + 1)) if content else 0
        ln = min(ln, content)
        off = int(rng.integers(0, content - ln + 1)) if content else 0
        rows.append((off, ln, oo))
        oo += ln + 1
    return rows, oo
