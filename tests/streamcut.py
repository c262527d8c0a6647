"""A plain model of how decode_all_stream (include/b200zstd.h, tier 1d) cuts a source into submissions.  It imports nothing from the
library.  With C the chunk size, a submission holds whole blocks and at most C bytes of input (frame headers, blocks, checksums and the
skippable frames between its frames), a decoded size bound of 4 * C (a Raw or RLE block counts its size, a Compressed block
min(128 KiB, window)), C // 16384 blocks and C // 4 sequences (each block's count rounded up to 4) -- or exactly one block.  A frame
header goes with its frame's first block.  Skippable frames in front of a submission are dropped.  The cutter stops at the end of the
source or at the first error it can see from the headers: a frame header, a skippable frame that runs past the source, a block header,
a truncated block or a missing checksum."""

ZSTD_MAGIC = 0xFD2FB528


def _le(b, n):
    return int.from_bytes(bytes(b[:n]), "little")


def frame_header(b):
    """(error name or None, header length, window or None, checksum flag, skip length or None) of the bytes b at a frame start."""
    if len(b) < 4:
        return "MAGIC_NUMBER_READ", 0, None, False, None
    magic = _le(b, 4)
    if 0x184D2A50 <= magic <= 0x184D2A5F:
        if len(b) < 8:
            return "FRAME_DESCRIPTOR_READ", 0, None, False, None
        return None, 8, None, False, _le(b[4:], 4)
    if magic != ZSTD_MAGIC:
        return "BAD_MAGIC_NUMBER", 0, None, False, None
    if len(b) < 5:
        return "FRAME_DESCRIPTOR_READ", 0, None, False, None
    d = b[4]
    single, flag = (d >> 5) & 1, d >> 6
    did_at = 6 - single
    fcs_at = did_at + [0, 1, 2, 4][d & 3]
    hlen = fcs_at + ([single, 2, 4, 8][flag])
    if len(b) < did_at:
        return "WINDOW_DESCRIPTOR_READ", 0, None, False, None
    if len(b) < fcs_at:
        return "DICTIONARY_ID_READ", 0, None, False, None
    if len(b) < hlen:
        return "FRAME_CONTENT_SIZE_READ", 0, None, False, None
    if single:
        window = _le(b[fcs_at:], hlen - fcs_at) + (256 if flag == 1 else 0)
    else:
        wd = b[5]
        base = 1 << (10 + (wd >> 3))
        window = base + (base // 8) * (wd & 7)
        if window > 128 << 20:
            return "WINDOW_SIZE_TOO_BIG", hlen, None, False, None
    if _le(b[did_at:], fcs_at - did_at):
        return "DICT_NOT_PROVIDED", hlen, None, False, None
    return None, hlen, window, bool((d >> 2) & 1), None


def block_seqs(c):
    """Sequences a Compressed block's content announces, rounded up to 4 (0 when its section headers do not parse)."""
    if not c:
        return 0
    lt, sf = c[0] & 3, (c[0] >> 2) & 3
    if lt in (0, 1):
        need = 1 if sf in (0, 2) else (2 if sf == 1 else 3)
    else:
        need = 3 if sf <= 1 else (4 if sf == 2 else 5)
    if len(c) < need:
        return 0
    if lt in (0, 1):
        regen = c[0] >> 3 if sf in (0, 2) else ((c[0] >> 4) + (c[1] << 4) if sf == 1 else (c[0] >> 4) + (c[1] << 4) + (c[2] << 12))
        upper = 1 if lt == 1 else regen
    else:
        if sf <= 1:
            upper = (c[1] >> 6) + (c[2] << 2)
        elif sf == 2:
            upper = (c[2] >> 2) + (c[3] << 6)
        else:
            upper = (c[2] >> 6) + (c[3] << 2) + (c[4] << 10)
    if len(c) - need < upper:
        return 0
    q = c[need + upper:]
    n = 0
    if not q or q[0] == 0:
        n = 0
    elif q[0] < 128:
        n = q[0] if len(q) >= 2 else 0
    elif q[0] < 255:
        n = ((q[0] - 128) << 8) + q[1] if len(q) >= 3 else 0
    else:
        n = q[1] + (q[2] << 8) + 0x7F00 if len(q) >= 4 else 0
    return (n + 3) & ~3


def cut(data, C):
    """[(start, end, in_bytes, out_bound, nblocks, nseq, nframes, flags)], end record {error_offset, status, error_frame,
    skippable_frames} -- what b200z_debug_stream_cut reports (status as an error name, None without an error)."""
    n = len(data)
    maxb, maxs = max(1, C // 16384), C // 4
    subs, skips, zi = [], 0, -1
    pos = 0
    cont = None            # (window, checksum flag) of the frame that continues
    end = None
    while end is None:
        start = pos
        sub = dict(in_bytes=0, out=0, blocks=0, seqs=0, frames=0, flags=0)
        active = None
        if cont is not None:
            active, cont = cont, None
            sub["frames"], sub["flags"] = 1, 1

        def fits(i, o, s):
            return sub["blocks"] == 0 or (sub["in_bytes"] + i <= C and sub["out"] + o <= 4 * C and sub["blocks"] + 1 <= maxb
                                          and sub["seqs"] + s <= maxs)

        def block(p, window, checksum):
            """Reads the block at p: ('err', name) / ('cut',) / ('ok', size, last)."""
            if n - p < 3:
                return ("err", "BLOCK_HEADER_READ")
            h = _le(data[p:], 3)
            t, size = (h >> 1) & 3, h >> 3
            if t == 3:
                return ("err", "FOUND_RESERVED_BLOCK")
            if size > 131072:
                return ("err", "BLOCK_SIZE_TOO_LARGE")
            c = 1 if t == 1 else size
            if n - p - 3 < c:
                return ("err", "BLOCK_CONTENT_READ" if t == 2 else "BLOCK_BODY_READ")
            out = min(131072, window) if t == 2 else size
            seqs = block_seqs(data[p + 3:p + 3 + c]) if t == 2 else 0
            return ("ok", 3 + c, bool(h & 1), out, seqs)

        while True:
            if active is None:
                if pos >= n:
                    end = dict(error_offset=n, status=None, error_frame=-1)
                    break
                err, hl, window, checksum, skip = frame_header(data[pos:pos + 18])
                if err is None and skip is not None:
                    if sub["frames"] == 0:
                        if n - pos < 8 + skip:
                            end = dict(error_offset=pos, status="FAILED_TO_SKIP_FRAME", error_frame=-1)
                            break
                        pos += 8 + skip
                        start = pos
                        skips += 1
                        continue
                    if sub["in_bytes"] + 8 + skip > C:
                        break
                    if n - pos < 8 + skip:
                        end = dict(error_offset=pos, status="FAILED_TO_SKIP_FRAME", error_frame=-1)
                        break
                    pos += 8 + skip
                    sub["in_bytes"] += 8 + skip
                    skips += 1
                    continue
                zstd = n - pos >= 4 and _le(data[pos:], 4) == ZSTD_MAGIC
                if err is not None:
                    end = dict(error_offset=pos, status=err, error_frame=zi + 1 if zstd else -1)
                    break
                b = block(pos + hl, window, checksum)
                if b[0] == "ok" and not fits(hl + b[1] + (4 if b[2] and checksum else 0), b[3], b[4]):
                    break
                zi += 1
                active = (window, checksum, pos, zi)
                sub["frames"] += 1
                pos += hl
                sub["in_bytes"] += hl
            window, checksum, at, z = active
            b = block(pos, window, checksum)
            if b[0] == "err":
                end = dict(error_offset=at, status=b[1], error_frame=z)
                break
            _, size, last, out, seqs = b
            if not fits(size + (4 if last and checksum else 0), out, seqs):
                cont = active
                sub["flags"] |= 2
                break
            pos += size
            sub["in_bytes"] += size
            sub["out"] += out
            sub["blocks"] += 1
            sub["seqs"] += seqs
            if last:
                active = None
                if checksum:
                    if n - pos < 4:
                        end = dict(error_offset=at, status="FAILED_TO_READ_CHECKSUM", error_frame=z)
                        break
                    pos += 4
                    sub["in_bytes"] += 4
        if sub["frames"]:
            subs.append((start, pos, sub["in_bytes"], sub["out"], sub["blocks"], sub["seqs"], sub["frames"], sub["flags"]))
    end["skippable_frames"] = skips
    return subs, end


def block_ends(data):
    """Every stream offset where a block or a frame (checksum included) ends, and where a skippable frame ends, over whole frames."""
    ends, pos, n = set(), 0, len(data)
    while pos < n:
        err, hl, window, checksum, skip = frame_header(data[pos:pos + 18])
        if err is not None:
            break
        if skip is not None:
            pos += 8 + skip
            ends.add(pos)
            continue
        p = pos + hl
        while n - p >= 3:
            h = _le(data[p:], 3)
            t, size = (h >> 1) & 3, h >> 3
            p += 3 + (1 if t == 1 else size)
            if p > n:
                break
            if h & 1:
                p += 4 if checksum else 0
                ends.add(p)
                break
            ends.add(p)
        else:
            break
        if p > n or not (h & 1):
            break
        pos = p
    return ends
