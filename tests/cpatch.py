"""Long matches into a dictionary (B200Z_FLAG_DICT_LONG, libzstd's --patch-from) written out plainly: what the long-match kernels
(csrc/ldm.cu: k_ldict, k_lcand<true>, k_lblock<true>) must find and the frame the compressor must write, with a dictionary whose
content is D, window_log > 17 and the flag.  The frame is X.

This module restates DESIGN.md section 4.11's delta-compression rule in Python, calling nothing in the library.  It keeps
tests/cldm.py's anchors, keys, block rule and forced pieces and the parse models' blocks (tests/cparse.py, clazy.py, copt.py,
cultra.py), and changes:

  dictionary anchors   cldm.anchors of D's last min(|D|, 2^27) bytes alone, positions counted in D: they depend on D only.  The
            frames' own anchors are cldm's, from each frame alone.
  frames    every frame of the submission has anchors, also frames of 131072 bytes or fewer.
  candidate the nearest earlier anchor of the same frame with the same key, as in cldm; when the frame has none, the last
            dictionary anchor with that key (the one nearest D's end) at offset p + |D| - its position.  Kept when the offset
            lies in (131072, 2^window_log]; a nearest candidate outside that range gives none (no fall back to the dictionary).
  block     cldm.block_matches over the virtual stream D || X: the check, the forward and the backward extension read across
            D's end, and its backward bound "where the source would leave the frame" becomes where it would leave D.
  parse     unchanged: the pieces are forced, their offsets enter LAZY's and OPT's repeat offsets, whose guards keep a repeat's
            source inside the frame, so no parse reads before its frame.
  header    exponent min(window_log, max(17, ceil(log2(n + |D|)))): every offset o <= min(position + |D|, 2^window_log) lies
            within the window.  ULTRA's far stage and repeat reach still follow the frame's own size (tests/cultra.py).

Without the flag, without a dictionary or at window_log 17 the output is cldm.parse's and cparse.reference_frame's.  `parse`
gives the blocks; `reference_frame` assembles the frame (cparse.reference_frame with the header's window widened)."""
import numpy as np

import cldm
import cparse

BLOCK, WINDOW = cldm.BLOCK, cldm.WINDOW
DICT_REACH = 1 << 27    # the dictionary bytes, from its end, whose anchors are listed (B200Z_WINDOW_LOG_MAX)
ANCHOR_CHUNK = 1 << 22  # bytes `anchors` hashes at a time, so that 2^27 bytes of dictionary need no 2^27-entry temporaries


def anchors(data, chunk=ANCHOR_CHUNK):
    """cldm.anchors(data), computed chunk by chunk: each chunk is hashed with the LDM_LEN - 1 + LDM_QUIET bytes before it, which
    settle both the hashes and the quiet rule of its first positions."""
    data = bytes(data)
    back = cldm.LDM_LEN - 1 + cldm.LDM_QUIET
    P, K = [], []
    for c0 in range(0, len(data), chunk):
        x0 = max(0, c0 - back)
        pos, keys = cldm.anchors(data[x0:c0 + chunk])
        keep = pos + x0 >= c0
        P.append(pos[keep] + x0)
        K.append(keys[keep])
    if not P:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.uint64)
    return np.concatenate(P), np.concatenate(K)


def dict_anchors(content):
    """(positions in D, keys) of the anchors of a dictionary's content D: the anchors of its last min(|D|, 2^27) bytes alone."""
    D = bytes(content)
    lo = max(0, len(D) - DICT_REACH)
    pos, keys = anchors(D[lo:])
    return pos + lo, keys


def candidates(frames, window_log, content):
    """Per frame, [(position, offset)] of its anchors with a kept candidate, in position order, the dictionary's included."""
    dpos, dkeys = dict_anchors(content)
    dlast = dict(zip(dkeys.tolist(), dpos.tolist()))   # the last (nearest D's end) wins
    last = {}
    out = []
    for fi, f in enumerate(frames):
        got = []
        pos, keys = anchors(f)
        for p, k in zip(pos.tolist(), keys.tolist()):
            prev = last.get(k)
            if prev is not None and prev[0] == fi:
                o = p - prev[1]
            else:
                o = p + len(content) - dlast[k] if k in dlast else 0
            if WINDOW < o <= (1 << window_log):
                got.append((p, o))
            last[k] = (fi, p)
        out.append(got)
    return out


def forced(frames, window_log, content):
    """Per frame, per block, the block's kept matches: cldm.block_matches over D || X (only D's last 2^27 bytes can be reached,
    since no offset exceeds 2^27), with block and anchor positions moved past the dictionary bytes in front of the frame."""
    Dt = bytes(content)[-DICT_REACH:] if content else b""
    out = []
    for f, cands in zip(frames, candidates(frames, window_log, content)):
        F = bytes(f)
        V, d = Dt + F, len(Dt)
        blocks, pos, i = [], 0, 0
        while True:
            n = min(BLOCK, len(F) - pos)
            mine = []
            while i < len(cands) and cands[i][0] < pos + n:
                mine.append((d + cands[i][0], cands[i][1]))
                i += 1
            blocks.append(cldm.block_matches(V, d + pos, n, mine) if mine else [])
            pos += n
            if pos >= len(F):
                break
        out.append(blocks)
    return out


def parse(frames, window_log, content=None, level=cparse.FASTEST, dict_long=True):
    """The parse of every frame of one submission at window_log and `level` against the dictionary `content`; with dict_long the
    long matches reach into it, else (and without a dictionary, or at window_log 17) this is cldm.parse."""
    if not dict_long or content is None or window_log <= cparse.WINDOW_LOG_MIN:
        return cldm.parse(frames, window_log, content, level)
    return cparse.parse(frames, content, level, forced(frames, window_log, content))


def header_dict_len(content, window_log, dict_long=True):
    """The dictionary length the frames' Window_Descriptor covers: |D| with the flag, a dictionary and window_log > 17, else 0."""
    return len(content) if dict_long and content is not None and window_log > cparse.WINDOW_LOG_MIN else 0


def frame_window_log(n, window_log, dict_len=0):
    """The Window_Descriptor exponent: cparse.frame_window_log of n + dict_len."""
    return cparse.frame_window_log(n + dict_len, window_log)


def reference_frame(data, blocks, window_log, dict_len=0, **kw):
    """cparse.reference_frame(data, blocks, window_log=window_log, **kw) with the Window_Descriptor (byte 5: Single_Segment is 0)
    of frame_window_log(len(data), window_log, dict_len)."""
    f = cparse.reference_frame(data, blocks, window_log=window_log, **kw)
    return f[:5] + bytes([(frame_window_log(len(data), window_log, dict_len) - 10) << 3]) + f[6:]
