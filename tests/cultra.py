"""The compressor's ULTRA level (an extension) written out plainly: what k_copt<DICT, true, true> and the far stage of ldm.cu must
produce for every block.

ULTRA is OPT (tests/copt.py states it) with three changes; everything else -- blocks, segments, `stop`, the near chain, CAP, SUFF, M,
prices, the DP, W, the dictionary entry, forced long-distance pieces (tests/cldm.py), packing and framing -- is OPT's.  Let Wf be
the frame's window, 2^(its Window_Descriptor exponent): 2^min(window_log, max(17, ceil(log2 n))) for a batch frame of n bytes,
2^window_log for the stream compressor's frame.

  far key   key8(q) = (u64le(q) * 0x9E3779B97F4A7C15 mod 2^64) >> 32 for every keyed position q: q + 8 <= the end of q's 128 KiB
            block of the frame (so a stream chunk's keys need no byte of the next chunk).
  far walk  after the chain's walk, unless that ended on a verification reaching its limit: the keyed positions p of the frame with
            key8(p) == key8(q), nearest first, from the nearest with q - p > 131072; at most FAR_DEPTH of them (collisions count),
            stopping at q - p > Wf.  Each is verified for min(CAP, stop - q) bytes and pushed by OPT's rule (strictly longer than
            every earlier candidate and >= 5; the shortest drops out beyond M); a verification reaching its limit ends the walk.
            The dictionary entry follows, as at OPT.
  repeats   a node's repeat o is verified when o <= back + i and o <= Wf (back: all of the frame before the block).

Where Wf = 131072 the level is OPT exactly: `Far.frame` gives no walk, and no far-stage kernel runs.

The model runs tests/copt.py's own segment loop and DP, not copies of them.  As k_copt<DICT, LONG, FAR> instantiates one kernel
body with FAR, `instantiate` gives a copt function the same code with some of the module names it reads bound otherwise: the DP
with WINDOW (its repeats' reach) bound to Wf, and the segment loop with that DP and with the finder `FarFrame.candidates`, which
is copt's finder followed by the far walk.  The segment loop gets the frame's whole offset before the block as `back`, so that
repeats and the taken match's source test reach up to Wf."""
import functools
import types

import numpy as np

import clazy
import copt
import cparse

BLOCK, WINDOW, MIN_MATCH = cparse.BLOCK, cparse.WINDOW, cparse.MIN_MATCH
FAR_DEPTH = 8            # D_F: far entries a position visits
FAR_KEY = 8              # bytes a far key hashes
KEY_MUL = 0x9E3779B97F4A7C15


def instantiate(fn, **names):
    """tests/copt.py's function fn, its code unchanged, with the module names in `names` bound to other values."""
    g = dict(vars(copt))
    g.update(names)
    return types.FunctionType(fn.__code__, g, fn.__name__, fn.__defaults__, fn.__closure__)


@functools.lru_cache(None)
def dp_at(wf):
    """copt's DP with repeats reaching up to wf."""
    return instantiate(copt.dp, WINDOW=wf)


def key8(F, p):
    """The far key of position p of frame F (p must be keyed)."""
    return ((int.from_bytes(bytes(F[p:p + 8]), "little") * KEY_MUL) & ((1 << 64) - 1)) >> 32


def keys(F):
    """key8 of every position of frame F, -1 where a position is not keyed."""
    a = np.frombuffer(bytes(F), dtype=np.uint8)
    m = len(a) - (FAR_KEY - 1)
    if m <= 0:
        return np.zeros(0, dtype=np.int64)
    w = np.zeros(m, dtype=np.uint64)
    for k in range(8):
        w |= a[k:k + m].astype(np.uint64) << np.uint64(8 * k)
    with np.errstate(over="ignore"):
        key = ((w * np.uint64(KEY_MUL)) >> np.uint64(32)).astype(np.int64)
    key[np.arange(m) % BLOCK + FAR_KEY > BLOCK] = -1
    return key


class FarFrame:
    """One frame's far walk: its keyed positions sorted by (key, position), as the GPU's stable sort orders them."""

    def __init__(self, F, wf):
        self.wf = wf
        self.key = keys(F)
        valid = np.nonzero(self.key >= 0)[0]
        self.pos = valid[np.argsort(self.key[valid], kind="stable")]
        self.skey = self.key[self.pos]
        self.rank = np.full(len(self.key), -1, dtype=np.int64)
        self.rank[self.pos] = np.arange(len(self.pos))
        self.segment = instantiate(copt._segment, candidates=self.candidates, dp=dp_at(wf))

    def candidates(self, F, base, back, q, stop, prev, H17, dic):
        """The finder's list at block position q: copt's (the chain, the dictionary entry), then the far walk unless a chain
        verification reached its limit.  The dictionary entry (back + q < 131072) and the far walk (q - p > 131072 inside the
        frame) never both apply, so the far walk may follow copt's whole list."""
        out = copt.candidates(F, base, back, q, stop, prev, H17, dic)
        fq = base + q
        lim = min(copt.OPT_CAP, stop - q)
        if fq <= WINDOW or (out and out[-1][0] == lim):
            return out
        best = out[-1][0] if out else MIN_MATCH - 1
        for c in self.walk(fq):
            ln = cparse._mlen(F, fq, F, c, lim)
            if ln > best:
                out.append((ln, fq - c, stop - q))
                best = ln
                if len(out) > copt.OPT_CANDS:
                    del out[0]
                if ln == lim:
                    break
        return out

    def walk(self, q):
        """The positions q's far walk visits, nearest first."""
        if q >= len(self.key) or self.key[q] < 0:
            return []
        k = int(self.rank[q])
        run = int(np.searchsorted(self.skey, self.key[q], "left"))
        t = run + int(np.searchsorted(self.pos[run:k], q - WINDOW, "left")) - 1   # the nearest with q - p > WINDOW
        out = []
        while t >= run and len(out) < FAR_DEPTH and q - int(self.pos[t]) <= self.wf:
            out.append(int(self.pos[t]))
            t -= 1
        return out


class Far:
    """ULTRA's far finder at window_log; stream: Wf = 2^window_log for every frame (the stream compressor's descriptor)."""

    def __init__(self, window_log, stream=False):
        self.window_log, self.stream = window_log, stream
        self._memo = [None, None]

    def frame_window(self, n):
        return 1 << (self.window_log if self.stream else cparse.frame_window_log(n, self.window_log))

    def frame(self, F):
        """F's FarFrame, or None where Wf = 131072 (ULTRA is OPT there)."""
        wf = self.frame_window(len(F))
        if wf <= WINDOW:
            return None
        if self._memo[0] is not F:
            self._memo[0], self._memo[1] = F, FarFrame(F, wf)
        return self._memo[1]


def _segment(F, base, n, back, s, e, t1, H13, _H13, H17, dic, pieces, far):
    """ULTRA's segment: OPT's where the frame's window is 131072, else copt's loop over the far finder and the DP at Wf, with
    all of the frame before the block as `back`."""
    fw = far.frame(F)
    if fw is None:
        return copt._segment(F, base, n, back, s, e, t1, H13, _H13, H17, dic, pieces)
    return fw.segment(F, base, n, base, s, e, t1, H13, _H13, H17, dic, pieces)


@functools.lru_cache(None)
def level(window_log, stream=False):
    """The ULTRA Level at window_log (cparse.parse / reference_frame take it)."""
    return cparse.Level(copt.OPT_HASH_LOG, copt.OPT_HASH_LOG, functools.partial(_segment, far=Far(window_log, stream)), clazy.records)


def parse(frames, window_log, content=None):
    """The parse of every frame of one submission at ULTRA and window_log, with tests/cldm.py's forced pieces."""
    import cldm
    return cldm.parse(frames, window_log, content, level(window_log))


def reference_frame(data, blocks, window_log, **kw):
    return cparse.reference_frame(data, blocks, level=level(window_log), window_log=window_log, **kw)


def brute_far(F, q, wf):
    """The far list by brute force: the keyed positions p with key8(p) == key8(q) and 131072 < q - p <= wf, nearest first, at most
    FAR_DEPTH."""
    K = keys(F)
    if q >= len(K) or K[q] < 0:
        return []
    out = []
    for p in range(q - WINDOW - 1, max(-1, q - wf - 1), -1):
        if K[p] == K[q]:
            out.append(p)
            if len(out) == FAR_DEPTH:
                break
    return out
