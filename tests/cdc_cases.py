"""Roll-32 candidates planted where the CDC scan (K1) and the cut selection (K1b) can go wrong, and a plain numpy
reference of both (test infrastructure only).  Written from DESIGN §3; it uses no oracle/ code, so it stays independent
of what it checks.

h_i = sum over k < 32 of u_{i-k} * M^k (mod 2^32), u_i the little-endian word that ends at byte i.  So h_i depends on
bytes i-34..i only and is linear in them: byte b_j adds b_j * C[i-j] to h_i.  That makes candidates cheap to control:
`plant` picks bytes p-1, p (and re-draws p-2 when no pair keeps the neighbours free of candidates) so that h_p has a
wanted class and no other position of p-2..p+34 becomes a candidate; `clear` re-draws the byte of every candidate in a range until none is left;
`every_byte_loose` makes each position of a range a loose candidate (loose_bits <= 8).  Plants at least SPACING bytes
apart do not touch each other's windows, so they are placed together, vectorised.

Random content holds a loose candidate about once in 4096 bytes at positions nobody chose; the cases below put them at
row offsets, region and tile starts, cut-rule boundaries, window edges of the big-file selector and piece ends of files
that span submits.  Every case is deterministic: its generator is seeded from its name."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from functools import partial
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

from tests import table_cases as tc

M = 0x9E3779BA
MASK32 = 0xFFFFFFFF
SPACING = 37                 # plants this far apart are independent (a plant touches bytes p-2..p, hashes up to p+34)
ROW = 128                    # K1: a thread owns one 128-byte row
SCAN_TILE = 4096             # K1: one TileRec per 4 KiB region (one warp, 32 rows)
SCAN_POOL_BLOCK = 256        # K1: pool entries a warp reserves per atomic
SELECT_BIG_FILE = 4 << 20    # K1b: files at least this long go to k_select_cuts_big
SELB_REGIONS = 4096          # k_select_cuts_big: regions of a staged window (16 MiB)
SELB_CANDS = 16384           # k_select_cuts_big: candidates a staged window holds
MAX_SIZE_LIMIT = (1 << 32) - (1 << 24) - 1   # MKSNAP_CDC_MAX_SIZE_LIMIT
NONE, LOOSE, STRICT = 0, 1, 2

_MPOW = np.array([pow(M, k, 1 << 32) for k in range(32)], dtype=np.uint32)
# C[d]: what byte j contributes to h_{j+d}, per unit of its value (it sits in u_j..u_{j+3} at shifts 24, 16, 8, 0)
C = [sum(pow(M, d - t, 1 << 32) << (24 - 8 * t) for t in range(4) if 0 <= d - t < 32) & MASK32 for d in range(35)]


@dataclass(frozen=True)
class Params:
    min_size: int
    normal_size: int
    max_size: int
    strict_bits: int
    loose_bits: int

    @property
    def strict_thr(self) -> int:
        return (1 << 32) - (1 << (32 - self.strict_bits))

    @property
    def loose_thr(self) -> int:
        return (1 << 32) - (1 << (32 - self.loose_bits))

    def astuple(self):
        return (self.min_size, self.normal_size, self.max_size, self.strict_bits, self.loose_bits)


DEFAULT = Params(4096, 16384, 131072, 16, 12)


# ---------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------
def roll_hash(buf) -> np.ndarray:
    """h_i for every byte of an arena buffer; bytes before offset 0 are zeros (the TMA box delivers them so)."""
    b = np.asarray(buf, dtype=np.uint8)
    n = b.size
    out = np.empty(n, dtype=np.uint32)
    step = 1 << 22
    for s in range(0, n, step):
        e = min(n, s + step)
        lo = max(0, s - 34)
        seg = np.zeros(e - s + 34, dtype=np.uint32)          # bytes s-34 .. e-1
        seg[34 - (s - lo):] = b[lo:e]
        u = seg[:-3] | (seg[1:-2] << 8) | (seg[2:-1] << 16) | (seg[3:] << 24)   # u at positions s-31 .. e-1
        h = np.zeros(e - s, dtype=np.uint32)
        for k in range(32):
            h += u[31 - k:31 - k + e - s] * _MPOW[k]
        out[s:e] = h
    return out


def hash_at(buf: np.ndarray, pos) -> np.ndarray:
    """h at the given positions (any shape), from the 35 bytes each depends on."""
    pos = np.asarray(pos, dtype=np.int64)
    idx = pos[..., None] + np.arange(-34, 1)
    B = np.where(idx >= 0, buf[np.clip(idx, 0, buf.size - 1)], 0).astype(np.uint32)
    U = B[..., 0:32] | (B[..., 1:33] << 8) | (B[..., 2:34] << 16) | (B[..., 3:35] << 24)
    return (U * _MPOW[::-1]).sum(axis=-1, dtype=np.uint32)


def classify(h, p: Params) -> np.ndarray:
    h = np.asarray(h, dtype=np.uint64)
    return np.where(h >= p.strict_thr, STRICT, np.where(h >= p.loose_thr, LOOSE, NONE)).astype(np.int8)


@dataclass
class Cands:
    """Candidate positions (arena offsets, ascending) of a buffer under one parameter set."""
    strict: np.ndarray
    loose: np.ndarray      # every candidate (strict ones included)

    @staticmethod
    def of(buf, p: Params, h: Optional[np.ndarray] = None) -> "Cands":
        h = roll_hash(buf) if h is None else h
        return Cands(np.flatnonzero(h >= np.uint32(p.strict_thr)), np.flatnonzero(h >= np.uint32(p.loose_thr)))


def file_cuts(off: int, n: int, c: Cands, p: Params) -> List[int]:
    """Chunk ends (arena offsets) of the file [off, off+n), DESIGN §3: from prev, if rem <= min the rest is one chunk;
    else the first L in [min, min(rem, max)] whose byte prev+L-1 is a strict candidate (L < normal) or a loose one
    (L >= normal) ends the chunk; none: cut at prev + min(rem, max)."""
    out, prev, end = [], off, off + n
    while prev < end:
        rem = end - prev
        if rem <= p.min_size:
            cut = end
        else:
            limit = prev + min(rem, p.max_size)          # positions < limit
            lo, npos = prev + p.min_size - 1, prev + p.normal_size - 1
            cut = limit
            i = int(np.searchsorted(c.strict, lo))
            if i < c.strict.size and c.strict[i] < min(npos, limit):
                cut = int(c.strict[i]) + 1
            else:
                j = int(np.searchsorted(c.loose, npos))
                if j < c.loose.size and c.loose[j] < limit:
                    cut = int(c.loose[j]) + 1
        out.append(cut)
        prev = cut
    return out


def chunk_table(arena, files, p: Params, cands: Optional[Cands] = None) -> dict:
    """-> dict(ends, digests, table, n_chunks, n_unique, root) for files [(off, len)] of an arena, in file order."""
    a = np.asarray(arena, dtype=np.uint8)
    c = Cands.of(a, p) if cands is None else cands
    mv = memoryview(a)
    ends, dig = [], []
    for off, n in files:
        prev = off
        for e in file_cuts(off, n, c, p):
            ends.append(e)
            dig.append(hashlib.sha256(mv[prev:e]).digest())
            prev = e
    digests = np.frombuffer(b"".join(dig), dtype=np.uint8).reshape(-1, 32) if dig else np.zeros((0, 32), np.uint8)
    table = tc.table_ref(digests)
    return dict(ends=np.array(ends, dtype=np.uint64), digests=digests, table=table, n_chunks=len(ends),
                n_unique=table.shape[0], root=tc.merkle_ref(table))


# ---------------------------------------------------------------------------------------------------------------
# planting
# ---------------------------------------------------------------------------------------------------------------
_NBR = np.arange(-2, 35)   # the positions a plant at p may disturb


def plant(buf: np.ndarray, pos, cls, p: Params, rng: np.random.Generator) -> None:
    """Make h_q of class cls (STRICT or LOOSE) at every q in pos; no position of q-2..q+34 that was not a candidate
    becomes one (one that was depends on the re-drawn bytes and may lose its class).  Positions must be >= 36 and at
    least SPACING apart; strict_bits <= 16."""
    pos = np.asarray(pos, dtype=np.int64).ravel()
    if pos.size == 0:
        return
    cls = np.broadcast_to(np.asarray(cls, dtype=np.int8), pos.shape).copy()
    srt = np.sort(pos)
    assert srt[0] >= 36 and srt[-1] + 34 < buf.size and (np.diff(srt) >= SPACING).all()
    assert p.strict_bits <= 16 and set(np.unique(cls).tolist()) <= {LOOSE, STRICT}
    for k in range(0, pos.size, 4096):
        _plant(buf, pos[k:k + 4096], cls[k:k + 4096], p, rng)


def _plant(buf, pos, cls, p, rng):
    before = classify(hash_at(buf, pos[:, None] + _NBR), p)
    keep = np.ones(_NBR.size, dtype=bool)
    keep[2] = False
    todo = np.arange(pos.size)
    xs = np.arange(256, dtype=np.int64)
    for attempt in range(200):
        if todo.size == 0:
            return
        P, want = pos[todo], cls[todo]
        if attempt:
            buf[P - 2] = rng.integers(0, 256, P.size, dtype=np.uint8)
        H = hash_at(buf, P).astype(np.int64)
        hz = (H - buf[P - 1].astype(np.int64) * C[1] - buf[P].astype(np.int64) * C[0]) & MASK32  # bytes p-1, p = 0
        hx = (hz[:, None] + xs[None, :] * C[1]) & MASK32
        ys = (0xFF - (hx >> 24)) & 0xFF                 # byte p makes the top byte 0xFF
        ok = classify((hx + (ys << 24)) & MASK32, p) == want[:, None]
        score = np.where(ok, rng.random(ok.shape), -1.0)
        x = score.argmax(axis=1)
        assert ok[np.arange(P.size), x].all()
        buf[P - 1] = x.astype(np.uint8)
        buf[P] = ys[np.arange(P.size), x].astype(np.uint8)
        after = classify(hash_at(buf, P[:, None] + _NBR), p)
        # a neighbour that was a candidate depends on the re-drawn bytes and cannot keep its class: it may change
        good = ((after == before[todo]) | (before[todo] != NONE) | ~keep).all(axis=1) & (after[:, 2] == want)
        todo = todo[~good]
    raise AssertionError(f"{todo.size} plants did not settle")


def clear(buf: np.ndarray, ranges, p: Params, rng: np.random.Generator, h: Optional[np.ndarray] = None) -> None:
    """Re-draw the byte of every candidate in the ranges [(a, b)] until no position of them is a candidate."""
    inr = np.zeros(buf.size + 64, dtype=bool)
    for a, b in ranges:
        inr[a:b] = True
    h = roll_hash(buf) if h is None else h
    q = np.flatnonzero((h >= np.uint32(p.loose_thr)) & inr[:buf.size])
    for _ in range(1000):
        if q.size == 0:
            return
        buf[q] = rng.integers(0, 256, q.size, dtype=np.uint8)
        near = np.unique((q[:, None] + np.arange(35)).ravel())
        near = near[near < buf.size]
        near = near[inr[near]]
        q = near[classify(hash_at(buf, near), p) != NONE]
    raise AssertionError("clear did not settle")


def every_byte_loose(buf: np.ndarray, a: int, b: int, p: Params) -> None:
    """Every position of [a, b) a loose candidate (loose_bits <= 8): left to right, byte i = 0xFF - the top byte of
    h_{i-1} * M + (u_i without byte i), so that the top byte of h_i is 0xFF."""
    assert p.loose_bits <= 8 and a >= 3
    h = int(hash_at(buf, [a - 1])[0])
    w = [int(x) for x in buf[a - 3:b]]
    for i in range(3, len(w)):
        t = (h * M + (w[i - 3] | (w[i - 2] << 8) | (w[i - 1] << 16))) & MASK32
        w[i] = (0xFF - (t >> 24)) & 0xFF
        h = (t + (w[i] << 24)) & MASK32
    buf[a:b] = np.array(w[3:], dtype=np.uint8)


def dense_block(n: int, p: Params) -> np.ndarray:
    """n bytes: 35 zeros, then bytes that make every later position loose.  Tiled, every copy behaves the same (each
    position from 35 on depends on bytes of its own copy only)."""
    out = np.zeros(n, dtype=np.uint8)
    every_byte_loose(out, 35, n, p)
    return out


# ---------------------------------------------------------------------------------------------------------------
# a model of k_select_cuts_big's staging (what it stages, not what it computes)
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class Staging:
    windows: int = 0
    shrunk: int = 0              # windows with fewer regions than wanted: more than SELB_CANDS candidates
    fallbacks: int = 0           # windows without progress: one cut by select_one_cut from global memory
    crossings: int = 0           # chunks that end past the end of the window in which the chase stopped before them
    edge_cuts: int = 0           # chunks that end exactly at that window end
    cuts: List[int] = field(default_factory=list)

    def note(self, prev: int, cut: int, stop: Optional[int]) -> None:
        """Record the chunk [prev, cut); `stop` = end of the window the chase last left (None: it did not)."""
        if stop is not None and prev < stop < cut:
            self.crossings += 1
        if stop is not None and cut == stop:
            self.edge_cuts += 1
        self.cuts.append(cut)


def select_big_model(off: int, n: int, c: Cands, p: Params) -> Staging:
    """Windows of k_select_cuts_big for a whole file (more_after = 0): a window starts at the region of the chase's
    prev, wants the regions up to the file's last one (at most SELB_REGIONS) and keeps the longest prefix of them whose
    candidates fit SELB_CANDS; the chase applies the rule inside it and stops when a search range leaves it."""
    st, prev, end = Staging(), off, off + n
    allc = c.loose
    last_stop = None                     # absolute end of the window in which the chase last stopped (NX_OUT)
    while prev < end:
        st.windows += 1
        t0, t_last = prev // SCAN_TILE, (end - 1) // SCAN_TILE
        want = min(t_last - t0 + 1, SELB_REGIONS)
        edges = np.searchsorted(allc, (t0 + np.arange(want + 1)) * SCAN_TILE)
        off_r = edges - edges[0]                       # s_off
        nreg = int(np.searchsorted(off_r, SELB_CANDS, side="right")) - 1
        nreg = min(nreg, want)
        if nreg < want:
            st.shrunk += 1
        wbase, wend = t0 * SCAN_TILE, nreg * SCAN_TILE
        fend = end - wbase if wbase + wend >= end else None
        progressed = False
        while True:
            rel = prev - wbase
            if fend is not None and rel >= fend:
                break
            rem = fend - rel if fend is not None else None
            if rem is not None and rem <= p.min_size:
                cut = end
            else:
                limit = rel + (min(rem, p.max_size) if rem is not None else p.max_size)
                if limit > wend and fend is None:
                    last_stop = wbase + wend
                    break
                cut = _first_cut(prev, wbase + limit, c, p, wbase + wend)
            last_stop = st.note(prev, cut, last_stop)
            prev, progressed = cut, True
        if not progressed and prev < end:
            st.fallbacks += 1
            limit = prev + min(end - prev, p.max_size)
            cut = end if end - prev <= p.min_size else _first_cut(prev, limit, c, p, None)
            last_stop = st.note(prev, cut, last_stop)
            prev = cut
    return st


def _first_cut(prev: int, limit: int, c: Cands, p: Params, staged_end: Optional[int]) -> int:
    lo, npos = prev + p.min_size - 1, prev + p.normal_size - 1
    for arr, a, b in ((c.strict, lo, min(npos, limit)), (c.loose, npos, limit)):
        i = int(np.searchsorted(arr, a))
        if i < arr.size and arr[i] < b:
            assert staged_end is None or arr[i] < staged_end
            return int(arr[i]) + 1
    return limit


# ---------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    arena: np.ndarray
    files: List[Tuple[int, int]]                     # (arena offset, length) of every file
    params: Params
    planted: List[Tuple[int, int, str]] = field(default_factory=list)   # (position, class, which edge it hits)
    cleared: List[Tuple[int, int]] = field(default_factory=list)        # ranges without a candidate but plants
    cuts: List[Tuple[int, bool, str]] = field(default_factory=list)     # (arena offset, is a chunk end, why)
    pieces: Optional[List[List[int]]] = None          # per file: piece lengths over submits (None: one submit)
    staging: Dict[int, str] = field(default_factory=dict)   # file index -> "edge" / "crossing" / "shrink" / "fallback"
    dense: List[Tuple[int, int]] = field(default_factory=list)          # ranges with a loose candidate at every byte


def _layout(lens, align=512, lead=4096):
    offs, pos = [], lead
    for n in lens:
        pos = -(-pos // align) * align
        offs.append(pos)
        pos += n
    return offs, -(-(pos + 4096) // 4096) * 4096


def _sweep(name: str) -> Case:
    """a. Row and tile sweep over 64 MiB: in every 4 KiB region a strict candidate in row 0 at row offset region mod 35,
    and at rows 1, 16 and 31 at row offsets that run through all 128 values over the regions.  min = 64 and every
    plant >= 64 bytes after the one before, so in the files whose background is cleared every plant ends a chunk.
    Every tile start of every scan shape is a region start."""
    rng = tc.rng_for(name)
    p = Params(64, 512, 4096, 16, 12)
    total = 64 << 20
    arena = rng.integers(0, 256, total, dtype=np.uint8)
    nfile = 32
    flen = total // nfile - 8192
    files = [(k * (total // nfile) + 4096, flen) for k in range(nfile)]
    cleared = [f for k, f in enumerate(files) if k % 2 == 0]
    clear(arena, [(o, o + n) for o, n in cleared], p, rng)
    n_reg = total // SCAN_TILE
    r = np.arange(n_reg, dtype=np.int64)
    o0 = r % 35
    o1 = r % ROW
    o16 = (r * 37 + 5) % ROW
    o31 = (r * 53 + 11) % ROW
    nxt = (r + 1) % 35
    o31 = np.where(ROW - o31 + nxt < 64, o31 - 64, o31)       # keep the next region's row-0 plant a cut
    pos = np.stack([r * SCAN_TILE + o0, r * SCAN_TILE + ROW + o1, r * SCAN_TILE + 16 * ROW + o16,
                    r * SCAN_TILE + 31 * ROW + o31], axis=1)
    infile = np.zeros(total, dtype=bool)
    for o, n in files:
        infile[o + 64:o + n - 64] = True                      # leave file starts and ends to the natural content
    pos = pos[infile[pos]]
    plant(arena, pos, STRICT, p, rng)
    planted = [(int(q), STRICT, "row%d+%d" % ((q % SCAN_TILE) // ROW, q % ROW)) for q in pos]
    cuts = []
    for o, n in cleared:
        for q in pos[(pos >= o) & (pos < o + n)]:
            cuts.append((int(q) + 1, True, "cleared background: the plant ends a chunk"))
    return Case(name, arena, files, p, planted, [(o, o + n) for o, n in cleared], cuts)


def _dense(name: str) -> Case:
    """b. Regions with a candidate at every byte (loose_bits 8: a lane holds 128, a warp region up to 4096, far more
    than SCAN_POOL_BLOCK), a region with one dense row, one with dense rows 0 and 31 only, one dense stretch across a
    region edge; sparse (natural) and empty (cleared) regions on both sides."""
    rng = tc.rng_for(name)
    p = Params(64, 256, 1024, 16, 8)
    total = 8 << 20
    arena = rng.integers(0, 256, total, dtype=np.uint8)
    files = [(4096, total - 3 * 4096)]
    base = 1 << 20
    dense = [(base, base + SCAN_TILE),                                      # one whole region
             (base + 3 * SCAN_TILE + 5 * ROW, base + 3 * SCAN_TILE + 6 * ROW),  # one row: 128 in a lane
             (base + 5 * SCAN_TILE, base + 5 * SCAN_TILE + ROW),              # row 0 ...
             (base + 5 * SCAN_TILE + 31 * ROW, base + 6 * SCAN_TILE),         # ... and row 31 of a region
             (base + 8 * SCAN_TILE - 700, base + 9 * SCAN_TILE + 900),       # across a region edge
             (base + 12 * SCAN_TILE, base + 16 * SCAN_TILE)]                  # four whole regions
    empty = [(base - 2 * SCAN_TILE, base - 40), (base + SCAN_TILE + 40, base + 3 * SCAN_TILE),
             (base + 16 * SCAN_TILE + 40, base + 18 * SCAN_TILE)]
    clear(arena, empty, p, rng)
    for a, b in dense:
        every_byte_loose(arena, a, b, p)
    planted = [(q, LOOSE, "dense") for a, b in dense for q in (a, b - 1)]
    return Case(name, arena, files, p, planted, empty, dense=dense)


def _boundary_patterns(p: Params):
    """(offset from prev, class, is the chunk end, name): every off-by-one pair of the cut rule."""
    mn, nm, mx = p.min_size, p.normal_size, p.max_size
    return [(mn - 2, STRICT, False, "strict at prev+min-2"), (mn - 1, STRICT, True, "strict at prev+min-1"),
            (nm - 2, LOOSE, False, "loose at prev+normal-2"), (nm - 1, LOOSE, True, "loose at prev+normal-1"),
            (nm - 2, STRICT, True, "strict at prev+normal-2"),
            (mx - 1, LOOSE, True, "loose at prev+max-1"), (mx, STRICT, False, "strict at prev+max")]


def _boundaries(name: str) -> Case:
    """c. The cut rule's boundaries at the default parameters: each pattern in a file of its own whose background is
    cleared (prev = the file start), and the same patterns one after another inside big files, after a chunk the
    pattern before ended; files of length min, min+1, max, max+1, 4 MiB-1 and 4 MiB (natural content and cleared)."""
    rng = tc.rng_for(name)
    p = DEFAULT
    pats = _boundary_patterns(p)
    small = [p.max_size + 9000] * len(pats)
    big_len = (4 << 20) + 3 * p.max_size
    sizes = [p.min_size, p.min_size + 1, p.max_size, p.max_size + 1, (4 << 20) - 1, 4 << 20]
    lens = small + [big_len, (4 << 20) - 1, 4 << 20] + sizes + sizes
    offs, total = _layout(lens)
    arena = rng.integers(0, 256, total, dtype=np.uint8)
    files = list(zip(offs, lens))
    clr = [(o, o + n) for o, n in files[:len(pats) + 3 + len(sizes)]]
    clear(arena, clr, p, rng)
    planted, cuts, plants = [], [], []
    for (o, _), (d, cls, is_cut, why) in zip(files, pats):
        plants.append((o + d, cls))
        planted.append((o + d, cls, why))
        cuts.append((o + d + 1, is_cut, why))
    for fi in range(len(pats), len(pats) + 3):          # big files: patterns in sequence
        o, n = files[fi]
        prev = o + p.max_size                            # the background is cleared: the first chunk is forced
        k = 0
        while True:
            d, cls, is_cut, why = pats[k % len(pats)]
            q = prev + d
            nxt = q + 1 if is_cut else prev + p.max_size
            if nxt + p.max_size > o + n:
                break
            plants.append((q, cls))
            planted.append((q, cls, why + " (big file)"))
            cuts.append((q + 1, is_cut, why + " (big file)"))
            cuts.append((nxt, True, "chunk after " + why))
            prev = nxt
            k += 1
    for cls in (STRICT, LOOSE):
        sel = [q for q, c in plants if c == cls]
        plant(arena, sel, cls, p, rng)
    return Case(name, arena, files, p, planted, clr, cuts)


def _windows(name: str) -> Case:
    """d. Big files at the default parameters and the big-file selector's 16 MiB windows: strict candidates at the
    last byte of the first window and at the first byte after it, a candidate-free stretch longer than max across the
    window edge, and a file with a loose candidate every 512 bytes over 20 MiB (more than SELB_CANDS per window, so
    windows shrink).  The window edges are those of the staging model."""
    rng = tc.rng_for(name)
    p = DEFAULT
    W = SELB_REGIONS * SCAN_TILE
    lens = [W + (3 << 20), W + (5 << 20) + 777, W + (4 << 20), 24 << 20]
    offs, total = _layout(lens, align=SCAN_TILE)
    arena = rng.integers(0, 256, total, dtype=np.uint8)
    files = list(zip(offs, lens))
    o0, o1, o2, o3 = offs
    e0, e1, e2 = o0 + W, o1 + W, o2 + W           # first window = the regions from the file start
    clear(arena, [(e0 - (1 << 20), e0 - 1), (e1 - (1 << 20), e1 + (64 << 10)), (e2 - 200_000, e2 + 200_000)], p, rng)
    plant(arena, [e0 - 1, e1], STRICT, p, rng)
    planted = [(e0 - 1, STRICT, "last byte of the first window"), (e1, STRICT, "first byte after the first window")]
    cleared = [(e0 - (1 << 20), e0 - 1), (e1 - (1 << 20), e1), (e1 + 1, e1 + (64 << 10)), (e2 - 200_000, e2 + 200_000)]
    q = o3 + 300 + np.arange(0, 20 << 20, 512)
    plant(arena, q, LOOSE, p, rng)
    planted += [(int(x), LOOSE, "dense window") for x in q]
    return Case(name, arena, files, p, planted, cleared,
                [(e0, True, "cut at the end of the first window"), (e1 + 1, True, "cut one byte past the first window")],
                staging={0: "edge", 1: "crossing", 2: "crossing", 3: "shrink"})


def _fallback(name: str) -> Case:
    """d. Every byte loose (loose_bits 8) over 1 MiB of a 40 MiB file: a staged window holds SELB_CANDS candidates,
    16 KiB of file, while a search range reaches prev + max = 128 KiB, so the chase makes no progress and each cut comes
    from select_one_cut over global memory."""
    rng = tc.rng_for(name)
    p = Params(4096, 16384, 131072, 16, 8)
    n = 40 << 20
    offs, total = _layout([n, 5 << 20], align=SCAN_TILE)
    arena = rng.integers(0, 256, total, dtype=np.uint8)
    a = offs[0] + (12 << 20)
    blk = dense_block(SCAN_TILE, p)
    arena[a:a + (1 << 20)] = np.tile(blk, (1 << 20) // SCAN_TILE)
    every_byte_loose(arena, offs[1] + (1 << 20), offs[1] + (1 << 20) + 20000, p)
    d1 = offs[1] + (1 << 20)
    return Case(name, arena, list(zip(offs, [n, 5 << 20])), p, staging={0: "fallback", 1: "fallback"},
                dense=[(a + k + 35, a + k + SCAN_TILE) for k in range(0, 1 << 20, SCAN_TILE)] + [(d1, d1 + 20000)])


def _long_chunks(mx: int, name: str) -> Case:
    """f. max = 1 MiB or 4 MiB over zero runs: chunks longer than the 64 length classes of k_len_order cover (2 KiB
    each, the last one open-ended)."""
    rng = tc.rng_for(name)
    p = Params(4096, 16384, mx, 16, 12)
    lens = [3 * mx + 5, mx, mx + 1, 10 << 20, 300_000]
    offs, total = _layout(lens)
    arena = np.zeros(total, dtype=np.uint8)
    arena[offs[3] + (5 << 20):offs[3] + (6 << 20)] = rng.integers(0, 256, 1 << 20, dtype=np.uint8)
    arena[offs[4]:offs[4] + lens[4]] = rng.integers(0, 256, lens[4], dtype=np.uint8)
    return Case(name, arena, list(zip(offs, lens)), p,
                cuts=[(offs[0] + mx, True, "forced at max"), (offs[0] + 3 * mx, True, "forced at max")])


def _continuation(big: bool, name: str) -> Case:
    """e. Files in pieces over submits (MKSNAP_X_MORE / MKSNAP_X_CONT): strict candidates at the last byte of a piece,
    at the first byte of the next and at the one after it; an open chunk of exactly max-1 bytes (cleared background:
    forced cuts every max, the piece ends one byte before the next); pieces whose end is not a multiple of 4 KiB, so the
    last staged region of a big piece reaches past it.  Big: both pieces of a file take k_select_cuts_big."""
    rng = tc.rng_for(name)
    p = DEFAULT
    mx = p.max_size
    K = ((5 << 20) if big else 600_000) // mx
    first = K * mx + mx - 1                # cleared background: forced cuts every max, so the piece leaves max - 1 open
    short = first - 1000                   # ... or max - 1001
    rest = (9 << 19) if big else 700_000
    lens = [first + rest] * 5 + [3 * mx + 1234]
    pieces = [[first, rest], [short, rest + 1000], [short, rest + 1000], [first, rest], [first, rest],
              [mx + 1000, mx, mx + 234]]
    offs, total = _layout(lens)
    arena = rng.integers(0, 256, total, dtype=np.uint8)
    files = list(zip(offs, lens))
    clr = [(o, o + n) for o, n in files[:4]]
    clear(arena, clr, p, rng)
    o = offs
    spots = [(o[0] + first - 1, "last byte of a piece"), (o[1] + short, "first byte of a continuation"),
             (o[2] + short + 1, "second byte of a continuation"),
             (o[5] + mx + 999, "last byte of a piece"), (o[5] + 2 * mx + 1000, "first byte of a piece")]
    plant(arena, [s for s, _ in spots], STRICT, p, rng)
    planted = [(s, STRICT, w) for s, w in spots]
    cuts = [(o[0] + first, True, "a candidate ends the chunk at the piece end"),
            (o[1] + short + 1, True, "after the continuation's first byte"),
            (o[2] + short + 2, True, "after the continuation's second byte"),
            (o[3] + first, False, "the open chunk is max - 1 long"),
            (o[3] + first + 1, True, "forced one byte into the continuation")]
    clr = [(a, b) for a, b in clr if not any(a <= s < b for s, _ in spots)] + \
          [(o[k], s) for k, (s, _) in zip(range(3), spots)]
    return Case(name, arena, files, p, planted, clr, cuts, pieces=pieces)


def _long_continuation(name: str) -> Case:
    """f. max = 1 MiB: a zero file whose open chunk (max - 1 bytes) continues at an arena offset >= carry_bytes."""
    rng = tc.rng_for(name)
    mx = 1 << 20
    p = Params(4096, 16384, mx, 16, 12)
    lens = [4 * mx + 4096, 2 * mx + 77]
    pieces = [[2 * mx - 1, 2 * mx + 4097], [2 * mx + 77]]
    offs, total = _layout(lens)
    arena = np.zeros(total, dtype=np.uint8)
    arena[offs[1]:offs[1] + lens[1]] = rng.integers(0, 256, lens[1], dtype=np.uint8)
    return Case(name, arena, list(zip(offs, lens)), p, pieces=pieces,
                cuts=[(offs[0] + mx, True, "forced"), (offs[0] + 2 * mx - 1, False, "piece end"),
                      (offs[0] + 2 * mx, True, "forced, one byte into the continuation")])


def _registry(items) -> Dict[str, Callable[[], Case]]:
    return {name: partial(fn, *args, name) for name, fn, *args in items}


SCAN_CASES = _registry([("sweep", _sweep), ("dense", _dense)])
SELECT_CASES = _registry([("boundaries", _boundaries), ("windows", _windows), ("fallback", _fallback),
                          ("long-1MiB", _long_chunks, 1 << 20), ("long-4MiB", _long_chunks, 4 << 20)])
CONT_CASES = _registry([("cont-small", _continuation, False), ("cont-big", _continuation, True),
                        ("cont-long", _long_continuation)])
ALL_CASES = {**SCAN_CASES, **SELECT_CASES, **CONT_CASES}


def case(name: str) -> Case:
    return ALL_CASES[name]()
