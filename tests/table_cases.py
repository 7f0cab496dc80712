"""Crafted chunk tables and a plain Python reference of the table, its Merkle root and the range exchange (test
infrastructure only).  Written from DESIGN §3 (table = bytewise-sorted unique digests, fan-out-256 Merkle root) and §7
(rank r owns the digests whose big-endian 64-bit prefix p has floor(p*R / 2^64) == r); it uses no oracle/ code, so it
stays independent of what it checks.

SHA-256 output is uniform, so real content never reaches most branches of K3 (32-bit radix sort, tie fix-up of runs of
equal prefix, long-run vote, overflow of the long-run list) or of the exchange (prefixes on a range boundary, crafted
range sizes, skew).  mksnap_chunks_add appends any 32-byte rows, so the cases here are rows chosen to reach them.
Every case is deterministic: its generator is seeded from its name."""
from __future__ import annotations

import hashlib
import random
import zlib
from dataclasses import dataclass, field
from functools import partial
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

CHUNKS_ADD_MAX = 65536  # rows per mksnap_chunks_add call
FIX_SHORT = 64          # K3: a run of more than this many rows of equal 32-bit prefix is a "long run"
FIX_LONG_CAP = 8192     # K3: long runs listed for k_fix_long_runs; further ones are sorted in k_fix_ties
ROW_ORDERS = ("random", "sorted", "reverse")
U64 = 1 << 64


# ---------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------
def _as_rows(rows) -> List[bytes]:
    if isinstance(rows, np.ndarray):
        b = np.ascontiguousarray(rows, dtype=np.uint8).tobytes()
        return [b[i:i + 32] for i in range(0, len(b), 32)]
    return [bytes(r) for r in rows]


def _to_array(rows: List[bytes]) -> np.ndarray:
    return np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(-1, 32).copy() if rows else np.zeros((0, 32), np.uint8)


def table_ref(rows) -> np.ndarray:
    """The chunk table: the distinct rows in bytewise order."""
    return _to_array(sorted(set(_as_rows(rows))))


def merkle_ref(table) -> bytes:
    """Fan-out-256 Merkle root, hashed at least once: SHA256("") for no rows, SHA256(row) for one row."""
    cur = _as_rows(table)
    if not cur:
        return hashlib.sha256(b"").digest()
    while True:
        cur = [hashlib.sha256(b"".join(cur[i:i + 256])).digest() for i in range(0, len(cur), 256)]
        if len(cur) == 1:
            return cur[0]


def prefix64(row) -> int:
    return int.from_bytes(bytes(row[:8]), "big")


def owner(prefix: int, R: int) -> int:
    return (prefix * R) >> 64


def boundary(j: int, R: int) -> int:
    """b_j = ceil(j * 2^64 / R): the least prefix rank j owns (b_0 = 0, b_R = 2^64)."""
    return -((-(j << 64)) // R)


def ranges_ref(union: np.ndarray, R: int) -> List[np.ndarray]:
    """The global sorted-unique table cut into the R owner ranges."""
    out: List[List[bytes]] = [[] for _ in range(R)]
    for row in _as_rows(union):
        out[owner(prefix64(row), R)].append(row)
    return [_to_array(x) for x in out]


def bounds_ref(table: np.ndarray, R: int) -> List[int]:
    """For a sorted table: bounds[j] = rows owned by ranks below j (R+1 entries)."""
    owners = [owner(prefix64(row), R) for row in _as_rows(table)]
    return [sum(1 for o in owners if o < j) for j in range(R + 1)]


def prefix_runs(rows) -> Dict[int, int]:
    """{run length: count} of the runs of >= 2 rows that share their top 32 bits (the radix key)."""
    counts: Dict[bytes, int] = {}
    for r in _as_rows(rows):
        counts[r[:4]] = counts.get(r[:4], 0) + 1
    out: Dict[int, int] = {}
    for c in counts.values():
        if c > 1:
            out[c] = out.get(c, 0) + 1
    return out


# ---------------------------------------------------------------------------------------------------------------
# row builders
# ---------------------------------------------------------------------------------------------------------------
def rng_for(name: str) -> np.random.Generator:
    return np.random.default_rng(zlib.crc32(name.encode()))


def craft(n: int, prefix32, b4_7=0, tail=None) -> np.ndarray:
    """n rows: bytes 0-3 = prefix32 (the radix key), 4-7 = b4_7 (both big-endian, scalar or per row), 8-31 = tail
    ([n, 24] or [24] bytes; zeros if None)."""
    out = np.zeros((n, 32), np.uint8)
    out[:, 0:4] = np.ascontiguousarray(np.broadcast_to(np.asarray(prefix32, dtype=">u4"), (n,))).view(np.uint8).reshape(n, 4)
    out[:, 4:8] = np.ascontiguousarray(np.broadcast_to(np.asarray(b4_7, dtype=">u4"), (n,))).view(np.uint8).reshape(n, 4)
    if tail is not None:
        out[:, 8:] = tail
    return out


def rows_with_prefix64(prefixes: Sequence[int], rng: np.random.Generator) -> np.ndarray:
    out = rng.integers(0, 256, (len(prefixes), 32), dtype=np.uint8)
    for i, p in enumerate(prefixes):
        out[i, :8] = np.frombuffer(int(p).to_bytes(8, "big"), dtype=np.uint8)
    return out


def distinct_prefixes(n: int, rng: np.random.Generator, avoid=()) -> np.ndarray:
    """n distinct 32-bit prefixes in random order."""
    got, seen = [], set(int(a) for a in avoid)
    while len(got) < n:
        for p in rng.integers(0, 1 << 32, 2 * n, dtype=np.uint64).tolist():
            if p not in seen and len(got) < n:
                seen.add(p)
                got.append(p)
    return np.array(got, dtype=np.uint64)


def tie_run(prefix: int, length: int, pos: int, order: str, rng: np.random.Generator) -> np.ndarray:
    """`length` rows equal except in byte `pos` (>= 4), all sharing the 32-bit prefix.  A byte holds 256 values, so a
    run longer than 256 rows mixes distinct rows and duplicates."""
    base = craft(1, prefix, int(rng.integers(0, 1 << 32)), rng.integers(0, 256, 24, dtype=np.uint8))[0]
    vals = rng.permutation(256)[:length] if length <= 256 else rng.integers(0, 256, length)
    if order == "sorted":
        vals = np.sort(vals)
    elif order == "reverse":
        vals = np.sort(vals)[::-1]
    out = np.repeat(base[None, :], length, axis=0)
    out[:, pos] = vals
    return out


def split_calls(rows: np.ndarray, at_most: int = CHUNKS_ADD_MAX) -> List[np.ndarray]:
    return [rows[i:i + at_most] for i in range(0, rows.shape[0], at_most)]


def random_rows(n: int, rng: np.random.Generator) -> np.ndarray:
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------
# single-table cases (sort, unique, Merkle root)
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    calls: List[np.ndarray]                 # mksnap_chunks_add calls, in order
    runs: Optional[Dict[int, int]] = None   # claimed prefix_runs() of all rows
    n_unique: Optional[int] = None          # claimed size of the table
    long_runs: Optional[int] = None         # claimed number of runs longer than FIX_SHORT

    @property
    def rows(self) -> np.ndarray:
        return np.concatenate(self.calls) if self.calls else np.zeros((0, 32), np.uint8)


TIE_LENGTHS = (2, 3, 63, 64, 65, 1000, 2048)   # FIX_SHORT = 64 sits between 64 and 65
TIE_BYTES = (4, 7, 8, 31)                       # first byte past the radix key, last byte of the u64 key, first past it, last
ODD_OFFSETS = (0, 1, 256, 512, 1023)            # thread 0, thread 0's first row, thread 255's first row, one stride on, last
ODD_RUN = 1024
RADIX_NS = (1, 2, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 65537)
MERKLE_NS = (0, 1, 2, 255, 256, 257, 258, 511, 512, 513, 65535, 65536, 65537, 131073)
OVERFLOW_RUNS = 8300                            # > FIX_LONG_CAP runs of 65 rows


def _ties(pos: int, order: str, name: str) -> Case:
    rng = rng_for(name)
    pref = distinct_prefixes(len(TIE_LENGTHS) + 500, rng)
    blocks = [tie_run(int(p), n, pos, order, rng) for p, n in zip(pref, TIE_LENGTHS)]
    filler = random_rows(500, rng)
    filler[:, :4] = craft(500, pref[len(TIE_LENGTHS):])[:, :4]   # singletons: no prefix shared with anything
    blocks += [filler[i:i + 100] for i in range(0, 500, 100)]
    rows = np.concatenate([blocks[i] for i in rng.permutation(len(blocks))])  # runs contiguous, their order kept
    return Case(name, [rows], runs={n: 1 for n in TIE_LENGTHS}, long_runs=3)


def _one_odd(off: int, name: str) -> Case:
    """Two long runs of ODD_RUN rows, duplicates of one digest except the row at `off`, which differs only in byte 31:
    below the duplicates in one run, above them in the other, so one of the two is out of order wherever it sits."""
    rng = rng_for(name)
    pref = distinct_prefixes(2, rng)
    blocks = []
    for p, delta in zip(pref, (-1, +1)):
        d = craft(1, int(p), int(rng.integers(0, 1 << 32)), rng.integers(0, 256, 24, dtype=np.uint8))[0]
        d[31] = 0x80
        run = np.repeat(d[None, :], ODD_RUN, axis=0)
        run[off, 31] = 0x80 + delta
        blocks.append(run)
    return Case(name, [np.concatenate(blocks)], runs={ODD_RUN: 2}, n_unique=4, long_runs=2)


def _half_dup(name: str) -> Case:
    """One run of 2048 rows: half one digest, half distinct rows with the same 32-bit prefix, shuffled."""
    rng = rng_for(name)
    p = int(distinct_prefixes(1, rng)[0])
    dup = np.repeat(craft(1, p, 7, rng.integers(0, 256, 24, dtype=np.uint8)), 1024, axis=0)
    dis = craft(1024, p, rng.integers(0, 1 << 32, 1024, dtype=np.uint64), rng.integers(0, 256, (1024, 24), dtype=np.uint8))
    rows = np.concatenate([dup, dis])[rng.permutation(2048)]
    return Case(name, [rows], runs={2048: 1}, n_unique=1025, long_runs=1)


def _overflow(name: str) -> Case:
    """OVERFLOW_RUNS runs of 65 rows with distinct prefixes (more long runs than FIX_LONG_CAP): every third run has
    distinct rows, the others are 65 copies of one digest."""
    rng = rng_for(name)
    pref = distinct_prefixes(OVERFLOW_RUNS, rng)
    blocks = []
    for k, p in enumerate(pref):
        if k % 3 == 0:
            blocks.append(craft(65, int(p), rng.integers(0, 1 << 32, 65, dtype=np.uint64), rng.integers(0, 256, (65, 24), dtype=np.uint8)))
        else:
            blocks.append(np.repeat(craft(1, int(p), 0, rng.integers(0, 256, 24, dtype=np.uint8)), 65, axis=0))
    rows = np.concatenate(blocks)
    rows = rows[rng.permutation(rows.shape[0])]
    n_mixed = (OVERFLOW_RUNS + 2) // 3
    return Case(name, split_calls(rows), runs={65: OVERFLOW_RUNS}, long_runs=OVERFLOW_RUNS,
                n_unique=65 * n_mixed + (OVERFLOW_RUNS - n_mixed))


def _radix_n(n: int, name: str) -> Case:
    """n random rows; about 1/8 repeat an earlier row and 1/8 take an earlier row's 32-bit prefix with a new tail."""
    rng = rng_for(name)
    rows = random_rows(n, rng)
    pick = rng.random(n)
    for i in range(1, n):
        j = int(rng.integers(0, i))
        if pick[i] < 0.125:
            rows[i] = rows[j]
        elif pick[i] < 0.25:
            rows[i, :4] = rows[j, :4]
    return Case(name, split_calls(rows))


def _extremes(run: int, name: str) -> Case:
    """Runs with prefix 00000000 and FFFFFFFF (they sort to the first and to the last rows: the gallop that finds a
    run's end reaches n), fed in the opposite order; bytes 4.. differ, with one duplicate in each run."""
    rng = rng_for(name)
    lo = craft(run, 0, rng.integers(0, 1 << 32, run, dtype=np.uint64), rng.integers(0, 256, (run, 24), dtype=np.uint8))
    hi = craft(run, 0xFFFFFFFF, rng.integers(0, 1 << 32, run, dtype=np.uint64), rng.integers(0, 256, (run, 24), dtype=np.uint8))
    lo[-1], hi[-1] = lo[0], hi[0]
    mid = random_rows(3000, rng)
    mid[:, :4] = craft(3000, distinct_prefixes(3000, rng, avoid=(0, 0xFFFFFFFF)))[:, :4]
    return Case(name, [np.concatenate([hi, mid, lo])], runs={run: 2}, n_unique=3000 + 2 * (run - 1),
                long_runs=2 if run > FIX_SHORT else 0)


def _digit(d: int, kind: str, name: str) -> Case:
    """Radix digit d (byte 3-d of the key; pass d sorts it) equal in every row ("const"), or taking all 256 values
    while the other three key bytes are fixed ("all256": 256 runs of 19-20 rows)."""
    rng = rng_for(name)
    n = 5000
    rows = random_rows(n, rng)
    b = 3 - d
    if kind == "const":
        rows[:, b] = 0xA5
    else:
        rows[:, :4] = rng.integers(0, 256, 4, dtype=np.uint8)
        rows[:, b] = rng.permutation(np.arange(n) % 256)
    return Case(name, [rows])


def _merkle(n: int, name: str) -> Case:
    """n distinct random rows, plus repeats of up to ten of them (n_unique = n)."""
    rng = rng_for(name)
    rows = random_rows(n, rng)
    rows = np.concatenate([rows, rows[: min(n, 10)]])
    return Case(name, split_calls(rows[rng.permutation(rows.shape[0])]), n_unique=n)


def _registry(items) -> Dict[str, Callable]:
    """(name, builder, *args) -> {name: builder(*args, name)}, built on demand."""
    return {name: partial(fn, *args, name) for name, fn, *args in items}


SORT_CASES = _registry(
    [(f"ties-byte{p}-{o}", _ties, p, o) for p in TIE_BYTES for o in ROW_ORDERS]
    + [(f"one-odd-at-{off}", _one_odd, off) for off in ODD_OFFSETS]
    + [("half-duplicates-2048", _half_dup), ("long-run-list-overflow", _overflow)]
    + [(f"radix-n{n}", _radix_n, n) for n in RADIX_NS]
    + [(f"prefix-extremes-run{r}", _extremes, r) for r in (5, 100)]
    + [(f"digit{d}-{k}", _digit, d, k) for d in range(4) for k in ("const", "all256")])
MERKLE_CASES = _registry([(f"merkle-n{n}", _merkle, n) for n in MERKLE_NS])


def case(name: str) -> Case:
    return (SORT_CASES.get(name) or MERKLE_CASES[name])()


def mix_case() -> Case:
    """Rows injected next to the chunks of a real CDC submit: tie runs, a long mixed run and duplicates across calls."""
    rng = rng_for("cdc-mix")
    pref = distinct_prefixes(3, rng)
    a = tie_run(int(pref[0]), 40, 31, "random", rng)
    b = tie_run(int(pref[1]), 300, 8, "reverse", rng)
    c = random_rows(5000, rng)
    rows = np.concatenate([a, b, c, c[:700], a[:5]])
    rows = rows[rng.permutation(rows.shape[0])]
    return Case("cdc-mix", split_calls(rows, 2000), runs={40: 1, 300: 1})


# ---------------------------------------------------------------------------------------------------------------
# range exchange cases
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class ExCase:
    name: str
    R: int
    ranks: List[List[np.ndarray]]                  # per rank: its chunks_add calls
    sizes: Optional[List[int]] = None              # claimed rows of every owner range of the global table
    edges: List[Tuple[int, int]] = field(default_factory=list)  # (prefix64, owner) of rows the case holds
    cap: int = 0                                   # max_chunks of every engine (0: room for every row)

    @property
    def rows(self) -> np.ndarray:
        calls = [c for r in self.ranks for c in r]
        return np.concatenate(calls) if calls else np.zeros((0, 32), np.uint8)

    def rank_rows(self, r: int) -> np.ndarray:
        return np.concatenate(self.ranks[r]) if self.ranks[r] else np.zeros((0, 32), np.uint8)


def _spread(rows: np.ndarray, R: int, rng: np.random.Generator, dup: float, on=None) -> List[List[np.ndarray]]:
    """Each row to one random rank of `on` (default: all), a fraction `dup` also to a second one."""
    on = list(range(R)) if on is None else list(on)
    per: List[List[np.ndarray]] = [[] for _ in range(R)]
    for i in range(rows.shape[0]):
        k = on[int(rng.integers(0, len(on)))]
        per[k].append(rows[i])
        if len(on) > 1 and rng.random() < dup:
            per[on[(on.index(k) + 1 + int(rng.integers(0, len(on) - 1))) % len(on)]].append(rows[i])
    return [split_calls(np.array(p, dtype=np.uint8).reshape(-1, 32)) if p else [] for p in per]


def _edge_prefixes(R: int, js) -> List[Tuple[int, int]]:
    out = [(0, 0), (U64 - 1, R - 1)]
    for j in js:
        b = boundary(j, R)
        out += [(b - 1, j - 1), (b, j)]
    return out


def _boundaries(R: int, name: str) -> ExCase:
    """Rows whose prefix is b_j - 1 and b_j for every boundary, 0 and 2^64 - 1 (two tails each), random rows; spread
    over the ranks, a third of them on two ranks."""
    rng = rng_for(name)
    edges = _edge_prefixes(R, range(1, R))
    rows = np.concatenate([rows_with_prefix64([p for p, _ in edges] * 2, rng), random_rows(300, rng)])
    return ExCase(name, R, _spread(rows[rng.permutation(rows.shape[0])], R, rng, 1 / 3), edges=edges)


def _sized(sizes: List[int], name: str) -> ExCase:
    """sizes[j] distinct rows with prefixes uniform in rank j's range, spread over the ranks (a fifth on two)."""
    rng = rng_for(name)
    R = len(sizes)
    py = random.Random(zlib.crc32(name.encode()))
    pref = [boundary(j, R) + py.randrange(boundary(j + 1, R) - boundary(j, R)) for j in range(R) for _ in range(sizes[j])]
    rows = rows_with_prefix64(pref, rng)
    return ExCase(name, R, _spread(rows[rng.permutation(rows.shape[0])], R, rng, 0.2), sizes=list(sizes))


def _skew_refused(name: str) -> ExCase:
    """Every row in range 0, more than rank 0's max_chunks in total (each rank alone fits)."""
    rng = rng_for(name)
    R, per = 3, 600
    b1 = boundary(1, R)
    py = random.Random(zlib.crc32(name.encode()))
    ranks = [[rows_with_prefix64([py.randrange(b1) for _ in range(per)], rng)] for _ in range(R)]
    return ExCase(name, R, ranks, sizes=[R * per, 0, 0], cap=1000)


EX_SIZES = {
    "sizes-255-1-0-256-258": [255, 1, 0, 256, 258],
    "sizes-1-1-1-1-253": [1, 1, 1, 1, 253],          # the first Merkle group spans all five ranks
    "sizes-256x4-1": [256, 256, 256, 256, 1],
    "sizes-u1": [0, 0, 1, 0],
    "sizes-u65537-r3": [21845, 21846, 21846],        # 257 level-1 rows after the exchange
    "skew-all-in-last": [0, 0, 0, 1000],
}
EX_CASES = _registry([(f"boundaries-r{R}", _boundaries, R) for R in (2, 3, 5, 7, 8)]
                     + [(name, _sized, sizes) for name, sizes in EX_SIZES.items()]
                     + [("skew-refused", _skew_refused)])


def ex_case(name: str) -> ExCase:
    return EX_CASES[name]()


R_MAX = 1024
WIDE_RANKS = (0, 1, 517, 1023)   # the only ranks of the 1024-rank case that hold rows


def wide_case() -> ExCase:
    """R = 1024 with rows on four ranks only: boundary prefixes around b_1, b_2, b_512, b_1023, prefixes owned by rank
    1023 (>= 0xFFC0...), 0 and 2^64 - 1, random rows."""
    name = "r1024"
    rng = rng_for(name)
    R = R_MAX
    edges = _edge_prefixes(R, (1, 2, 512, 1023))
    top = [0xFFC0 << 48, (0xFFC0 << 48) + 12345, U64 - 2]
    edges += [(p, R - 1) for p in top]
    rows = np.concatenate([rows_with_prefix64([p for p, _ in edges] * 2, rng), random_rows(300, rng)])
    return ExCase(name, R, _spread(rows[rng.permutation(rows.shape[0])], R, rng, 1 / 3, on=WIDE_RANKS), edges=edges, cap=4096)
