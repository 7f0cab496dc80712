"""Serial-stream SHA-256 cases (K4, k_sha256_streams) and long chunks (K2, k_sha256_ranges), with a plain reference
(test infrastructure only).  The reference of a stream is hashlib.sha256 over the concatenation of its pieces; of a
chunk, hashlib over its bytes, with the table and root of tests/table_cases.py.  Nothing here uses oracle/ code.

A case is a list of submits: the arena contents (random bytes, or the engine's synthetic generator so that a device can
fill a large arena without an upload) and its ranges (arena_off, len, slot, flags).  A stream's pieces travel in
increasing submits; every piece but the last carries MKSNAP_R_MORE.  The reference walks the submits in order, so only
one arena is materialised at a time.  Every case is deterministic: its generator is seeded from its name.

What the suite otherwise never submits:
- ragged_many: about 2^18 ranges in one submit, so each lane of K4 refills many times while its neighbours are deep
  inside long streams;
- continued_mix: streams of 1-4 pieces over 4 submits, every final-tail class after 0-3 resumed pieces, finals of 0
  bytes, fresh streams next to resumed ones, slots reused after their stream finished;
- long_streams: bit lengths of 2^32 and more (the high length word);
- long_chunks: chunks of 2^29 - 1 .. 2^29 + 64 bytes through K2;
- contract(): what the engine accepts and refuses, each refusal followed by a valid session on the same handle."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from functools import lru_cache
from typing import Dict, List, Optional, Tuple

import numpy as np

from tests import table_cases as tc

R_MORE = 1                  # MKSNAP_R_MORE
E_INVAL, E_CAPACITY, E_STATE = -1, -4, -5
H100_SMS = 132
K4_PAIRS_PER_SM = 4         # mksnap_arena_submit launches min(ceil(n / 32), 4 * SMs) pairs of 32 lanes
GOLDEN64 = 0x9E3779B97F4A7C15
RANGE_DTYPE = np.dtype([("arena_off", "<u8"), ("len", "<u8"), ("stream", "<u4"), ("flags", "<u4")])  # mksnap_range
rng_for = tc.rng_for


# ---------------------------------------------------------------------------------------------------------------
# content and reference
# ---------------------------------------------------------------------------------------------------------------
def synth(byte_off: int, n: int, seed: int) -> np.ndarray:
    """mksnap_synth_fill's content (include/mksnap.h): LE u64 word i (absolute in the slot) =
    splitmix64-finaliser(seed + (i + 1) * GOLDEN64).  byte_off and n multiples of 8."""
    assert byte_off % 8 == 0 and n % 8 == 0
    out = np.empty(n // 8, dtype=np.uint64)
    w0, step = byte_off // 8, 1 << 22
    for a in range(0, out.size, step):
        z = np.arange(w0 + a + 1, w0 + min(a + step, out.size) + 1, dtype=np.uint64)
        z *= np.uint64(GOLDEN64)
        z += np.uint64(seed)
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
        out[a:a + z.size] = z
    return out.view(np.uint8)


@dataclass
class Submit:
    used: int
    ranges: np.ndarray                  # RANGE_DTYPE
    data: Optional[np.ndarray] = None   # arena[0, used), or
    seed: Optional[int] = None          # synth(0, used, seed) (used a multiple of 16)

    def arena(self) -> np.ndarray:
        return self.data if self.data is not None else synth(0, self.used, self.seed)


@dataclass
class Stream:
    slot: int
    pieces: List[Tuple[int, int, int]]  # (submit, arena_off, len); all but the last carry MKSNAP_R_MORE

    @property
    def more(self) -> int:
        return len(self.pieces) - 1

    @property
    def total(self) -> int:
        return sum(n for _, _, n in self.pieces)


@dataclass
class Case:
    name: str
    arena_bytes: int                    # capacity of each arena the case needs
    max_extents: int                    # = max_streams
    submits: List[Submit]
    streams: List[Stream] = field(default_factory=list)
    expect: Dict[int, bytes] = field(default_factory=dict)  # slot -> digest of the stream that finished last on it
    n_streams: int = 0                  # highest finished slot + 1


def reference(submits: List[Submit]) -> Tuple[Dict[int, bytes], int]:
    """hashlib.sha256 over the concatenation of every stream's pieces -> ({slot: digest}, highest finished slot + 1).
    Asserts the piece rules on the way: MORE pieces are non-empty multiples of 64, one piece per slot per submit, no
    stream left open at the end."""
    open_: Dict[int, "hashlib._Hash"] = {}
    out: Dict[int, bytes] = {}
    for s in submits:
        a = memoryview(s.arena())
        assert len(set(int(x) for x in s.ranges["stream"])) == s.ranges.size, "two pieces of one slot in one submit"
        for off, n, slot, flags in s.ranges.tolist():
            assert off % 16 == 0 and off + n <= s.used
            h = open_.pop(slot, None) or hashlib.sha256()
            h.update(a[off:off + n])
            if flags & R_MORE:
                assert n > 0 and n % 64 == 0, "a MORE piece is a non-empty multiple of 64 bytes"
                open_[slot] = h
            else:
                out[slot] = h.digest()
        del a
    assert not open_, "a stream is left open"
    return out, max(out) + 1 if out else 0


def ranges_array(rows) -> np.ndarray:
    return np.array([tuple(r) for r in rows], dtype=RANGE_DTYPE) if rows else np.zeros(0, RANGE_DTYPE)


def _case(name, arena_bytes, max_extents, contents, streams, rng) -> Case:
    """contents: per submit (used, data, seed).  The ranges of a submit are shuffled, so resumed, fresh and finishing
    pieces sit next to each other in one warp."""
    rows: List[list] = [[] for _ in contents]
    for st in streams:
        for k, (s, off, n) in enumerate(st.pieces):
            rows[s].append((off, n, st.slot, R_MORE if k < st.more else 0))
    subs = []
    for (used, data, seed), r in zip(contents, rows):
        r = [r[i] for i in rng.permutation(len(r))]
        subs.append(Submit(used, ranges_array(r), data, seed))
    expect, n_streams = reference(subs)
    return Case(name, arena_bytes, max_extents, subs, streams, expect, n_streams)


# ---------------------------------------------------------------------------------------------------------------
# generators
# ---------------------------------------------------------------------------------------------------------------
RAGGED_N = 1 << 18
RAGGED_ARENA = 256 << 20
RAGGED_BLOCKS = (0, 1, 2, 3, 17)        # full blocks before the tail
RAGGED_LONG = 64                        # ranges of 1-8 MiB


def ragged_many(name: str = "ragged_many") -> Case:
    """2^18 one-shot ranges in one submit: every length residue mod 64 with 0, 1, 2, 3 and 17 full blocks (0 bytes
    included), every 16-byte offset class mod 64, 64 ranges of 1-8 MiB spread through the list; ranges share bytes."""
    rng = rng_for(name)
    data = np.frombuffer(rng.bytes(RAGGED_ARENA), dtype=np.uint8)
    combos = [(64 * b + r, c) for b in RAGGED_BLOCKS for r in range(64) for c in (0, 16, 32, 48)]
    n_short = RAGGED_N - RAGGED_LONG
    pick = np.concatenate([rng.permutation(len(combos)) for _ in range(-(-n_short // len(combos)))])[:n_short]
    lens = np.array([combos[i][0] for i in pick], dtype=np.int64)
    cls = np.array([combos[i][1] for i in pick], dtype=np.int64)
    offs = 64 * rng.integers(0, (RAGGED_ARENA - 64 * 18) // 64, n_short) + cls
    long_lens = rng.integers(1 << 20, (8 << 20) + 1, RAGGED_LONG)
    long_offs = 16 * rng.integers(0, (RAGGED_ARENA - (8 << 20)) // 16, RAGGED_LONG)
    at = np.sort(rng.choice(RAGGED_N, RAGGED_LONG, replace=False))
    is_long = np.zeros(RAGGED_N, dtype=bool)
    is_long[at] = True
    all_lens, all_offs = np.empty(RAGGED_N, np.int64), np.empty(RAGGED_N, np.int64)
    all_lens[is_long], all_offs[is_long] = long_lens, long_offs
    all_lens[~is_long], all_offs[~is_long] = lens, offs
    slots = rng.permutation(RAGGED_N)
    streams = [Stream(int(s), [(0, int(o), int(n))]) for o, n, s in zip(all_offs, all_lens, slots)]
    rows = [(int(o), int(n), int(s), 0) for o, n, s in zip(all_offs, all_lens, slots)]   # list order = fetch order
    sub = Submit(RAGGED_ARENA, ranges_array(rows), data)
    expect, n_streams = reference([sub])
    return Case(name, RAGGED_ARENA, RAGGED_N, [sub], streams, expect, n_streams)


MIX_SUBMITS = 4
MIX_ARENA = 16 << 20
MIX_MAX_STREAMS = 8192
MIX_MORE_K = (1, 2, 7, "large")         # MORE pieces are 64 * k bytes; large: 1000-4000 blocks
MIX_FINAL_BLOCKS = (0, 1, 5)            # full blocks of a tail-class final piece
MIX_FRESH_PER_SUBMIT = 96
MIX_RANDOM = 3000
MIX_REUSE = 0.15                        # chance that a stream starting after submit 0 takes a slot that finished


def _more_len(rng, k) -> int:
    return 64 * (int(rng.integers(1000, 4001)) if k == "large" else k)


def continued_mix(name: str = "continued_mix") -> Case:
    """About 4 000 streams over 4 submits, each in 1-4 pieces: every final length mod 64 with 0, 1 and 5 full blocks
    after 0, 1, 2 and 3 MORE pieces (finals of 0 bytes among them), MORE pieces of 64, 128, 448 and 64-256 KiB bytes,
    fresh one-shot streams in every submit, slots scattered up to max_streams - 1, slots reused after their stream
    finished."""
    rng = rng_for(name)
    specs = []                                          # (submits, piece lengths)

    def add(more: int, final: int, first: Optional[int] = None):
        lo = 0 if first is None else first
        hi = MIX_SUBMITS - more - 1 if first is None else first
        s0 = int(rng.integers(lo, hi + 1))
        subs = sorted([s0] + list(rng.choice(np.arange(s0 + 1, MIX_SUBMITS), more, replace=False)))
        lens = [_more_len(rng, MIX_MORE_K[int(rng.integers(len(MIX_MORE_K)))]) for _ in range(more)] + [final]
        specs.append((subs, lens))

    for more in range(4):
        for r in range(64):
            for b in MIX_FINAL_BLOCKS:
                add(more, 64 * b + r)
    for s in range(MIX_SUBMITS):
        for _ in range(MIX_FRESH_PER_SUBMIT):
            add(0, int(rng.integers(0, 2000)), first=s)
    for _ in range(MIX_RANDOM):
        add(int(rng.integers(0, 4)), int(rng.integers(0, 64 * 40)))
    # slots: the last slot first, then scattered; a stream that starts after submit 0 may take a finished slot
    pool = [MIX_MAX_STREAMS - 1] + [int(x) for x in rng.permutation(MIX_MAX_STREAMS - 1)]
    order = sorted(range(len(specs)), key=lambda i: (specs[i][0][0], float(rng.random())))
    ended: List[Tuple[int, int]] = []                   # (last submit, slot) of streams whose slot is free again
    streams = []
    for i in order:
        subs, lens = specs[i]
        free = [j for j, (end, _) in enumerate(ended) if end < subs[0]]
        if free and rng.random() < MIX_REUSE:
            slot = ended.pop(free[int(rng.integers(len(free)))])[1]
        else:
            slot = pool.pop(0)
        pieces = [(s, 16 * int(rng.integers(0, (MIX_ARENA - n) // 16 + 1)), n) for s, n in zip(subs, lens)]
        streams.append(Stream(slot, pieces))
        ended.append((subs[-1], slot))
    contents = [(MIX_ARENA, np.frombuffer(rng.bytes(MIX_ARENA), dtype=np.uint8), None) for _ in range(MIX_SUBMITS)]
    return _case(name, MIX_ARENA, MIX_MAX_STREAMS, contents, streams, rng)


LONG_ONE = (1 << 29) + 57               # one piece: 8 * len >= 2^32
LONG_PIECE = 200 << 20                  # three MORE pieces: 600 MiB
LONG_ARENA = (1 << 29) + 4096


def long_streams(name: str = "long_streams") -> Case:
    """Bit lengths of 2^32 and more: one piece of 2^29 + 57 bytes; two streams of 3 x 200 MiB MORE pieces, one ending in
    a final of 0 bytes, the other in a 56-byte final (the length then takes an extra block).  Synthetic content."""
    rng = rng_for(name)
    contents = [((1 << 29) + 64, None, 0x51A0), (LONG_PIECE + 64, None, 0x51A1), (LONG_PIECE + 64, None, 0x51A2),
                (4096, None, 0x51A3)]
    streams = [Stream(3, [(0, 0, LONG_ONE)]),
               Stream(0, [(0, 0, LONG_PIECE), (1, 0, LONG_PIECE), (2, 0, LONG_PIECE), (3, 0, 0)]),
               Stream(7, [(0, 16, LONG_PIECE), (1, 48, LONG_PIECE), (2, 32, LONG_PIECE), (3, 32, 56)])]
    return _case(name, LONG_ARENA, 64, contents, streams, rng)


STREAM_CASES = {"ragged_many": ragged_many, "continued_mix": continued_mix, "long_streams": long_streams}
MULTI_SUBMIT = ("continued_mix", "long_streams")


@lru_cache(maxsize=None)
def case(name: str) -> Case:
    return STREAM_CASES[name](name)


# ---------------------------------------------------------------------------------------------------------------
# K2: chunks longer than 2^29 bytes (the high length word of the chunk SHA-256)
# ---------------------------------------------------------------------------------------------------------------
LONG_CHUNK_MIN = (1 << 29) + 256        # min = normal = max: a file of at most min bytes is one chunk (rem <= min)
LONG_CHUNK_LENS = tuple((1 << 29) + d for d in (-1, 0, 1, 55, 56, 63, 64))


@dataclass
class ChunkCase:
    name: str
    params: Tuple[int, int, int, int, int]  # mksnap_cdc_params
    arena: np.ndarray
    files: List[Tuple[int, int]]            # CDC extents (arena_off, len), in submit order
    want: dict                              # ends, digests, table, n_chunks, n_unique, root


@lru_cache(maxsize=None)
def long_chunks(name: str = "long_chunks") -> ChunkCase:
    """Files of 2^29 - 1, 2^29, 2^29 + 1, + 55, + 56, + 63 and + 64 bytes, each one chunk; they start 16 bytes apart in
    one arena of random bytes (so they share bytes and every start has its own alignment)."""
    rng = rng_for(name)
    files = [(16 * i, n) for i, n in enumerate(LONG_CHUNK_LENS)]
    size = -(-max(o + n for o, n in files) // 512) * 512
    arena = np.frombuffer(rng.bytes(size), dtype=np.uint8)
    mv = memoryview(arena)
    digests = np.frombuffer(b"".join(hashlib.sha256(mv[o:o + n]).digest() for o, n in files),
                            dtype=np.uint8).reshape(-1, 32)
    table = tc.table_ref(digests)
    want = dict(ends=np.array([o + n for o, n in files], dtype=np.uint64), digests=digests, table=table,
                n_chunks=len(files), n_unique=len(table), root=tc.merkle_ref(table))
    p = (LONG_CHUNK_MIN, LONG_CHUNK_MIN, LONG_CHUNK_MIN, 16, 12)
    return ChunkCase(name, p, arena, files, want)


# ---------------------------------------------------------------------------------------------------------------
# the stream contract: one table for the engine and the CPU mock
# ---------------------------------------------------------------------------------------------------------------
CONTRACT_MAX = 64                       # max_extents (= max_streams) of the contract handle
CONTRACT_ARENA = 4096


@dataclass
class Outcome:
    name: str
    submits: List[Submit]               # all but the last succeed; the last too when `at` is "finish"
    at: str                             # "submit" or "finish": the call that returns `code`
    code: int                           # 0: accepted; the streams then match `expect`
    then: Case                          # a valid session on the same handle afterwards
    same_session: bool = False          # `then` continues the refused session instead of beginning a new one
    expect: Dict[int, bytes] = field(default_factory=dict)
    n_streams: int = 0


def _small(rng) -> np.ndarray:
    return np.frombuffer(rng.bytes(CONTRACT_ARENA), dtype=np.uint8)


def _one_submit(name, data, rows) -> Case:
    sub = Submit(CONTRACT_ARENA, ranges_array(rows), data)
    expect, n = reference([sub])
    return Case(name, CONTRACT_ARENA, CONTRACT_MAX, [sub], [], expect, n)


@lru_cache(maxsize=None)
def contract() -> List[Outcome]:
    rng = rng_for("contract")
    M = CONTRACT_MAX
    out = []

    def valid(tag, slot=5):
        d = _small(rng)
        return _one_submit(f"{tag}-then", d, [(0, 1000, slot, 0), (1024, 64, M - 1, 0)])

    def refused(tag, rows, code):
        out.append(Outcome(tag, [Submit(CONTRACT_ARENA, ranges_array(rows), _small(rng))], "submit", code, valid(tag)))

    last = _one_submit("last-slot", _small(rng), [(16, 777, M - 1, 0)])
    out.append(Outcome("last-slot-accepted", last.submits, "finish", 0, valid("last-slot"), expect=last.expect,
                       n_streams=last.n_streams))
    refused("slot-past-the-end", [(0, 100, M, 0)], E_CAPACITY)
    refused("two-pieces-one-slot", [(0, 64, 3, R_MORE), (64, 100, 3, 0)], E_INVAL)
    refused("two-finals-one-slot", [(0, 10, 3, 0), (64, 10, 3, 0)], E_INVAL)
    refused("more-piece-of-0-bytes", [(0, 0, 3, R_MORE)], E_INVAL)
    refused("more-piece-of-100-bytes", [(0, 100, 3, R_MORE)], E_INVAL)
    refused("unaligned-range", [(8, 64, 3, 0)], E_INVAL)
    refused("range-past-used", [(CONTRACT_ARENA - 48, 64, 3, 0)], E_INVAL)
    # finish with a stream left open; begin resets the midstate, so the same slot then digests only its own bytes
    open_sub = Submit(CONTRACT_ARENA, ranges_array([(0, 128, 5, R_MORE), (256, 10, 9, 0)]), _small(rng))
    out.append(Outcome("finish-with-an-open-stream", [open_sub], "finish", E_STATE, valid("finish-open", slot=5)))
    # the refusal leaves the session open: the final piece still completes the stream
    final = Submit(CONTRACT_ARENA, ranges_array([(512, 33, 5, 0)]), _small(rng))
    expect, n = reference([open_sub, final])
    out.append(Outcome("finish-refused-then-final-piece", [open_sub], "finish", E_STATE,
                       Case("final-piece", CONTRACT_ARENA, M, [final], [], expect, n), same_session=True))
    return out


# ---------------------------------------------------------------------------------------------------------------
# running a case on an engine (the device engine or the CPU mock, behind one small driver interface)
# ---------------------------------------------------------------------------------------------------------------
class Driver:
    """begin(); submit(Submit); finish() -> n_streams; stream_digests(n) -> (n, 32) uint8.  Errors raise an exception
    with a `code` attribute (MKSNAP_E_*)."""


def check_streams(name, n_streams, rows, expect, want_n):
    assert n_streams == want_n, f"{name}: n_streams {n_streams}, want {want_n}"
    bad = [s for s, d in expect.items() if rows[s].tobytes() != d]
    assert not bad, f"{name}: {len(bad)} of {len(expect)} finished slots differ, first {sorted(bad)[:8]}"


def run_case(drv, c: Case, begin: bool = True):
    if begin:
        drv.begin()
    for s in c.submits:
        drv.submit(s)
    n = drv.finish()
    check_streams(c.name, n, drv.stream_digests(n), c.expect, c.n_streams)


def _expect_code(fn, code, what):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 -- MksnapError of either engine
        got = getattr(e, "code", None)
        assert got == code, f"{what}: code {got}, want {code} ({e})"
        return
    raise AssertionError(f"{what}: accepted, want code {code}")


def run_outcome(drv, o: Outcome):
    drv.begin()
    for i, s in enumerate(o.submits):
        if o.at == "submit" and i == len(o.submits) - 1:
            _expect_code(lambda: drv.submit(s), o.code, f"{o.name}: submit")
        else:
            drv.submit(s)
    if o.at == "finish":
        if o.code == 0:
            n = drv.finish()
            check_streams(o.name, n, drv.stream_digests(n), o.expect, o.n_streams)
        else:
            _expect_code(drv.finish, o.code, f"{o.name}: finish")
    run_case(drv, o.then, begin=not o.same_session)
