"""Deferred serial streams (MKSNAP_R_DEFER, the engine's stream log) in the shape of tests/stream_cases.py: one table that
the CPU mock (tests/test_stream_defer_cpu.py) and the device engine (tests/test_gpu_stream_defer.py) both run.  The
reference is stream_cases.reference, hashlib over each stream's pieces: deferring a stream changes when it is hashed,
never its digest.

A case is a stream_cases.Case plus the size of the stream log reserved before the session.  Cases:
- tails_<k>_submits: deferred streams over k = 1-4 submits with every final length mod 64 (after 0 and 1 full blocks),
  finals of 0 bytes, pieces of one submit interleaved in the log (one flush round per piece);
- layers_in_order: streams whose pieces follow one another in the log, the way layers applied in order leave them (one
  merged range per stream);
- mixed_session: deferred and inline streams side by side in every submit, slots of both kinds reused;
- small_log: a log a few pieces long, so that pieces that do not fit force flushes mid-session, across MORE pieces;
- larger_than_log: pieces larger than the whole log (hashed in their own submit) between pieces the log takes;
- slot_reuse: a slot whose deferred stream waits in the log carries an inline stream next, another carries a second
  deferred stream (two rounds of one flush), and an empty deferred stream."""
from __future__ import annotations

from dataclasses import dataclass
from functools import lru_cache
from typing import List

import numpy as np

from tests import stream_cases as sc

R_MORE, R_DEFER = sc.R_MORE, 2
ARENA = 64 << 10
MAX_STREAMS = 1024


@dataclass
class DeferCase:
    case: sc.Case
    log_bytes: int


def _build(name, n_submits, streams, log_bytes, inline=(), arena=ARENA) -> DeferCase:
    """streams: stream_cases.Stream list; every stream is deferred unless its index is in `inline`.  The ranges of a
    submit keep list order (= log order)."""
    rng = sc.rng_for(name)
    rows: List[list] = [[] for _ in range(n_submits)]
    for j, st in enumerate(streams):
        d = 0 if j in inline else R_DEFER
        for k, (s, off, n) in enumerate(st.pieces):
            rows[s].append((off, n, st.slot, (R_MORE if k < st.more else 0) | d))
    subs = [sc.Submit(arena, sc.ranges_array(r), np.frombuffer(rng.bytes(arena), dtype=np.uint8)) for r in rows]
    expect, n_streams = sc.reference(subs)
    return DeferCase(sc.Case(name, arena, MAX_STREAMS, subs, streams, expect, n_streams), log_bytes)


def _off(rng, n, arena=ARENA) -> int:
    return 16 * int(rng.integers(0, (arena - n) // 16 + 1))


def tails(k: int) -> DeferCase:
    """Every final tail after k - 1 MORE pieces: 64 residues x (0, 1 full blocks), each stream over submits 0 .. k-1."""
    name = "tails_%d_submits" % k
    rng = sc.rng_for(name)
    streams = []
    for b in (0, 1):
        for r in range(64):
            lens = [64 * int(rng.integers(1, 9)) for _ in range(k - 1)] + [64 * b + r]
            streams.append(sc.Stream(len(streams), [(s, _off(rng, n), n) for s, n in enumerate(lens)]))
    return _build(name, k, streams, 1 << 20)


def layers_in_order() -> DeferCase:
    """Six streams, each in 1-4 consecutive submits, one after another (stream i's pieces precede stream i+1's)."""
    name = "layers_in_order"
    rng = sc.rng_for(name)
    streams, s = [], 0
    for i in range(6):
        k = 1 + i % 4
        lens = [64 * int(rng.integers(16, 200)) for _ in range(k - 1)] + [int(rng.integers(0, 3000))]
        streams.append(sc.Stream(i, [(s + j, _off(rng, n), n) for j, n in enumerate(lens)]))
        s += k - 1   # the next stream starts in the submit where this one ends
    return _build(name, s + 1, streams, 1 << 20)


def mixed_session() -> DeferCase:
    """Four submits; in each, fresh deferred and inline streams, continued streams of both kinds, slots reused by the
    other kind after their stream finished."""
    name = "mixed_session"
    rng = sc.rng_for(name)
    streams, inline, free, nxt = [], set(), [], 0
    for s0 in range(4):
        for _ in range(40):
            more = int(rng.integers(0, 4 - s0))
            subs = sorted([s0] + list(rng.choice(np.arange(s0 + 1, 4), more, replace=False))) if more else [s0]
            lens = [64 * int(rng.integers(1, 20)) for _ in range(more)] + [int(rng.integers(0, 700))]
            ready = [f for f in free if f[0] < s0]
            if ready and rng.random() < 0.3:
                free.remove(ready[0])
                slot = ready[0][1]
            else:
                slot, nxt = nxt, nxt + 1
            if rng.random() < 0.5:
                inline.add(len(streams))
            streams.append(sc.Stream(slot, [(s, _off(rng, n), n) for s, n in zip(subs, lens)]))
            free.append((subs[-1], slot))
    return _build(name, 4, streams, 1 << 20, inline)


def small_log() -> DeferCase:
    """A 4 KiB log and 24 streams of 1-3 pieces of up to 1.5 KiB over 6 submits: the log fills every few pieces."""
    name = "small_log"
    rng = sc.rng_for(name)
    streams = []
    for i in range(24):
        more = int(rng.integers(0, 3))
        s0 = int(rng.integers(0, 6 - more))
        subs = sorted([s0] + list(rng.choice(np.arange(s0 + 1, 6), more, replace=False))) if more else [s0]
        lens = [64 * int(rng.integers(1, 24)) for _ in range(more)] + [int(rng.integers(0, 1500))]
        streams.append(sc.Stream(i, [(s, _off(rng, n), n) for s, n in zip(subs, lens)]))
    return _build(name, 6, streams, 4096)


def larger_than_log() -> DeferCase:
    """A 1 KiB log: streams whose pieces alternate between larger and smaller than the log, finals of both kinds."""
    name = "larger_than_log"
    rng = sc.rng_for(name)
    plans = [[4096, 256, 8192, 100], [512, 2048, 0], [64, 64, 64, 1500], [3000], [640, 128, 1024, 1025]]
    streams = []
    for i, lens in enumerate(plans):
        streams.append(sc.Stream(i, [(s, _off(rng, n), n) for s, n in enumerate(lens)]))
    return _build(name, 4, streams, 1024)


def slot_reuse() -> DeferCase:
    """Slot 3: a deferred stream finishes in submit 1 and waits in the log; an inline stream takes the slot in submit 3
    (the log is hashed first).  Slot 4: two deferred streams, both waiting in the log then (two rounds of that flush).
    Slot 5: an empty deferred stream; slot 6: a deferred stream ending in a final piece of 0 bytes."""
    name = "slot_reuse"
    rng = sc.rng_for(name)
    spec = [(3, [(0, 640), (1, 77)], False), (3, [(3, 999)], True), (4, [(0, 128), (1, 5)], False),
            (4, [(2, 192), (3, 64)], False), (5, [(1, 0)], False), (6, [(0, 64), (2, 0)], False)]
    streams, inline = [], set()
    for slot, pieces, inl in spec:
        if inl:
            inline.add(len(streams))
        streams.append(sc.Stream(slot, [(s, _off(rng, n), n) for s, n in pieces]))
    return _build(name, 4, streams, 1 << 16, inline)


CASES = {"tails_1_submits": lambda: tails(1), "tails_2_submits": lambda: tails(2), "tails_3_submits": lambda: tails(3),
         "tails_4_submits": lambda: tails(4), "layers_in_order": layers_in_order, "mixed_session": mixed_session,
         "small_log": small_log, "larger_than_log": larger_than_log, "slot_reuse": slot_reuse}


@lru_cache(maxsize=None)
def case(name: str) -> DeferCase:
    return CASES[name]()


# ---------------------------------------------------------------------------------------------------------------
# the contract of deferred streams (a 64 KiB log)
# ---------------------------------------------------------------------------------------------------------------
CONTRACT_LOG = 1 << 16


def _sub(rng, rows):
    return sc.Submit(sc.CONTRACT_ARENA, sc.ranges_array(rows), np.frombuffer(rng.bytes(sc.CONTRACT_ARENA), dtype=np.uint8))


@lru_cache(maxsize=None)
def contract() -> List[sc.Outcome]:
    rng = sc.rng_for("defer_contract")
    M, D = sc.CONTRACT_MAX, R_DEFER
    out = []

    def valid(tag):
        subs = [_sub(rng, [(0, 1000, 5, D), (1024, 64, M - 1, 0)])]
        expect, n = sc.reference(subs)
        return sc.Case(tag + "-then", sc.CONTRACT_ARENA, M, subs, [], expect, n)

    out.append(sc.Outcome("deferred-then-inline-piece", [_sub(rng, [(0, 128, 5, R_MORE | D)]), _sub(rng, [(0, 10, 5, 0)])],
                          "submit", sc.E_INVAL, valid("deferred-then-inline")))
    out.append(sc.Outcome("inline-then-deferred-piece", [_sub(rng, [(0, 128, 5, R_MORE)]), _sub(rng, [(0, 10, 5, D)])],
                          "submit", sc.E_INVAL, valid("inline-then-deferred")))
    out.append(sc.Outcome("deferred-more-piece-of-100-bytes", [_sub(rng, [(0, 100, 3, R_MORE | D)])], "submit", sc.E_INVAL,
                          valid("deferred-more-100")))
    open_sub = _sub(rng, [(0, 128, 5, R_MORE | D), (256, 10, 9, D), (512, 64, 7, R_MORE)])
    out.append(sc.Outcome("finish-with-an-open-deferred-stream", [open_sub], "finish", sc.E_STATE, valid("finish-open")))
    final = _sub(rng, [(512, 33, 5, D), (1024, 0, 7, 0)])
    expect, n = sc.reference([open_sub, final])
    out.append(sc.Outcome("finish-refused-then-final-deferred-piece", [open_sub], "finish", sc.E_STATE,
                          sc.Case("final-piece", sc.CONTRACT_ARENA, M, [final], [], expect, n), same_session=True))
    return out


def run(drv, dc: DeferCase):
    """drv: a stream_cases driver with reserve_stream_log(bytes)."""
    drv.reserve_stream_log(dc.log_bytes)
    sc.run_case(drv, dc.case)
