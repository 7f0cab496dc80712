"""CPU: the serial-stream cases of tests/stream_cases.py check what they claim, and the CPU mock engine
(tests/mock_engine/mock_mksnap.cpp) runs continued_mix, long_streams and the contract table, so that the mock and the
device engine (tests/test_gpu_stream_sha.py) are held to one table."""
import ctypes as C
import functools
import hashlib

import numpy as np
import pytest

from tests import mock_engine
from tests import stream_cases as sc


# ---------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------
def test_synth_matches_the_oracle_generator(oracle_lib):
    """The case module restates mksnap_synth_fill's generator; the oracle's C copy must agree (offsets included)."""
    for off, n, seed in ((0, 4096, 99), (4096, 1 << 16, 0x51A0), (8 << 20, 4096, 0xC2)):
        np.testing.assert_array_equal(sc.synth(off, n, seed), oracle_lib.synth_fill(off, n, seed))


def test_reference_is_hashlib_over_the_pieces():
    rng = np.random.default_rng(1)
    a, b = (np.frombuffer(rng.bytes(4096), dtype=np.uint8) for _ in range(2))
    subs = [sc.Submit(4096, sc.ranges_array([(0, 128, 2, sc.R_MORE), (16, 5, 0, 0)]), a),
            sc.Submit(4096, sc.ranges_array([(64, 64, 2, sc.R_MORE)]), b),
            sc.Submit(4096, sc.ranges_array([(0, 0, 2, 0)]), a)]
    exp, n = sc.reference(subs)
    assert n == 3 and set(exp) == {0, 2}
    assert exp[2] == hashlib.sha256(a[:128].tobytes() + b[64:128].tobytes()).digest()
    assert exp[0] == hashlib.sha256(a[16:21].tobytes()).digest()
    with pytest.raises(AssertionError):         # left open
        sc.reference(subs[:2])


# ---------------------------------------------------------------------------------------------------------------
# the generators' claims
# ---------------------------------------------------------------------------------------------------------------
def _final_len(st):
    return st.pieces[-1][2]


def test_ragged_many_claims():
    c = sc.case("ragged_many")
    assert len(c.submits) == 1 and c.max_extents == sc.RAGGED_N
    r = c.submits[0].ranges
    assert r.size == sc.RAGGED_N and c.submits[0].used == sc.RAGGED_ARENA
    assert not (r["flags"] & sc.R_MORE).any() and np.unique(r["stream"]).size == r.size
    lens, offs = r["len"].astype(np.int64), r["arena_off"].astype(np.int64)
    short = lens < (1 << 20)
    classes = set(zip((lens[short] // 64).tolist(), (lens[short] % 64).tolist(), (offs[short] % 64).tolist()))
    assert classes == {(b, t, o) for b in sc.RAGGED_BLOCKS for t in range(64) for o in (0, 16, 32, 48)}
    assert (lens == 0).sum() >= 100
    long_at = np.flatnonzero(~short)
    assert long_at.size == sc.RAGGED_LONG and (lens[long_at] <= 8 << 20).all()
    assert long_at[0] < sc.RAGGED_N // 8 and long_at[-1] > sc.RAGGED_N * 7 // 8
    # ranges share bytes
    o = np.argsort(offs)
    assert (offs[o][1:] < (offs + lens)[o][:-1]).any()
    # every lane takes on average at least 10 pieces on an H100 (132 SMs)
    lanes = min(-(-r.size // 32), sc.K4_PAIRS_PER_SM * sc.H100_SMS) * 32
    assert r.size / lanes >= 10
    assert c.n_streams == sc.RAGGED_N and len(c.expect) == sc.RAGGED_N


def test_continued_mix_claims():
    c = sc.case("continued_mix")
    S = sc.MIX_SUBMITS
    assert len(c.submits) == S and 3500 <= len(c.streams) <= 5000
    # tail classes: every final length mod 64 with 0, 1 and several full blocks after 0, 1, 2 and 3 MORE pieces
    seen = {(st.more, _final_len(st) % 64, min(_final_len(st) // 64, 2)) for st in c.streams}
    assert seen >= {(m, r, b) for m in range(4) for r in range(64) for b in range(3)}
    assert {st.more for st in c.streams if _final_len(st) == 0} >= {1, 2, 3}
    # piece rules
    ks = set()
    for st in c.streams:
        subs = [s for s, _, _ in st.pieces]
        assert subs == sorted(set(subs)) and 1 <= len(subs) <= 4
        for _, _, n in st.pieces[:-1]:
            assert n > 0 and n % 64 == 0
            ks.add(n // 64 if n // 64 in (1, 2, 7) else "large")
    assert ks == {1, 2, 7, "large"}
    assert max(st.pieces[0][2] for st in c.streams if st.more) >= 64 * 1000
    for s in c.submits:
        assert np.unique(s.ranges["stream"]).size == s.ranges.size
    # fresh one-shot streams in every submit, next to resumed ones from submit 1 on
    for k in range(S):
        fresh = [st for st in c.streams if st.more == 0 and st.pieces[0][0] == k]
        resumed = [st for st in c.streams if any(s == k for s, _, _ in st.pieces[1:])]
        assert len(fresh) >= sc.MIX_FRESH_PER_SUBMIT and (k == 0 or len(resumed) >= 100)
    # a stream whose pieces skip a submit
    assert any(np.diff([s for s, _, _ in st.pieces]).max(initial=1) > 1 for st in c.streams)
    # slots scattered up to max_streams - 1; slots reused after their stream finished (some in submit 0)
    slots = [st.slot for st in c.streams]
    assert max(slots) == c.max_extents - 1 and c.n_streams == c.max_extents
    by_slot = {}
    for st in c.streams:
        by_slot.setdefault(st.slot, []).append(st)
    reused = [v for v in by_slot.values() if len(v) > 1]
    assert len(reused) >= 100
    assert sum(1 for v in reused if v[0].pieces[-1][0] == 0) >= 20
    for v in reused:
        for a, b in zip(v, v[1:]):
            assert a.pieces[-1][0] < b.pieces[0][0]
    # the expected row of a reused slot is its LAST stream's digest
    assert set(c.expect) == set(by_slot)


def test_long_streams_claims():
    c = sc.case("long_streams")
    totals = {st.slot: st.total for st in c.streams}
    assert all(8 * t >= 1 << 32 for t in totals.values())
    assert (1 << 29) < min(totals.values()) and max(totals.values()) >= 600 << 20
    finals = sorted(_final_len(st) for st in c.streams if st.more)
    assert finals == [0, 56]
    assert any(st.more == 0 and st.total == (1 << 29) + 57 for st in c.streams)
    assert all(s.seed is not None and s.used % 16 == 0 and s.used <= c.arena_bytes for s in c.submits)


def test_long_chunks_claims():
    lc = sc.long_chunks()
    mn, nm, mx = lc.params[:3]
    assert mn == nm == mx
    assert sorted(n for _, n in lc.files) == sorted((1 << 29) + d for d in (-1, 0, 1, 55, 56, 63, 64))
    from tests import cdc_cases as cc
    p = cc.Params(*lc.params)
    none = cc.Cands(np.zeros(0, np.int64), np.zeros(0, np.int64))
    for (off, n), end in zip(lc.files, lc.want["ends"]):
        assert n <= mn and cc.file_cuts(off, n, none, p) == [off + n] == [int(end)]
        assert off % 16 == 0
    assert lc.want["n_unique"] == len(lc.files)


def test_contract_table_shape():
    t = sc.contract()
    names = [o.name for o in t]
    assert len(set(names)) == len(names)
    codes = {o.name: o.code for o in t}
    assert codes["last-slot-accepted"] == 0 and codes["slot-past-the-end"] == sc.E_CAPACITY
    assert codes["finish-with-an-open-stream"] == sc.E_STATE
    assert sum(1 for v in codes.values() if v == sc.E_INVAL) >= 6


@pytest.mark.parametrize("name", list(sc.STREAM_CASES) + ["long_chunks", "contract"])
def test_generators_are_deterministic(name):
    gen = {"long_chunks": sc.long_chunks.__wrapped__, "contract": sc.contract.__wrapped__}.get(name)
    if gen is None:
        a, b = sc.STREAM_CASES[name](name), sc.case(name)
        assert a.expect == b.expect and a.n_streams == b.n_streams
        for x, y in zip(a.submits, b.submits):
            np.testing.assert_array_equal(x.ranges, y.ranges)
            assert x.seed == y.seed and (x.data is None or np.array_equal(x.data, y.data))
    elif name == "long_chunks":
        a, b = gen(), sc.long_chunks()
        assert a.files == b.files and a.want["root"] == b.want["root"] and np.array_equal(a.arena, b.arena)
    else:
        a, b = gen(), sc.contract()
        assert [(o.name, o.code, o.then.expect) for o in a] == [(o.name, o.code, o.then.expect) for o in b]


# ---------------------------------------------------------------------------------------------------------------
# the CPU mock engine on the same cases
# ---------------------------------------------------------------------------------------------------------------
@functools.cache
def _lib():
    """The mock loaded into this process (RTLD_LOCAL: nothing else binds to it)."""
    lib = C.CDLL(mock_engine.build())
    P, U64 = C.c_void_p, C.c_uint64
    for name, res, args in (("mksnap_create", C.c_int, [P, C.POINTER(P)]), ("mksnap_destroy", None, [P]),
                            ("mksnap_last_error", C.c_char_p, [P]), ("mksnap_begin", C.c_int, [P]),
                            ("mksnap_arena_acquire", C.c_int, [P, C.POINTER(P), C.POINTER(U64), C.POINTER(C.c_int32)]),
                            ("mksnap_arena_submit", C.c_int, [P, C.c_int32, U64, P, U64, P, U64]),
                            ("mksnap_finish", C.c_int, [P, P]), ("mksnap_reserve_stream_log", C.c_int, [P, U64]),
                            ("mksnap_get_stream_digests", C.c_int, [P, P, U64]), ("mock_log_flushes", U64, [P])):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


class MockDriver:
    """stream_cases' driver interface over the CPU mock: pinned-arena style submits (acquire, copy, submit)."""

    def __init__(self, arena_bytes: int, max_extents: int):
        from makisu_b200.abi import Config
        self.lib, self.h = _lib(), C.c_void_p()
        cfg = Config()
        cfg.n_host_arenas, cfg.host_arena_bytes, cfg.max_extents = 2, arena_bytes, max_extents
        assert self.lib.mksnap_create(C.byref(cfg), C.byref(self.h)) == 0

    def close(self):
        self.lib.mksnap_destroy(self.h)

    def _ck(self, rc, where):
        if rc:
            from makisu_b200.abi import MksnapError
            raise MksnapError(rc, where, (self.lib.mksnap_last_error(self.h) or b"").decode())

    def begin(self):
        self._ck(self.lib.mksnap_begin(self.h), "mksnap_begin")

    def submit(self, s: sc.Submit):
        ptr, cap, aid = C.c_void_p(), C.c_uint64(), C.c_int32()
        self._ck(self.lib.mksnap_arena_acquire(self.h, C.byref(ptr), C.byref(cap), C.byref(aid)), "mksnap_arena_acquire")
        a = np.ascontiguousarray(s.arena())
        C.memmove(ptr, a.ctypes.data, s.used)
        r = np.ascontiguousarray(s.ranges)
        self._ck(self.lib.mksnap_arena_submit(self.h, aid.value, s.used, None, 0, r.ctypes.data if r.size else None,
                                              r.size), "mksnap_arena_submit")

    def finish(self) -> int:
        from makisu_b200.abi import Result
        res = Result()
        self._ck(self.lib.mksnap_finish(self.h, C.byref(res)), "mksnap_finish")
        return res.n_streams

    def stream_digests(self, n: int) -> np.ndarray:
        t = np.empty((max(n, 1), 32), dtype=np.uint8)
        self._ck(self.lib.mksnap_get_stream_digests(self.h, t.ctypes.data, n), "mksnap_get_stream_digests")
        return t[:n]


@pytest.mark.parametrize("name", sc.MULTI_SUBMIT)
def test_mock_engine_runs_the_stream_cases(name):
    c = sc.case(name)
    d = MockDriver(c.arena_bytes, c.max_extents)
    try:
        sc.run_case(d, c)
    finally:
        d.close()


@pytest.mark.parametrize("outcome", sc.contract(), ids=lambda o: o.name)
def test_mock_engine_keeps_the_stream_contract(outcome):
    d = MockDriver(sc.CONTRACT_ARENA, sc.CONTRACT_MAX)
    try:
        sc.run_outcome(d, outcome)
    finally:
        d.close()
