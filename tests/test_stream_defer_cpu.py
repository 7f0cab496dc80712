"""CPU: deferred serial streams (MKSNAP_R_DEFER) on the CPU mock engine (tests/mock_engine/mock_mksnap_defer.cpp): the
cases and contract of tests/defer_cases.py, the same table the device engine runs in tests/test_gpu_stream_defer.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import defer_cases as dc
from tests import stream_cases as sc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def build_mock(out) -> str:
    obj, so = str(out / "mkoracle.o"), str(out / "libmock_defer.so")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "oracle", "mkoracle.c"), "-o", obj])
    # -Bsymbolic: the mock's own calls bind inside it even when libmksnap or the oracle is loaded globally
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wl,-Bsymbolic",
                           os.path.join(HERE, "mock_engine", "mock_mksnap_defer.cpp"), obj, "-o", so])
    return so


@pytest.fixture(scope="module")
def mock_lib(tmp_path_factory):
    lib = C.CDLL(build_mock(tmp_path_factory.mktemp("mock_defer")))
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
    """stream_cases' driver interface over the mock, plus reserve_stream_log."""

    def __init__(self, lib, arena_bytes: int, max_extents: int):
        from makisu_b200.abi import Config
        self.lib, self.h = lib, C.c_void_p()
        cfg = Config()
        cfg.n_host_arenas, cfg.host_arena_bytes, cfg.max_extents = 2, arena_bytes, max_extents
        assert lib.mksnap_create(C.byref(cfg), C.byref(self.h)) == 0

    def close(self):
        self.lib.mksnap_destroy(self.h)

    def _ck(self, rc, where):
        if rc:
            from makisu_b200.abi import MksnapError
            raise MksnapError(rc, where, (self.lib.mksnap_last_error(self.h) or b"").decode())

    def reserve_stream_log(self, n: int):
        self._ck(self.lib.mksnap_reserve_stream_log(self.h, n), "mksnap_reserve_stream_log")

    def flushes(self) -> int:
        return int(self.lib.mock_log_flushes(self.h))

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


@pytest.mark.parametrize("name", list(dc.CASES))
def test_mock_runs_the_defer_cases(mock_lib, name):
    c = dc.case(name)
    d = MockDriver(mock_lib, c.case.arena_bytes, c.case.max_extents)
    try:
        dc.run(d, c)
        if name == "small_log":
            assert d.flushes() >= 4      # pieces that did not fit forced flushes before finish
    finally:
        d.close()


@pytest.mark.parametrize("outcome", dc.contract(), ids=lambda o: o.name)
def test_mock_keeps_the_defer_contract(mock_lib, outcome):
    d = MockDriver(mock_lib, sc.CONTRACT_ARENA, sc.CONTRACT_MAX)
    try:
        d.reserve_stream_log(dc.CONTRACT_LOG)
        sc.run_outcome(d, outcome)
    finally:
        d.close()


def test_mock_refuses_a_resize_while_pieces_wait(mock_lib):
    d = MockDriver(mock_lib, sc.CONTRACT_ARENA, sc.CONTRACT_MAX)
    try:
        d.reserve_stream_log(dc.CONTRACT_LOG)
        d.begin()
        d.reserve_stream_log(1 << 12)                   # nothing waits yet
        d.submit(dc._sub(sc.rng_for("resize"), [(0, 100, 1, dc.R_DEFER)]))
        with pytest.raises(Exception) as ei:
            d.reserve_stream_log(0)
        assert ei.value.code == sc.E_STATE
        d.finish()
        d.reserve_stream_log(0)
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------------------------
# the cases check what they claim
# ---------------------------------------------------------------------------------------------------------------
def _log_pieces(c: dc.DeferCase):
    return [(s, r) for s, sub in enumerate(c.case.submits) for r in sub.ranges.tolist() if r[3] & dc.R_DEFER]


def test_tails_cover_every_final_tail():
    for k in range(1, 5):
        c = dc.case("tails_%d_submits" % k).case
        finals = {(len(st.pieces), st.pieces[-1][2] % 64, st.pieces[-1][2] // 64) for st in c.streams}
        assert finals == {(k, r, b) for r in range(64) for b in (0, 1)}
        assert all(r[3] & dc.R_DEFER for s in c.submits for r in s.ranges.tolist())
    assert any(st.pieces[-1][2] == 0 for st in dc.case("tails_4_submits").case.streams)


def test_mixed_session_and_slot_reuse_claims():
    c = dc.case("mixed_session").case
    kinds = {bool(r[3] & dc.R_DEFER) for s in c.submits for r in s.ranges.tolist()}
    assert kinds == {True, False}
    by_slot = {}
    for st in c.streams:
        by_slot.setdefault(st.slot, []).append(st)
    assert sum(1 for v in by_slot.values() if len(v) > 1) >= 5
    r = dc.case("slot_reuse")
    assert {st.slot for st in r.case.streams} == {3, 4, 5, 6} and len(r.case.streams) == 6


def test_small_and_large_pieces_against_the_log():
    small = dc.case("small_log")
    assert sum(r[1] for _, r in _log_pieces(small)) > 4 * small.log_bytes
    big = dc.case("larger_than_log")
    lens = [r[1] for _, r in _log_pieces(big)]
    assert any(n > big.log_bytes for n in lens) and any(n <= big.log_bytes for n in lens)
    assert any(n == big.log_bytes for n in lens)


def test_layers_in_order_leave_each_stream_contiguous():
    c = dc.case("layers_in_order")
    order = [r[2] for _, r in _log_pieces(c)]
    assert order == sorted(order) and len(set(order)) == 6
