"""CPU: deferred serial streams (MKSNAP_R_DEFER) on the CPU mock engine (tests/mock_engine/mock_mksnap.cpp): the
cases and contract of tests/defer_cases.py, the same table the device engine runs in tests/test_gpu_stream_defer.py."""
import pytest

from tests import defer_cases as dc
from tests import stream_cases as sc
from tests.test_stream_reference_cpu import MockDriver as _StreamDriver


class MockDriver(_StreamDriver):
    """stream_cases' driver interface over the mock, plus reserve_stream_log."""

    def reserve_stream_log(self, n: int):
        self._ck(self.lib.mksnap_reserve_stream_log(self.h, n), "mksnap_reserve_stream_log")

    def flushes(self) -> int:
        return int(self.lib.mock_log_flushes(self.h))


@pytest.mark.parametrize("name", list(dc.CASES))
def test_mock_runs_the_defer_cases(name):
    c = dc.case(name)
    d = MockDriver(c.case.arena_bytes, c.case.max_extents)
    try:
        dc.run(d, c)
        if name == "small_log":
            assert d.flushes() >= 4      # pieces that did not fit forced flushes before finish
    finally:
        d.close()


@pytest.mark.parametrize("outcome", dc.contract(), ids=lambda o: o.name)
def test_mock_keeps_the_defer_contract(outcome):
    d = MockDriver(sc.CONTRACT_ARENA, sc.CONTRACT_MAX)
    try:
        d.reserve_stream_log(dc.CONTRACT_LOG)
        sc.run_outcome(d, outcome)
    finally:
        d.close()


def test_mock_refuses_a_resize_while_pieces_wait():
    d = MockDriver(sc.CONTRACT_ARENA, sc.CONTRACT_MAX)
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
