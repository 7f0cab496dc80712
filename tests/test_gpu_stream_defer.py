"""-m gpu: deferred serial streams (MKSNAP_R_DEFER) on the device: the cases and contract of tests/defer_cases.py (the
table the CPU mock keeps) against hashlib, through pinned host arenas and device-resident slots, and one deferred
stream past 2^32 bits whose pieces sit beyond 4 GiB in the stream log.

Only the rows of slots on which a stream finished in the session are compared; the others are unspecified."""
import ctypes
import hashlib

import numpy as np
import pytest

from tests import defer_cases as dc
from tests import stream_cases as sc

pytestmark = pytest.mark.gpu


class EngineDriver:
    def __init__(self, e, via_host: bool):
        self.e, self.via_host = e, via_host

    def reserve_stream_log(self, n: int):
        self.e.reserve_stream_log(n)

    def begin(self):
        self.e.begin()

    def submit(self, s: sc.Submit):
        from makisu_b200.abi import Range
        r = np.ascontiguousarray(s.ranges)
        ra = (Range * max(1, r.size)).from_buffer(r if r.size else np.zeros(1, sc.RANGE_DTYPE))
        if self.via_host:
            ptr, _, aid = self.e.arena_acquire()
            ctypes.memmove(ptr, np.ascontiguousarray(s.arena()).ctypes.data, s.used)
            self.e.arena_submit(aid, s.used, [], ra if r.size else [])
            return
        self.e.sync()                           # the previous submit has read slot 0
        self.e.device_upload(0, 0, s.arena())
        self.e.device_submit(0, s.used, [], ra if r.size else [])

    def finish(self) -> int:
        return self.e.finish().n_streams

    def stream_digests(self, n: int) -> np.ndarray:
        return self.e.get_stream_digests(n)


def _engine(arena_bytes, max_extents, via_host):
    from makisu_b200.abi import Engine
    kw = dict(n_host_arenas=2, host_arena_bytes=arena_bytes) if via_host else {}
    return Engine(device=0, device_arena_bytes=arena_bytes, max_extents=max_extents, **kw)


@pytest.mark.parametrize("via_host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("name", list(dc.CASES))
def test_defer_cases(name, via_host):
    c = dc.case(name)
    with _engine(c.case.arena_bytes, c.case.max_extents, via_host) as e:
        dc.run(EngineDriver(e, via_host), c)


@pytest.mark.parametrize("outcome", dc.contract(), ids=lambda o: o.name)
def test_defer_contract(outcome):
    with _engine(sc.CONTRACT_ARENA, sc.CONTRACT_MAX, False) as e:
        e.reserve_stream_log(dc.CONTRACT_LOG)
        sc.run_outcome(EngineDriver(e, False), outcome)


def test_resize_refused_while_pieces_wait():
    from makisu_b200.abi import MksnapError
    with _engine(sc.CONTRACT_ARENA, sc.CONTRACT_MAX, False) as e:
        d = EngineDriver(e, False)
        e.reserve_stream_log(dc.CONTRACT_LOG)
        e.begin()
        e.reserve_stream_log(1 << 12)            # nothing waits yet
        sub = dc._sub(sc.rng_for("resize"), [(0, 100, 1, dc.R_DEFER)])
        d.submit(sub)
        with pytest.raises(MksnapError) as ei:
            e.reserve_stream_log(0)
        assert ei.value.code == sc.E_STATE
        e.finish()
        assert e.get_stream_digests(2)[1].tobytes() == hashlib.sha256(sub.arena()[:100].tobytes()).digest()
        e.reserve_stream_log(0)


def test_flush_time_is_reported():
    c = dc.case("small_log")
    with _engine(c.case.arena_bytes, c.case.max_extents, True) as e:
        dc.run(EngineDriver(e, True), c)
        assert e.stats().ms_flush > 0


PAD_PIECE, PAD_STREAMS = 64 << 20, 64      # 4 GiB of other streams' pieces in the log first
LONG = (1 << 29) + 57                      # 8 * LONG >= 2^32


def test_deferred_stream_past_2_32_bits_beyond_4_gib_of_log():
    """64 one-piece deferred streams of 64 MiB fill the first 4 GiB of the log; then a deferred stream of 2^29 + 57
    bytes in two pieces (the second at a log offset past 4 GiB + 256 MiB).  One flush at finish hashes all 65."""
    from makisu_b200.abi import Range
    arena = 1 << 30
    with _engine(arena, 128, False) as e:
        e.reserve_stream_log(PAD_STREAMS * PAD_PIECE + LONG + 4096)
        e.begin()
        e.synth_fill(0, 0, arena, 0xD1)
        per = arena // PAD_PIECE
        for s in range(PAD_STREAMS // per):
            rs = []
            for i in range(per):
                r = Range()
                r.arena_off, r.len, r.stream, r.flags = i * PAD_PIECE, PAD_PIECE, s * per + i, dc.R_DEFER
                rs.append(r)
            e.device_submit(0, arena, [], rs)
        first = 1 << 28
        e.sync()
        e.synth_fill(0, 0, arena, 0xD2)
        tail = []
        for off, n, flags in ((0, first, dc.R_DEFER | dc.R_MORE), (first + 4096, LONG - first, dc.R_DEFER)):
            r = Range()
            r.arena_off, r.len, r.stream, r.flags = off, n, 100, flags
            e.device_submit(0, arena, [], [r])
            tail.append((off, n))
        res = e.finish()
        rows = e.get_stream_digests(res.n_streams)
    assert res.n_streams == 101
    pad = sc.synth(0, arena, 0xD1)
    for i in range(per):
        want = hashlib.sha256(memoryview(pad)[i * PAD_PIECE:(i + 1) * PAD_PIECE]).digest()
        assert all(rows[s * per + i].tobytes() == want for s in range(PAD_STREAMS // per))
    del pad
    long = sc.synth(0, arena, 0xD2)
    h = hashlib.sha256()
    for off, n in tail:
        h.update(memoryview(long)[off:off + n])
    assert rows[100].tobytes() == h.digest()
