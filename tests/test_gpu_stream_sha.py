"""-m gpu: the serial-stream SHA-256 (K4, k_sha256_streams) on the cases of tests/stream_cases.py against hashlib:
lane refills over 2^18 ranges, streams resumed over submits next to fresh ones, finals of 0 bytes, bit lengths of 2^32
and more, and the stream contract (the same table the CPU mock keeps).  Also K2 (k_sha256_ranges, both compiled
variants) on chunks of 2^29 bytes and more.

Only the rows of slots on which a stream finished in the session are compared; the others are unspecified."""
import ctypes

import numpy as np
import pytest

from tests import stream_cases as sc

pytestmark = pytest.mark.gpu


class EngineDriver:
    """stream_cases' driver interface over the device engine: device arenas (synth_fill or upload) or pinned host
    arenas (acquire, copy, submit)."""

    def __init__(self, e, via_host: bool):
        self.e, self.via_host = e, via_host

    def begin(self):
        self.e.begin()

    def submit(self, s: sc.Submit):
        from makisu_b200.abi import Range
        r = np.ascontiguousarray(s.ranges)
        ra = (Range * max(1, r.size)).from_buffer(r if r.size else np.zeros(1, sc.RANGE_DTYPE))
        if self.via_host:
            ptr, _, aid = self.e.arena_acquire()
            a = np.ascontiguousarray(s.arena())
            ctypes.memmove(ptr, a.ctypes.data, s.used)
            self.e.arena_submit(aid, s.used, [], ra if r.size else [])
            return
        self.e.sync()                           # the previous submit has read slot 0
        if s.seed is not None:
            self.e.synth_fill(0, 0, s.used, s.seed)
        else:
            self.e.device_upload(0, 0, s.data)
        self.e.device_submit(0, s.used, [], ra if r.size else [])

    def finish(self) -> int:
        return self.e.finish().n_streams

    def stream_digests(self, n: int) -> np.ndarray:
        return self.e.get_stream_digests(n)


def _engine(c: sc.Case, via_host: bool):
    from makisu_b200.abi import Engine
    kw = dict(n_host_arenas=2, host_arena_bytes=c.arena_bytes) if via_host else {}
    return Engine(device=0, device_arena_bytes=c.arena_bytes, max_extents=c.max_extents, **kw)


def test_long_streams_synth_content_is_the_reference_content():
    """The reference hashes stream_cases.synth; the device fills the same bytes with mksnap_synth_fill."""
    c = sc.case("long_streams")
    s = c.submits[1]
    with _engine(c, False) as e:
        e.begin()
        e.synth_fill(0, 0, s.used, s.seed)
        got = e.device_download(0, 0, s.used)
        e.finish()
    np.testing.assert_array_equal(got, s.arena())


@pytest.mark.parametrize("via_host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("name", list(sc.STREAM_CASES))
def test_stream_cases(name, via_host):
    """Every finished slot's row equals hashlib over its stream's pieces; n_streams = highest finished slot + 1."""
    if via_host and name not in sc.MULTI_SUBMIT:
        pytest.skip("single-submit case: the device arena path covers it")
    c = sc.case(name)
    with _engine(c, via_host) as e:
        sc.run_case(EngineDriver(e, via_host), c)


def test_ragged_many_refills_every_lane():
    """The launch really is capped: on this device each lane takes at least 10 pieces on average."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = sc.case("ragged_many").submits[0].ranges.size
    assert n / (min(-(-n // 32), sc.K4_PAIRS_PER_SM * sms) * 32) >= 10


@pytest.mark.parametrize("outcome", sc.contract(), ids=lambda o: o.name)
def test_stream_contract(outcome):
    """What the engine accepts and refuses (slot range, one piece per slot per submit, MORE pieces non-empty multiples
    of 64, bounds, finish with a stream left open), each followed by a valid session on the same handle."""
    c = sc.Case("contract", sc.CONTRACT_ARENA, sc.CONTRACT_MAX, [])
    with _engine(c, False) as e:
        sc.run_outcome(EngineDriver(e, False), outcome)


@pytest.mark.parametrize("flags", ["tar-digest", "file-digests"])
def test_ingest_members_split_over_1mib_arenas(flags, tmp_path):
    """libmkhost's tar stream on the engine when a member larger than the arena comes first: the arena is flushed before
    it holds any stream byte, and that empty piece must not go out as an (illegal) empty MKSNAP_R_MORE piece."""
    from makisu_b200 import host
    from makisu_b200.abi import Engine
    from tests import gzip_corpus as gc

    def make_engine(arena_bytes):
        return Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                      max_extents=1 << 12)

    f = host.MKHOST_FILE_DIGESTS if flags == "file-digests" else 0
    for name, blob in gc.layer_blobs():
        gc.check_ingest(make_engine, str(tmp_path), name, blob, f, arena_bytes=1 << 20)


@pytest.mark.parametrize("fma", ["1", "0"], ids=["fma", "plain-adds"])
def test_long_chunks(fma, monkeypatch):
    """K2 on one-chunk files of 2^29 - 1 .. 2^29 + 64 bytes (8 * len crosses 2^32): ends, digests, table, root."""
    from makisu_b200.abi import CdcParams, Engine, Extent, MKSNAP_X_CDC
    monkeypatch.setenv("MKSNAP_SHA_FMA", fma)
    lc = sc.long_chunks()
    ext = []
    for off, n in lc.files:
        x = Extent()
        x.arena_off, x.len, x.crc_suffix, x.flags = off, n, 0, MKSNAP_X_CDC
        ext.append(x)
    with Engine(device=0, device_arena_bytes=lc.arena.size, max_extents=16, cdc=CdcParams(*lc.params)) as e:
        e.begin()
        e.device_upload(0, 0, lc.arena)
        e.device_submit(0, lc.arena.size, ext)
        res = e.finish()
        w = lc.want
        assert res.n_chunks == w["n_chunks"]
        ends, dig = e.get_chunks(res.n_chunks)
        np.testing.assert_array_equal(ends, w["ends"])
        np.testing.assert_array_equal(dig, w["digests"])
        assert res.n_unique == w["n_unique"]
        np.testing.assert_array_equal(e.get_table(res.n_unique), w["table"])
        assert bytes(res.root) == w["root"]
