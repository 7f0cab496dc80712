"""-m gpu: K3 (radix sort on the top 32 bits, tie fix-up, long-run vote and its overflow, unique), the Merkle root and the
range-partitioned exchange on crafted chunk tables.  The rows of tests/table_cases.py go in through mksnap_chunks_add
(no content behind them) and every result is compared with that module's plain Python reference: table, n_unique,
root, the appended rows in call order, and for the exchange every rank's range, root and counters."""
import ctypes
import resource
import time

import numpy as np
import pytest

from tests import table_cases as tc
from tests.util import cdc_extents, pack

pytestmark = pytest.mark.gpu

INJECTED_END = np.uint64(2 ** 64 - 1)   # chunk end of a row appended by mksnap_chunks_add
MAX_ROWS = 600_000                       # the largest case: 8 300 runs of 65 rows


def _engine(max_chunks):
    from makisu_b200.abi import Engine
    return Engine(device=0, device_arena_bytes=1 << 20, max_extents=16, max_chunks=max_chunks)


@pytest.fixture(scope="module")
def eng():
    e = _engine(MAX_ROWS)
    yield e
    e.close()


def _session(e, calls):
    e.begin()
    for x in calls:
        e.chunks_add(x)
    t0 = time.perf_counter()
    res = e.finish()
    return res, time.perf_counter() - t0


def _check_table(e, res, rows, pre=0):
    """res of a session holding `pre` computed chunks followed by the appended `rows` (all of them in `rows` if pre=0)."""
    table = tc.table_ref(rows)
    assert res.n_chunks == rows.shape[0]
    assert res.n_unique == table.shape[0]
    if table.shape[0]:
        np.testing.assert_array_equal(e.get_table(res.n_unique), table)
    assert bytes(res.root) == tc.merkle_ref(table)
    if rows.shape[0]:
        ends, dig = e.get_chunks(res.n_chunks)
        assert (ends[pre:] == INJECTED_END).all()
        np.testing.assert_array_equal(dig, rows)
    return table


@pytest.mark.parametrize("name", list(tc.SORT_CASES) + list(tc.MERKLE_CASES))
def test_table_edges(eng, name):
    c = tc.case(name)
    res, sec = _session(eng, c.calls)
    _check_table(eng, res, c.rows)
    if c.runs and max(c.runs) >= 1000:   # runs one GPU thread insertion-sorts
        print(f"\n{name}: finish {sec * 1e3:.1f} ms, longest run {max(c.runs)} rows")


def test_injected_rows_next_to_cdc_chunks(eng, oracle_lib):
    """Appended rows behind the chunks of a real CDC submit, some equal to those chunks, some repeated across calls;
    and the same multiset in two other shuffles and call splits gives the identical table and root."""
    rng = np.random.default_rng(0x51)
    segs = [rng.integers(0, 256, n, dtype=np.uint8) for n in (300_000, 5_000, 200_000)]
    arena, offs = pack(segs)
    lens = [len(s) for s in segs]
    want = oracle_lib.chunk_table(arena, offs, lens)
    c = tc.mix_case()
    calls = c.calls[:2] + [want["digests"][::3]] + c.calls[2:]
    injected = np.concatenate(calls)
    n_cdc = want["n_chunks"]
    eng.begin()
    eng.device_upload(0, 0, arena)
    eng.device_submit(0, arena.size, cdc_extents(offs, lens))
    for x in calls:
        eng.chunks_add(x)
    res = eng.finish()
    table = _check_table(eng, res, np.concatenate([want["digests"], injected]), pre=n_cdc)
    ends, _ = eng.get_chunks(res.n_chunks)
    np.testing.assert_array_equal(ends[:n_cdc], want["ends"])
    assert table.shape[0] < res.n_chunks
    for seed, per_call in ((1, 65536), (2, 777)):
        shuffled = injected[np.random.default_rng(seed).permutation(injected.shape[0])]
        r, _ = _session(eng, tc.split_calls(shuffled, per_call))
        assert r.n_unique == tc.table_ref(injected).shape[0]
        if seed == 1:
            first = (bytes(r.root), eng.get_table(r.n_unique).tobytes())
            assert first[0] == tc.merkle_ref(tc.table_ref(injected))
        else:
            assert (bytes(r.root), eng.get_table(r.n_unique).tobytes()) == first


@pytest.mark.parametrize("name", ["ties-byte31-random", "half-duplicates-2048", "long-run-list-overflow", "merkle-n65537"])
def test_allgather_world_of_one(name):
    """The same crafted tables merged by mksnap_allgather_tables on a one-rank communicator: result == finish()."""
    from makisu_b200.abi import Engine
    c = tc.case(name)
    with _engine(MAX_ROWS) as e:
        e.comm_init(Engine.comm_unique_id(), 1, 0)
        r, _ = _session(e, c.calls)
        table = _check_table(e, r, c.rows)
        g = e.allgather_tables()
        assert (g.n_chunks, g.n_unique, bytes(g.root)) == (r.n_chunks, r.n_unique, bytes(r.root))
        np.testing.assert_array_equal(e.get_table(g.n_unique), table)


# ---------------------------------------------------------------------------------------------------------------
# range exchange between R engines of this process (mksnap_exchange_tables_local)
# ---------------------------------------------------------------------------------------------------------------
def _exchange(engines, c):
    from makisu_b200.abi import Engine
    local = []
    for e, calls in zip(engines, c.ranks):
        r, _ = _session(e, calls)
        assert r.n_chunks == sum(x.shape[0] for x in calls)
        local.append(r)
    return local, Engine.exchange_tables_local(engines)


def _check_exchange(engines, c, local, outs):
    union = tc.table_ref(c.rows)
    root = tc.merkle_ref(union)
    ranges = tc.ranges_ref(union, c.R)
    crc = 0
    for r in local:
        crc ^= r.crc_pure
    got = []
    for k, (e, o) in enumerate(zip(engines, outs)):
        assert bytes(o.root) == root, k
        assert (o.n_unique, o.n_chunks, o.crc_pure) == (union.shape[0], c.rows.shape[0], crc), k
        assert (o.n_files, o.cdc_bytes, o.crc_bytes) == (sum(r.n_files for r in local), sum(r.cdc_bytes for r in local),
                                                         sum(r.crc_bytes for r in local)), k
        rows = e.get_table(e.table_rows())
        np.testing.assert_array_equal(rows, ranges[k], err_msg=f"rank {k}")
        got.append(rows.tobytes())
    assert b"".join(got) == union.tobytes()


@pytest.mark.parametrize("name", [n for n in tc.EX_CASES if n != "skew-refused"])
def test_exchange_edges(name):
    c = tc.ex_case(name)
    engines = [_engine(c.cap or c.rows.shape[0] + 64) for _ in range(c.R)]
    try:
        local, outs = _exchange(engines, c)
        _check_exchange(engines, c, local, outs)
    finally:
        for e in engines:
            e.close()


def test_exchange_skew_refused_then_handles_still_work():
    """Every row in range 0, more than rank 0's max_chunks: E_CAPACITY ("skewed") on every rank, and afterwards the
    same handles run sessions and a valid exchange."""
    from makisu_b200.abi import MksnapError
    c = tc.ex_case("skew-refused")
    engines = [_engine(c.cap) for _ in range(c.R)]
    try:
        with pytest.raises(MksnapError, match="E_CAPACITY.*skewed"):
            _exchange(engines, c)
        ok = tc.ex_case("boundaries-r3")
        assert ok.R == c.R and ok.rows.shape[0] <= c.cap
        local, outs = _exchange(engines, ok)
        _check_exchange(engines, ok, local, outs)
    finally:
        for e in engines:
            e.close()


def _host_available_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _device_free_bytes():
    """cuMemGetInfo on the context the engines made current (the device's primary context)."""
    free, total = ctypes.c_size_t(), ctypes.c_size_t()
    rc = ctypes.CDLL("libcuda.so.1").cuMemGetInfo_v2(ctypes.byref(free), ctypes.byref(total))
    assert rc == 0, f"cuMemGetInfo_v2: {rc}"
    return free.value


def test_exchange_1024_ranks():
    """R = 1024, the most the exchange takes: 1024 minimal engines, rows on four of them, prefixes owned by rank 1023.
    R = 1025 is refused (E_INVAL).  Every handle holds about 17 MiB of exchange buffers at R = 1024, and the local
    exchange keeps every rank's copy of the gathered header (R x (8 + R) words) on the host."""
    from makisu_b200.abi import Engine, MksnapError
    c = tc.wide_case()
    R = c.R
    engines = []
    try:
        t0 = time.perf_counter()
        engines.append(_engine(c.cap))
        free0 = _device_free_bytes()
        for _ in range(16):
            engines.append(_engine(c.cap))
        per_engine = (free0 - _device_free_bytes()) / 16
        x_bytes = (R + 1) * 8 + R * (8 + R) * 8 + R * 8192 + 256 * 32   # d_xbounds, d_xhdr, d_xrec, d_xtail
        need = (R + 1) * per_engine + R * (x_bytes + (2 << 20)) + (2 << 30)
        host_need = R * R * (8 + R) * 8 + (4 << 30)
        if free0 < need or _host_available_bytes() < host_need:
            pytest.skip(f"1024-rank exchange needs ~{need / 2**30:.1f} GiB free device memory (have {free0 / 2**30:.1f}) "
                        f"and ~{host_need / 2**30:.1f} GiB host memory (have {_host_available_bytes() / 2**30:.1f})")
        while len(engines) < R + 1:
            engines.append(_engine(c.cap))
        t_create = time.perf_counter() - t0
        for e in engines:   # every handle finished; the 1025th holds nothing
            e.begin()
            e.finish()
        with pytest.raises(MksnapError, match="E_INVAL"):
            Engine.exchange_tables_local(engines)
        engines.pop().close()
        t1 = time.perf_counter()
        local, outs = _exchange(engines, c)
        t_exchange = time.perf_counter() - t1
        used = free0 - _device_free_bytes() + per_engine
        _check_exchange(engines, c, local, outs)
        print(f"\n1024-rank exchange: ran; {R + 1} engines created in {t_create:.1f} s, sessions + exchange "
              f"{t_exchange:.1f} s; device memory held after the exchange {used / 2**30:.2f} GiB "
              f"({per_engine / 2**20:.1f} MiB per engine before it); process peak RSS "
              f"{resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GiB")
    finally:
        for e in engines:
            e.close()
