"""CPU: the plain reference of tests/table_cases.py against the oracle and the host model of the exchange, on every case
the GPU file (test_gpu_table_edges.py) runs; and the generators themselves: deterministic, and holding exactly the
run lengths, table sizes and range sizes each case claims."""
import hashlib

import numpy as np
import pytest

from tests import table_cases as tc


def _sha(b):
    return hashlib.sha256(b).digest()


def _same(a: np.ndarray, b: np.ndarray):
    assert a.shape == b.shape and a.tobytes() == b.tobytes()


def _long_runs(runs):
    return sum(c for n, c in runs.items() if n > tc.FIX_SHORT)


@pytest.mark.parametrize("name", list(tc.SORT_CASES) + list(tc.MERKLE_CASES))
def test_table_case(oracle_lib, name):
    c = tc.case(name)
    again = tc.case(name)
    assert len(c.calls) == len(again.calls) and all(a.tobytes() == b.tobytes() for a, b in zip(c.calls, again.calls))
    assert all(0 < x.shape[0] <= tc.CHUNKS_ADD_MAX and x.dtype == np.uint8 for x in c.calls)
    rows = c.rows
    table = tc.table_ref(rows)
    _same(table, oracle_lib.sort_unique(rows) if rows.shape[0] else np.zeros((0, 32), np.uint8))
    assert tc.merkle_ref(table) == oracle_lib.merkle_root(table)
    runs = tc.prefix_runs(rows)
    if c.runs is not None:
        assert runs == c.runs
    if c.long_runs is not None:
        assert _long_runs(runs) == c.long_runs
    if c.n_unique is not None:
        assert table.shape[0] == c.n_unique


def test_case_families_reach_the_branches_they_name():
    # the FIX_SHORT edge, runs that mix duplicates with distinct rows, and the FIX_LONG_CAP overflow
    ties = tc.case("ties-byte31-reverse")
    assert {64, 65} <= set(tc.prefix_runs(ties.rows)) and tc.table_ref(ties.rows).shape[0] < ties.rows.shape[0]
    over = tc.case("long-run-list-overflow")
    assert over.long_runs > tc.FIX_LONG_CAP and len(over.calls) == 9 and over.rows.shape[0] == 65 * tc.OVERFLOW_RUNS
    # one-odd: the odd row sits at the claimed offset of each run, below the duplicates in one run, above in the other
    for off in tc.ODD_OFFSETS:
        rows = tc.case(f"one-odd-at-{off}").rows.reshape(2, tc.ODD_RUN, 32)
        for run, sign in zip(rows, (-1, 1)):
            odd = [i for i in range(tc.ODD_RUN) if run[i].tobytes() != run[(off + 1) % tc.ODD_RUN].tobytes()]
            assert odd == [off] and int(run[off, 31]) - int(run[(off + 1) % tc.ODD_RUN, 31]) == sign
    # radix digits: constant, or all 256 values
    for d in range(4):
        assert len(set(tc.case(f"digit{d}-const").rows[:, 3 - d])) == 1
        assert len(set(tc.case(f"digit{d}-all256").rows[:, 3 - d])) == 256
    # Merkle edges: the last level-0 group holds 1 or 2 rows (one or two SHA-256 padding blocks), and 2 vs 3 levels
    assert [n % 256 for n in (257, 258, 513, 65537)] == [1, 2, 1, 1] and -(-131073 // 256) == 513


def test_boundary_prefixes():
    for R in (2, 3, 5, 7, 8, tc.R_MAX):
        assert tc.boundary(0, R) == 0 and tc.boundary(R, R) == 1 << 64
        for j in range(1, R):
            b = tc.boundary(j, R)
            assert tc.owner(b, R) == j and tc.owner(b - 1, R) == j - 1
    b1 = tc.boundary(1, 3)
    assert b1 == 0x5555555555555556 and (b1 - 1) >> 32 == b1 >> 32   # one 32-bit tie run across the boundary
    assert tc.boundary(1023, 1024) == 0xFFC0 << 48


def _check_exchange(oracle_lib, c: tc.ExCase):
    from makisu_b200 import shard
    union = tc.table_ref(c.rows)
    ranges = tc.ranges_ref(union, c.R)
    _same(np.concatenate(ranges), union)
    local = [tc.table_ref(c.rank_rows(r)) for r in range(c.R)]
    root, model = shard.exchange_tables_model(local, _sha)
    assert root == tc.merkle_ref(union) == oracle_lib.merkle_root(union)
    for r in range(c.R):
        _same(model[r], ranges[r])
        assert shard.range_bounds(local[r], c.R) == tc.bounds_ref(local[r], c.R)
    if c.sizes is not None:
        assert [x.shape[0] for x in ranges] == c.sizes
    for p, o in c.edges:
        assert tc.owner(p, c.R) == o and any(tc.prefix64(row) == p for row in ranges[o])
    return union, ranges


@pytest.mark.parametrize("name", list(tc.EX_CASES))
def test_exchange_case(oracle_lib, name):
    c = tc.ex_case(name)
    again = tc.ex_case(name)
    assert [[x.tobytes() for x in r] for r in c.ranks] == [[x.tobytes() for x in r] for r in again.ranks]
    assert len(c.ranks) == c.R and all(x.shape[0] <= tc.CHUNKS_ADD_MAX for r in c.ranks for x in r)
    union, ranges = _check_exchange(oracle_lib, c)
    if name.startswith("boundaries"):   # every range holds rows, and some rows sit on two ranks
        assert all(x.shape[0] for x in ranges) and union.shape[0] < c.rows.shape[0]
    if name == "skew-refused":
        assert all(c.rank_rows(r).shape[0] <= c.cap for r in range(c.R)) and union.shape[0] > c.cap


def test_exchange_case_1024_ranks(oracle_lib):
    c = tc.wide_case()
    assert c.R == tc.R_MAX and {r for r in range(c.R) if c.ranks[r]} == set(tc.WIDE_RANKS)
    assert [[x.tobytes() for x in r] for r in c.ranks] == [[x.tobytes() for x in r] for r in tc.wide_case().ranks]
    union, ranges = _check_exchange(oracle_lib, c)
    assert ranges[tc.R_MAX - 1].shape[0] >= 6 and all(c.rank_rows(r).shape[0] <= c.cap for r in range(c.R))


def test_exchange_plan_of_crafted_sizes():
    """x_plan (the device code's statement of shard.level0_plan) on the crafted range sizes: who hashes which group."""
    from makisu_b200 import shard
    for sizes in tc.EX_SIZES.values():
        plans = [shard.level0_plan(sizes, r) for r in range(len(sizes))]
        assert sum(p["groups"] for p in plans) == -(-sum(sizes) // 256)
    p = shard.level0_plan([1, 1, 1, 1, 253], 0)
    assert (p["groups"], p["tail_own"], p["borrowed"]) == (1, 1, 255)   # rank 0's one row + the heads of ranks 1-4
    assert sum(shard.level0_plan([21845, 21846, 21846], r)["groups"] for r in range(3)) == 257
