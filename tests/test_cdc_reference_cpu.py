"""The CDC reference and case generators of tests/cdc_cases.py, checked on the CPU: the numpy reference against the
oracle's C code (roll_at, cdc_cuts) on random content and on every crafted case, every claim a generator makes about
what it planted, and a model of k_select_cuts_big's staging that shows each big-file case reaches the path it names."""
import functools

import numpy as np
import pytest

from tests import cdc_cases as cc


@functools.lru_cache(maxsize=None)
def _case(name):
    c = cc.case(name)
    return c, cc.Cands.of(c.arena, c.params)


def _oparams(olib, p):
    return olib.CdcParams(*p.astuple())


PARAM_SETS = [cc.DEFAULT, cc.Params(64, 256, 1024, 10, 6), cc.Params(64, 64, 64, 8, 8), cc.Params(100, 1000, 5000, 12, 9),
              cc.Params(64, 512, 4096, 16, 12), cc.Params(64, 256, 1024, 16, 8), cc.Params(4096, 16384, 131072, 16, 8),
              cc.Params(4096, 16384, 1 << 20, 16, 12)]


def test_roll_hash_matches_oracle(oracle_lib):
    rng = np.random.default_rng(1)
    d = rng.integers(0, 256, 200_000, dtype=np.uint8)
    h = cc.roll_hash(d)
    for i in [0, 1, 2, 3, 30, 31, 32, 33, 34, 35, 4095, 4096, 123_457, d.size - 1]:
        assert int(h[i]) == oracle_lib.roll_at(d, i), i
    idx = rng.integers(0, d.size, 300)
    np.testing.assert_array_equal(cc.hash_at(d, idx), h[idx])
    np.testing.assert_array_equal(cc.hash_at(d, np.arange(40)), h[:40])
    assert oracle_lib.roll_multiplier() == cc.M
    # the byte coefficients: changing byte j by delta changes h_{j+d} by delta * C[d], and nothing else
    e = d.copy()
    e[1000] ^= 0x5A
    diff = (cc.roll_hash(e).astype(np.int64) - h.astype(np.int64)) & cc.MASK32
    delta = (int(e[1000]) - int(d[1000])) & cc.MASK32
    assert np.flatnonzero(diff).max() <= 1034 and np.flatnonzero(diff).min() >= 1000
    assert [int(diff[1000 + k]) for k in range(35)] == [(delta * cc.C[k]) & cc.MASK32 for k in range(35)]


@pytest.mark.parametrize("p", PARAM_SETS, ids=lambda p: "-".join(map(str, p.astuple())))
def test_cut_rule_matches_oracle_on_random_content(oracle_lib, p):
    rng = np.random.default_rng(sum(p.astuple()))
    d = rng.integers(0, 256, 3_000_000, dtype=np.uint8)
    d[100_000:600_000] = 0
    d[900_000:2_400_000:3] = 0x41
    c = cc.Cands.of(d, p)
    for off, n in [(0, d.size), (12345, 1_000_000), (4096, p.min_size), (4096, p.min_size + 1), (0, 0)]:
        want = [off + int(x) for x in oracle_lib.cdc_cuts(d[off:off + n], _oparams(oracle_lib, p))]
        assert cc.file_cuts(off, n, c, p) == want


def test_plant_clear_and_every_byte_loose():
    rng = np.random.default_rng(7)
    p = cc.DEFAULT
    d = rng.integers(0, 256, 1 << 20, dtype=np.uint8)
    h0 = cc.classify(cc.roll_hash(d), p)
    pos = np.arange(1000, 900_000, 991)
    cls = np.where(np.arange(pos.size) % 2 == 0, cc.STRICT, cc.LOOSE).astype(np.int8)
    e = d.copy()
    cc.plant(e, pos, cls, p, rng)
    h1 = cc.classify(cc.roll_hash(e), p)
    np.testing.assert_array_equal(h1[pos], cls)
    other = np.ones(d.size, dtype=bool)
    other[pos] = False
    assert not (h1[other & (h0 == cc.NONE)]).any()                # no new candidate
    near = np.zeros(d.size, dtype=bool)
    for k in range(-2, 35):
        near[pos + k] = True
    np.testing.assert_array_equal(h1[~near], h0[~near])          # nothing changed away from the plants
    cc.clear(e, [(500_000, 700_000)], p, rng)
    h2 = cc.classify(cc.roll_hash(e), p)
    assert not h2[500_000:700_000].any()
    np.testing.assert_array_equal(h2[:500_000], h1[:500_000])
    q = cc.Params(64, 256, 1024, 16, 8)
    cc.every_byte_loose(e, 800_000, 804_096, q)
    assert (cc.classify(cc.roll_hash(e), q)[800_000:804_096] != cc.NONE).all()
    blk = np.tile(cc.dense_block(4096, q), 5)
    k = cc.classify(cc.roll_hash(np.concatenate([d[:4096], blk])), q)[4096:].reshape(5, 4096)
    assert (k[:, 35:] != cc.NONE).all()


@pytest.mark.parametrize("name", list(cc.ALL_CASES))
def test_case_reference_matches_oracle(oracle_lib, name):
    c, cands = _case(name)
    for off, n in c.files:
        want = [off + int(x) for x in oracle_lib.cdc_cuts(c.arena[off:off + n], _oparams(oracle_lib, c.params))]
        assert cc.file_cuts(off, n, cands, c.params) == want, (off, n)


@pytest.mark.parametrize("name", list(cc.ALL_CASES))
def test_case_claims(name):
    c, cands = _case(name)
    h = cc.classify(cc.roll_hash(c.arena), c.params)
    for q, cls, why in c.planted:
        assert h[q] == cls, (q, why)
    others = h.copy()
    others[[q for q, _, _ in c.planted]] = cc.NONE
    for a, b in c.cleared:
        assert not others[a:b].any(), (a, b)          # no candidate but the planted ones
    for a, b in c.dense:
        assert (h[a:b] != cc.NONE).all(), (a, b)
    ends = {e for off, n in c.files for e in cc.file_cuts(off, n, cands, c.params)}
    for e, is_end, why in c.cuts:
        assert (e in ends) == is_end, (e, why)
    if c.pieces is not None:
        assert [sum(x) for x in c.pieces] == [n for _, n in c.files]


def test_sweep_covers_every_row_offset_and_region_start():
    c, cands = _case("sweep")
    pos = np.array([q for q, _, _ in c.planted])
    reg, inreg = pos // cc.SCAN_TILE, pos % cc.SCAN_TILE
    row, off = inreg // cc.ROW, inreg % cc.ROW
    for r in (1, 16, 31):
        assert set(off[row == r].tolist()) >= (set(range(cc.ROW)) if r != 31 else set(range(99))), r
    # every region inside a file holds a row-0 plant, so every tile start of every scan shape has one
    for o, n in c.files:
        full = np.arange(-(-(o + 64) // cc.SCAN_TILE), (o + n - 64) // cc.SCAN_TILE)
        assert set(full.tolist()) <= set(reg[row == 0].tolist())
    assert set((off[row == 0] % 35).tolist()) == set(range(35)) and set(off[row == 0].tolist()) == set(range(35))
    assert c.arena.size >= 64 << 20
    # with the background cleared every plant ends a chunk
    cleared_plants = sum(1 for q in pos if any(a <= q < b for a, b in c.cleared))
    assert sum(1 for _, is_end, _ in c.cuts if is_end) == cleared_plants > 10_000


def test_dense_case_overfills_lanes_and_pool_blocks():
    c, cands = _case("dense")
    per_region = np.bincount(cands.loose // cc.SCAN_TILE)
    assert per_region.max() == cc.SCAN_TILE > cc.SCAN_POOL_BLOCK
    per_row = np.bincount(cands.loose // cc.ROW)
    assert per_row.max() == cc.ROW                                   # one lane with a candidate at every byte
    assert (per_row > 1).sum() > 100                                 # lanes with more than one candidate


@pytest.mark.parametrize("name", ["windows", "fallback"])
def test_big_file_staging_reaches_its_path(name):
    c, cands = _case(name)
    for fi, path in c.staging.items():
        off, n = c.files[fi]
        assert n >= cc.SELECT_BIG_FILE
        st = cc.select_big_model(off, n, cands, c.params)
        assert st.cuts == cc.file_cuts(off, n, cands, c.params)      # the model computes what the rule does
        got = {"edge": st.edge_cuts, "crossing": st.crossings, "shrink": st.shrunk, "fallback": st.fallbacks}[path]
        assert got > 0, (fi, path, st.windows)


@pytest.mark.parametrize("params", [(64, 128, 256, 8, 6), (64, 256, 1024, 4, 3), (4096, 16384, 131072, 16, 12)])
def test_random_content_never_takes_the_fallback(params):
    """The densest parameter sets of the existing big-file tests stage windows of far more than max bytes, so with
    random content a whole file never reaches select_one_cut from k_select_cuts_big: only the end of a piece whose
    file continues does (or the dense windows of the fallback case)."""
    p = cc.Params(*params)
    d = np.random.default_rng(5).integers(0, 256, 24 << 20, dtype=np.uint8)
    st = cc.select_big_model(4096, d.size - 8192, cc.Cands.of(d, p), p)
    assert st.fallbacks == 0 and st.windows >= 2
