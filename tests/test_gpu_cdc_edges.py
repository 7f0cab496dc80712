"""-m gpu: the CDC scan (K1, k_roll_scan) and the cut selection (K1b, k_select_cuts / k_select_cuts_big) on planted
Roll-32 candidates (tests/cdc_cases.py), against the numpy reference: chunk count, every chunk end and digest, the
table and the root.

The scan cases run on every compiled k_roll_scan shape (MKSNAP_SCAN_CFG) and on the CRC variant (the same submit with
CRC extents, its CRC-32 checked against zlib); the selection cases on the default shape and the CRC variant; files over
submits through device and pinned host arenas.  Also: a candidate pool overflow (MKSNAP_E_CAPACITY, then a normal
session on the same engine), the largest max_size the engine accepts, and K2's plain-add variant (MKSNAP_SHA_FMA=0)."""
import ctypes
import functools
import zlib

import numpy as np
import pytest

from tests import cdc_cases as cc

pytestmark = pytest.mark.gpu

N_SCAN_SHAPES = 7          # MK_SCAN_SHAPES in mksnap.cu
SHAPES = [str(i) for i in range(N_SCAN_SHAPES)] + ["crc"]


@functools.lru_cache(maxsize=None)
def _ref(name):
    c = cc.case(name)
    return c, cc.chunk_table(c.arena, c.files, c.params)


def _cdc(p: cc.Params):
    from makisu_b200.abi import CdcParams
    return CdcParams(*p.astuple())


def _extents(files, crc: bool):
    from makisu_b200.abi import Extent, MKSNAP_X_CDC, MKSNAP_X_CRC
    out, after = [], sum(n for _, n in files)
    for off, n in files:
        after -= n
        x = Extent()
        x.arena_off, x.len, x.crc_suffix = off, n, after if crc else 0
        x.flags = MKSNAP_X_CDC | (MKSNAP_X_CRC if crc else 0)
        out.append(x)
    return out


def _check(e, res, want, want_ends=None):
    assert res.n_chunks == want["n_chunks"]
    ends, dig = e.get_chunks(res.n_chunks)
    np.testing.assert_array_equal(ends, want["ends"] if want_ends is None else want_ends)
    np.testing.assert_array_equal(dig, want["digests"])
    assert res.n_unique == want["n_unique"]
    np.testing.assert_array_equal(e.get_table(res.n_unique), want["table"])
    assert bytes(res.root) == want["root"]


def _one_submit(c, want, crc: bool, **kw):
    from makisu_b200.abi import Engine
    with Engine(device=0, device_arena_bytes=c.arena.size, max_extents=len(c.files) + 8, cdc=_cdc(c.params), **kw) as e:
        e.begin()
        e.device_upload(0, 0, c.arena)
        e.device_submit(0, c.arena.size, _extents(c.files, crc))
        res = e.finish()
        _check(e, res, want)
        if crc:
            assert e.ctx_crc32(res) == zlib.crc32(b"".join(c.arena[o:o + n].tobytes() for o, n in c.files))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("name", list(cc.SCAN_CASES))
def test_scan_shapes_on_planted_candidates(name, shape, monkeypatch):
    """Candidates at every row offset and in the first row of every tile (64 MiB: every CTA goes round its stage ring
    at least twice in every shape), and regions with a candidate at every byte."""
    c, want = _ref(name)
    monkeypatch.setenv("MKSNAP_SCAN_CFG", "0" if shape == "crc" else shape)
    _one_submit(c, want, crc=shape == "crc")


@pytest.mark.parametrize("crc", [False, True], ids=["scan", "crc-scan"])
@pytest.mark.parametrize("name", list(cc.SELECT_CASES))
def test_cut_selection_on_planted_candidates(name, crc):
    """Cut-rule boundaries (min-2 / min-1, normal-2 / normal-1, max-1 / max) in small and big files, the big-file
    selector's window edges, shrunk windows and its fallback to select_one_cut, chunks longer than the length classes."""
    c, want = _ref(name)
    _one_submit(c, want, crc)


def _split_session(e, c, cap, carry, via_host):
    """One session over the pieces of c.files: a file's first piece joins the current arena (flushed first when it does
    not fit), every later piece opens a new submit at arena offset `carry`.  -> (result, chunk ends in session-stream
    coordinates of the reference's chunks)."""
    from makisu_b200.abi import Extent, MKSNAP_X_CDC, MKSNAP_X_CONT, MKSNAP_X_MORE
    arena = np.zeros(cap, dtype=np.uint8)
    ext, pos, base = [], 0, 0
    where = []                                  # per file: [(file offset, piece length, stream offset of its start)]

    def flush():
        nonlocal arena, ext, pos, base
        if via_host:
            ptr, _, aid = e.arena_acquire()
            ctypes.memmove(ptr, arena.ctypes.data, pos)
            e.arena_submit(aid, pos, ext)
        else:
            e.sync()
            e.device_upload(0, 0, arena[:pos])
            e.device_submit(0, pos, ext)
        base += pos
        arena = np.zeros(cap, dtype=np.uint8)
        ext, pos = [], 0

    e.begin()
    for (off, n), pieces in zip(c.files, c.pieces or [[n] for _, n in c.files]):
        done, w = 0, []
        for k, m in enumerate(pieces):
            first, last = k == 0, k == len(pieces) - 1
            if not first:
                flush()
                pos = carry
            elif (pos + 511) // 512 * 512 + m > cap:
                flush()
            pos = (pos + 511) // 512 * 512
            arena[pos:pos + m] = c.arena[off + done:off + done + m]
            x = Extent()
            x.arena_off, x.len, x.crc_suffix = pos, m, 0
            x.flags = MKSNAP_X_CDC | (0 if first else MKSNAP_X_CONT) | (0 if last else MKSNAP_X_MORE)
            x.reserved = 0 if last else min(n - done - m, 0xFFFFFFFF)
            ext.append(x)
            w.append((done, m, base + pos))
            pos += m
            done += m
        where.append(w)
    flush()
    res = e.finish()
    ends = []
    for (off, n), w in zip(c.files, where):
        for cut in cc.file_cuts(off, n, _cands(c), c.params):
            x = cut - off
            s, m, at = next(t for t in w if t[0] < x <= t[0] + t[1])
            ends.append(at + x - s)
    return res, np.array(ends, dtype=np.uint64)


@functools.lru_cache(maxsize=None)
def _cands_of(name):
    c, _ = _ref(name)
    return cc.Cands.of(c.arena, c.params)


def _cands(c):
    return _cands_of(c.name)


@pytest.mark.parametrize("via_host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("name", list(cc.CONT_CASES))
def test_files_over_submits_with_planted_candidates(name, via_host):
    """Candidates at a piece's last byte, at the continuation's first and second byte, an open chunk of max - 1 bytes,
    small and big pieces, and (max = 1 MiB) a continuation behind a carry area of 1 MiB."""
    from makisu_b200.abi import Engine
    c, want = _ref(name)
    cap = 16 << 20
    kw = dict(n_host_arenas=2, host_arena_bytes=cap) if via_host else {}
    with Engine(device=0, device_arena_bytes=cap, max_extents=64, cdc=_cdc(c.params), **kw) as e:
        carry = e.limits().carry_bytes
        assert carry == -(-c.params.max_size // 512) * 512
        res, ends = _split_session(e, c, cap, carry, via_host)
        _check(e, res, want, ends)


def test_pool_overflow_is_a_capacity_error_and_the_engine_recovers():
    """8 MiB with a candidate at nearly every byte (loose_bits 8) overfill the candidate pool of a 64 MiB arena,
    max(2^20, (2^26 >> 8) * 8) + 2 * SMs * 32 * 256 entries: finish reports MKSNAP_E_CAPACITY, and the next session on
    the same engine is exact."""
    from makisu_b200.abi import Engine, MksnapError
    p = cc.Params(4096, 16384, 131072, 16, 8)
    dense = np.tile(cc.dense_block(cc.SCAN_TILE, p), 2048)
    assert int((cc.roll_hash(dense) >= np.uint32(p.loose_thr)).sum()) > 8_000_000
    arena_bytes = 64 << 20
    with Engine(device=0, device_arena_bytes=arena_bytes, max_extents=64, cdc=_cdc(p)) as e:
        e.begin()
        e.device_upload(0, 0, dense)
        e.device_submit(0, dense.size, _extents([(0, dense.size)], False))
        with pytest.raises(MksnapError) as ei:
            e.finish()
        assert ei.value.code == -4 and "candidate pool overflow" in str(ei.value)
        import torch
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        cap = max(1 << 20, (arena_bytes >> p.loose_bits) * 8) + 2 * sms * 32 * cc.SCAN_POOL_BLOCK
        assert f"capacity {cap} entries" in str(ei.value)
        rng = np.random.default_rng(77)
        arena = rng.integers(0, 256, 8 << 20, dtype=np.uint8)
        files = [(0, 3 << 20), (3 << 20, (5 << 20) - 512)]
        e.begin()
        e.device_upload(0, 0, arena)
        e.device_submit(0, arena.size, _extents(files, False))
        _check(e, e.finish(), cc.chunk_table(arena, files, p))


def test_max_size_limit():
    """max_size above MKSNAP_CDC_MAX_SIZE_LIMIT is refused; at the limit every search range of a big file leaves the
    staged window (each cut comes from select_one_cut), and a 20 MiB zero file is one chunk."""
    from makisu_b200.abi import Engine, MksnapError
    with pytest.raises(MksnapError) as ei:
        Engine(device=0, device_arena_bytes=1 << 20, max_extents=8, cdc=_cdc(cc.Params(4096, 16384, cc.MAX_SIZE_LIMIT + 1, 16, 12)))
    assert ei.value.code == -1
    p = cc.Params(4096, 16384, cc.MAX_SIZE_LIMIT, 16, 12)
    rng = np.random.default_rng(91)
    arena = np.zeros(64 << 20, dtype=np.uint8)
    arena[4096:4096 + (40 << 20)] = rng.integers(0, 256, 40 << 20, dtype=np.uint8)
    files = [(4096, 40 << 20), ((41 << 20), 20 << 20), ((62 << 20), 1 << 20)]
    want = cc.chunk_table(arena, files, p)
    assert int(want["ends"][-2]) == (41 << 20) + (20 << 20) and int(want["ends"][-3]) <= 41 << 20
    with Engine(device=0, device_arena_bytes=arena.size, max_extents=8, cdc=_cdc(p)) as e:
        e.begin()
        e.device_upload(0, 0, arena)
        e.device_submit(0, arena.size, _extents(files, False))
        _check(e, e.finish(), want)


def test_chunk_digests_every_alignment_and_tail_plain_adds(monkeypatch):
    """The chunk SHA-256 kernel's other compiled variant (additions on the ALU pipe, MKSNAP_SHA_FMA=0) on the
    alignment and tail cases of test_gpu_chunk_sha_alignment."""
    from tests import test_gpu_chunk_sha_alignment as align
    monkeypatch.setenv("MKSNAP_SHA_FMA", "0")
    align.test_chunk_digests_every_alignment_and_tail()
