"""CPU: cacheIDs of a whole build plan (mkhost_plan_cache_ids).

The oracle chain (tests/plan_oracle.py) is checked against hand-chained per-step oracle calls, mksnap_crc_prepend
against zlib, and the host plan logic of libmkhost against the oracle under the CPU mock of the engine
(tests/mock_engine/mock_mksnap.cpp, whose fold entry points restate k_crc_fold with the oracle's arithmetic).  Mock
scenarios run in a fresh process that loads the mock with RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_plan_cache_ids_cpu <mock.so> <scenario> <tmpdir>"""
import os
import sys
import zlib

import numpy as np
import pytest

from makisu_b200 import abi
from makisu_b200.host import PlanStep
from oracle import ctx_crc
from tests import mock_engine, plan_oracle

T = 1_500_000_000


def _mk(root, rel, data=b""):
    p = os.path.join(root, rel)
    os.makedirs(os.path.dirname(p), exist_ok=True)
    with open(p, "wb") as f:
        f.write(data)
    os.utime(p, (T, T))
    return p


def _ctx(tmp, seed=7, big=0):
    c = os.path.join(tmp, "ctx")
    rng = np.random.default_rng(seed)
    _mk(c, "Dockerfile", b"FROM scratch\n")
    _mk(c, "requirements.txt", b"numpy\nscipy\n")
    for d in range(3):
        for i in range(4):
            _mk(c, f"d{d}/f{i}.bin", rng.integers(0, 256, int(rng.integers(1, 50_000)), dtype=np.uint8).tobytes())
    _mk(c, "d0/empty", b"")
    _mk(c, "a.json", b'{"a": 1}')
    _mk(c, "b.json", b"")
    os.makedirs(os.path.join(c, "emptydir"))
    os.symlink("d0/f1.bin", os.path.join(c, "link"))
    if big:
        _mk(c, "d1/big.bin", rng.integers(0, 256, big, dtype=np.uint8).tobytes())
    return c


def _plan():
    """Two stages plus a remote image named by a COPY --from: FROM, RUN/ENV (commit true and false), COPY, ADD, globs,
    overlapping sources and COPY --from."""
    return [
        PlanStep.from_image("debian:8"),
        PlanStep.copy("COPY", "requirements.txt /app/", ["requirements.txt"]),
        PlanStep.base("RUN", "pip install -r /app/requirements.txt", True),
        PlanStep.copy("COPY", ". /app/", ["."]),
        PlanStep.base("ENV", "A=1", False),
        PlanStep.copy("ADD", "d0 d1/f2.bin /x/", ["d0", "d1/f2.bin"]),
        PlanStep.copy("COPY", "*.json /cfg/", ["*.json"]),
        PlanStep.from_image("alpine:3", remote=True),
        PlanStep.from_image("busybox"),
        PlanStep.copy("COPY", "--from=0 /app /app", ["/app"], from_stage="0"),
        PlanStep.copy("COPY", "--from=alpine:3 /bin/sh /sh", ["/bin/sh"], from_stage="alpine:3"),
        PlanStep.copy("COPY", "d0/f1.bin link /y/", ["d0/f1.bin", "link"]),
        PlanStep.base("RUN", "true", False),
    ]


def test_oracle_plan_equals_hand_chained_steps(tmp_path):
    c = _ctx(str(tmp_path))
    seed = ctx_crc.plan_seed(True, False)
    got = plan_oracle.plan_cache_ids(seed, c, _plan())
    s0 = ctx_crc.from_step_cache_id(seed, "debian:8")
    s1 = ctx_crc.copy_step_cache_id(s0, "COPY", "requirements.txt /app/", c, ["requirements.txt"])
    s2 = ctx_crc.base_step_cache_id(s1, "RUN", "pip install -r /app/requirements.txt", True)
    s3 = ctx_crc.copy_step_cache_id(s2, "COPY", ". /app/", c, ["."])
    s4 = ctx_crc.base_step_cache_id(s3, "ENV", "A=1", False)
    s5 = ctx_crc.copy_step_cache_id(s4, "ADD", "d0 d1/f2.bin /x/", c, ["d0", "d1/f2.bin"])
    s6 = ctx_crc.copy_step_cache_id(s5, "COPY", "*.json /cfg/", c, ["*.json"])
    r7 = ctx_crc.from_step_cache_id(s6, "alpine:3")       # the remote-image stage: seeded like the stage after it
    s8 = ctx_crc.from_step_cache_id(s6, "busybox")        # ... which had taken its seed before the insertion
    s9 = ctx_crc.copy_step_cache_id(s8, "COPY", "--from=0 /app /app", c, ["/app"], from_stage="0")
    s10 = ctx_crc.copy_step_cache_id(s9, "COPY", "--from=alpine:3 /bin/sh /sh", c, ["/bin/sh"], from_stage="alpine:3")
    s11 = ctx_crc.copy_step_cache_id(s10, "COPY", "d0/f1.bin link /y/", c, ["d0/f1.bin", "link"])
    s12 = ctx_crc.base_step_cache_id(s11, "RUN", "true", False)
    assert got == [s0, s1, s2, s3, s4, s5, s6, r7, s8, s9, s10, s11, s12]
    assert s9 == "%x" % zlib.crc32((s8 + "COPY" + "--from=0 /app /app").encode())  # COPY --from hashes no content


def test_seed_chain_through_short_hex_ids(tmp_path):
    """%x has no zero padding: an ID below 0x10000000 makes the next prefix shorter.  Find RUN args that force one."""
    c = _ctx(str(tmp_path))
    seed = ctx_crc.plan_seed(True, False)
    s0 = ctx_crc.from_step_cache_id(seed, "scratch")
    k = next(k for k in range(10_000) if len(ctx_crc.base_step_cache_id(s0, "RUN", "echo %d" % k, True)) < 7)
    steps = [PlanStep.from_image("scratch"), PlanStep.base("RUN", "echo %d" % k, True),
             PlanStep.copy("COPY", ". /app/", ["."]), PlanStep.base("RUN", "true", True)]
    ids = plan_oracle.plan_cache_ids(seed, c, steps)
    assert len(ids[1]) < 7
    assert ids[2] == ctx_crc.copy_step_cache_id(ids[1], "COPY", ". /app/", c, ["."])
    assert ids[2] != ctx_crc.copy_step_cache_id(ids[1].rjust(8, "0"), "COPY", ". /app/", c, ["."])
    # the engine's prepend arithmetic over the short prefix, from pure(rest) and len(rest)
    rest = b"".join(os.fsencode(s.data) if s.kind == "bytes" else open(s.path, "rb").read()
                    for s in ctx_crc.context_segments(c, ["."]))
    pure_rest = zlib.crc32(rest) ^ zlib.crc32(bytes(len(rest)))
    assert "%x" % abi.crc_prepend((ids[1] + "COPY. /app/").encode(), pure_rest, len(rest)) == ids[2]


def test_crc_prepend_matches_zlib():
    rng = np.random.default_rng(3)
    for n_pre, n_rest in [(0, 0), (0, 5), (7, 0), (1, 1), (40, 1000), (300, 70_000)]:
        pre, rest = rng.bytes(n_pre), rng.bytes(n_rest)
        pure_rest = zlib.crc32(rest) ^ zlib.crc32(bytes(n_rest))
        assert abi.crc_prepend(pre, pure_rest, n_rest) == zlib.crc32(pre + rest)
    # len(rest) beyond 2^32: rest = 0^L has pure value 0 and crc(0^L) = 0xFFFFFFFF * x^(8L) ^ 0xFFFFFFFF
    import oracle.lib as olib
    o = olib.L()
    L = (1 << 32) + 12345
    crc_zeros = o.mko_crc32_mulmod(0xFFFFFFFF, o.mko_crc32_xpow8n(L)) ^ 0xFFFFFFFF
    assert abi.crc_prepend(b"seedCOPYx", 0, L) == o.mko_crc32_combine(zlib.crc32(b"seedCOPYx"), crc_zeros, L)


# ---------------------------------------------------------------------------------------------------------------
# host plan logic under the mock engine
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scenario", ["ids_and_bytes_sent", "warm_cache_and_one_touched_file", "more_steps_than_stream_slots",
                                      "extent_table_overrun_is_an_error"])
def test_plan_against_the_mock_engine(tmp_path, scenario):
    r = mock_engine.run("tests.test_host_plan_cache_ids_cpu", scenario, tmp_path)
    assert "SCENARIO-OK" in r.stdout, r.stdout[-3000:]


def _engine(factory, arena=1 << 20, max_extents=1 << 10):
    return factory(arena, n_host_arenas=2, max_extents=max_extents)


def ids_and_bytes_sent(factory, tmp):
    from makisu_b200 import host
    c = _ctx(tmp, big=3_000_000)  # larger than the 1 MiB arena, covered by two steps
    seed = ctx_crc.plan_seed(True, False)
    steps = _plan()
    eng = _engine(factory, max_extents=16)  # fold in pieces of 16 uses, many submits
    ids, st = host.plan_cache_ids(eng, seed, c, steps, n_threads=3)
    assert ids == plan_oracle.plan_cache_ids(seed, c, steps)
    assert st["bytes_sent"] == plan_oracle.unique_file_bytes(c, steps)
    occ = [g for s in steps if s.kind == 1 and not s.from_stage for g in ctx_crc.context_segments(c, list(s.from_paths))
           if g.kind == "file"]
    assert st["files_total"] == len(occ) and st["bytes_total"] == sum(g.size for g in occ) > st["bytes_sent"]
    assert st["files_reused"] == 0
    # every COPY step on its own, through the single-step entry point, agrees
    for i, s in enumerate(steps):
        if s.kind == 1 and not s.from_stage:
            crc, _ = host.context_crc32(eng, (ids[i - 1] + s.directive + s.args).encode(), c, list(s.from_paths))
            assert "%x" % crc == ids[i]
    # a missing source fails like the single-step call does
    bad = steps[:3] + [PlanStep.copy("COPY", "nope /x", ["nope"])]
    try:
        host.plan_cache_ids(eng, seed, c, bad)
        raise AssertionError("missing source accepted")
    except host.HostError as e:
        assert str(e).startswith("hash context sources: ") and "nope" in str(e), e


def warm_cache_and_one_touched_file(factory, tmp):
    from makisu_b200 import host
    c = _ctx(tmp)
    seed = ctx_crc.plan_seed(True, False)
    steps = [PlanStep.from_image("scratch"), PlanStep.copy("COPY", ". /app/", ["."]), PlanStep.copy("COPY", "d0 /d0/", ["d0"]),
             PlanStep.copy("COPY", "d0/f1.bin /x", ["d0/f1.bin"]), PlanStep.base("RUN", "true", True)]
    eng = _engine(factory)
    cache = host.CrcCache()
    ids, st = host.plan_cache_ids(eng, seed, c, steps, cache=cache)
    assert ids == plan_oracle.plan_cache_ids(seed, c, steps)
    assert st["bytes_sent"] == plan_oracle.unique_file_bytes(c, steps) and len(cache) > 0
    ids2, st2 = host.plan_cache_ids(eng, seed, c, steps, cache=cache)
    empties = sum(1 for s in steps[1:4] for g in ctx_crc.context_segments(c, list(s.from_paths)) if g.kind == "file" and not g.size)
    assert ids2 == ids and st2["bytes_sent"] == 0 and st2["files_reused"] == st2["files_total"] - empties  # nothing to cache
    # the single-step cached entry point reads the same remembered values
    crc, _, st3 = cache.context_crc32(eng, (ids[2] + "COPY" + "d0/f1.bin /x").encode(), c, ["d0/f1.bin"])
    assert "%x" % crc == ids[3] and st3["bytes_sent"] == 0
    # rewrite one file that three steps cover: it alone travels, once
    p = os.path.join(c, "d0", "f1.bin")
    size = os.path.getsize(p)
    with open(p, "wb") as f:
        f.write(np.random.default_rng(99).bytes(size))
    ids3, st4 = host.plan_cache_ids(eng, seed, c, steps, cache=cache)
    assert ids3 == plan_oracle.plan_cache_ids(seed, c, steps) and ids3[1:4] != ids[1:4]
    assert st4["bytes_sent"] == size
    ids4, st5 = host.plan_cache_ids(eng, seed, c, steps, cache=cache)
    assert ids4 == ids3 and st5["bytes_sent"] == 0


def more_steps_than_stream_slots(factory, tmp):
    from makisu_b200 import host
    c = _ctx(tmp)
    seed = ctx_crc.plan_seed(False, True)
    dirs = ["d0", "d1", "d2", "d0/f1.bin", "link", "requirements.txt"]
    steps = [PlanStep.from_image("scratch")] + [PlanStep.copy("COPY", "%s /s%d/" % (d, i), [d]) for i, d in enumerate(dirs * 2)]
    eng = _engine(factory, max_extents=8)  # 8 stream slots: 12 COPY steps need two sessions
    before = eng.submits()
    ids, st = host.plan_cache_ids(eng, seed, c, steps)
    assert ids == plan_oracle.plan_cache_ids(seed, c, steps)
    assert st["bytes_sent"] == plan_oracle.unique_file_bytes(c, steps)  # the second session reads nothing again
    assert eng.submits() > before


def extent_table_overrun_is_an_error(factory, tmp):
    """More unique segments in one session than the per-extent table keeps (the mock keeps 4 * max_extents values):
    a capacity error, never IDs folded from values that were not kept."""
    from makisu_b200 import host
    c = os.path.join(tmp, "many")
    for i in range(60):
        _mk(c, "f%03d" % i, b"x" * (i + 1))
    eng = _engine(factory, max_extents=16)
    seed = ctx_crc.plan_seed(True, False)
    try:
        host.plan_cache_ids(eng, seed, c, [PlanStep.from_image("scratch"), PlanStep.copy("COPY", ". /", ["."])])
        raise AssertionError("plan beyond the per-extent table accepted")
    except host.HostError as e:
        assert "crc fold" in str(e) and "per-extent table" in str(e), e
    # the handle is usable afterwards
    small = os.path.join(tmp, "small")
    _mk(small, "a", b"abc")
    steps = [PlanStep.from_image("scratch"), PlanStep.copy("COPY", "a /a", ["a"])]
    assert host.plan_cache_ids(eng, seed, small, steps)[0] == plan_oracle.plan_cache_ids(seed, small, steps)


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=True)
    from tests.mock_engine.scenarios import MockEngineFactory
    globals()[scenario](MockEngineFactory(mock), tmp)
    print("SCENARIO-OK", scenario)


if __name__ == "__main__":
    main()
