"""GPU: cacheIDs of a whole build plan in one engine session (mkhost_plan_cache_ids, k_crc_fold)."""
import json
import os
import zlib

import numpy as np
import pytest

from makisu_b200 import abi, host
from makisu_b200.abi import MKSNAP_U_VALUE, MKSNAP_X_CRC, CrcUse, Engine, Extent, MksnapError
from makisu_b200.host import PlanStep
from oracle import ctx_crc
from oracle import lib as olib
from tests import plan_oracle, plan_reference_contexts

pytestmark = pytest.mark.gpu
T = 1_500_000_000
ARENA = 4 << 20


def _mk(root, rel, data=b""):
    p = os.path.join(root, rel)
    os.makedirs(os.path.dirname(p), exist_ok=True)
    with open(p, "wb") as f:
        f.write(data)
    os.utime(p, (T, T))
    return p


def _random_ctx(root, seed):
    rng = np.random.default_rng(seed)
    _mk(root, "Dockerfile", b"FROM scratch\n")
    _mk(root, "big/huge.bin", rng.bytes(10 * ARENA // 4 + 12345))  # larger than the arena, in two steps
    for i in range(3000):
        _mk(root, "small/s%02d/f%04d" % (i % 37, i), rng.bytes(int(rng.integers(0, 700))))
    for i in range(20):
        _mk(root, "mixed/e%02d" % i, b"")
        os.makedirs(os.path.join(root, "mixed", "dir%02d" % i), exist_ok=True)
        os.symlink("../small/s01", os.path.join(root, "mixed", "l%02d" % i))
    os.mkfifo(os.path.join(root, "mixed", "fifo"))  # skipped by the walk
    return [PlanStep.from_image("scratch"),
            PlanStep.copy("COPY", "big/huge.bin /h", ["big/huge.bin"]),
            PlanStep.base("RUN", "true", True),
            PlanStep.copy("COPY", ". /app/", ["."]),
            PlanStep.copy("ADD", "small/s0* mixed /x/", ["small/s0*", "mixed"]),
            PlanStep.copy("COPY", "mixed/e00 /e", ["mixed/e00"]),
            PlanStep.copy("COPY", "--from=0 / /", ["/"], from_stage="0"),
            PlanStep.base("ENV", "A=1", False)]


@pytest.fixture(scope="module")
def eng():
    with Engine(device=0, device_arena_bytes=ARENA, n_host_arenas=3, host_arena_bytes=ARENA, max_extents=1 << 12) as e:
        yield e


@pytest.mark.parametrize("seed", [1, 2])
def test_plan_ids_equal_oracle_and_single_steps(eng, tmp_path, seed):
    c = str(tmp_path / "ctx")
    steps = _random_ctx(c, seed)
    sd = ctx_crc.plan_seed(True, False)
    ids, st = host.plan_cache_ids(eng, sd, c, steps, n_threads=4)
    assert ids == plan_oracle.plan_cache_ids(sd, c, steps)
    assert st["bytes_sent"] == plan_oracle.unique_file_bytes(c, steps) < st["bytes_total"]
    for i, s in enumerate(steps):  # one mkhost_context_crc32 per COPY step, chained by the caller
        if s.kind == host.MKHOST_STEP_COPY and not s.from_stage:
            crc, _ = host.context_crc32(eng, (ids[i - 1] + s.directive + s.args).encode(), c, list(s.from_paths))
            assert "%x" % crc == ids[i]


def test_plan_warm_cache_sends_nothing(eng, tmp_path):
    c = str(tmp_path / "ctx")
    steps = _random_ctx(c, 3)
    sd = ctx_crc.plan_seed(True, False)
    cache = host.CrcCache()
    ids, st = host.plan_cache_ids(eng, sd, c, steps, cache=cache)
    ids2, st2 = host.plan_cache_ids(eng, sd, c, steps, cache=cache)
    assert ids2 == ids == plan_oracle.plan_cache_ids(sd, c, steps)
    assert st["bytes_sent"] > 0 and st2["bytes_sent"] == 0 and st2["files_reused"] > 0


def test_plans_of_reference_build_contexts(eng, tmp_path):
    root = plan_reference_contexts.unpack(str(tmp_path))
    want = json.load(open(plan_reference_contexts.GOLDEN))
    sd = plan_reference_contexts.SEED
    assert want["seed"] == sd
    for name, steps in plan_reference_contexts.PLANS.items():
        c = os.path.join(root, name)
        ids, _ = host.plan_cache_ids(eng, sd, c, steps)
        assert ids == want["plans"][name] == plan_oracle.plan_cache_ids(sd, c, steps), name


def _pure(b: bytes) -> int:
    return zlib.crc32(b) ^ zlib.crc32(bytes(len(b)))


def _shift(v: int, nbytes: int) -> int:
    o = olib.L()
    return o.mko_crc32_mulmod(v, o.mko_crc32_xpow8n(nbytes))


def test_crc_fold_kernel_against_oracle_arithmetic(tmp_path):
    rng = np.random.default_rng(11)
    lens = [int(x) for x in rng.integers(0, 5000, 300)] + [1, 0, 70_000]
    data = [rng.bytes(n) for n in lens]
    with Engine(device=0, device_arena_bytes=ARENA, max_extents=1 << 14) as e:
        # extents packed into device slot 0
        arena, exts, pos = bytearray(), [], 0
        for d in data:
            pos = (pos + 15) // 16 * 16
            arena += bytes(pos - len(arena)) + d
            exts.append(Extent(pos, len(d), 0, MKSNAP_X_CRC, 0))
            pos += len(d)
        arena += bytes((-len(arena)) % 512)
        e.device_upload(0, 0, bytes(arena))
        n_streams = 40
        uses, want = [], [0] * n_streams
        big = [(1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 40) + 7, 3 * (1 << 32) - 5]
        for i in range(6000):
            # stream 3 alone spans many warps, the rest interleave; streams 5 and 17 stay empty
            stream = 3 if i < 2500 else int(rng.choice([s for s in range(n_streams) if s not in (5, 17)]))
            suffix = big[i % len(big)] if i % 97 == 0 else int(rng.integers(0, 1 << 20))
            if i % 3 == 0:
                v = int(rng.integers(0, 1 << 32))
                uses.append((suffix, v, stream, MKSNAP_U_VALUE))
            else:
                k = int(rng.integers(0, len(data)))
                v = _pure(data[k])
                uses.append((suffix, k, stream, 0))
            want[stream] ^= _shift(v, suffix)
        for rep in range(2):  # the second session starts from zeroed streams
            e.begin()
            e.device_submit(0, len(arena), exts)
            # invalid src / stream are refused and change nothing
            for bad in [(0, len(data), 0, 0), (0, 0, 1 << 14, 0), (0, 0, 0, 2)]:
                with pytest.raises(MksnapError) as ei:
                    e.crc_fold([bad])
                assert ei.value.code == -1
            with pytest.raises(MksnapError) as ei:
                e.crc_fold((CrcUse * ((1 << 14) + 1))())
            assert ei.value.code == -4
            e.crc_fold(uses[:4000])
            e.crc_fold(uses[4000:])
            e.finish()
            got = [int(x) for x in e.get_crc_streams()]
            assert got == want
            assert got[5] == got[17] == 0
        with pytest.raises(MksnapError) as ei:  # out of sequence
            e.crc_fold(uses[:1])
        assert ei.value.code == -5
        e.begin()
        e.finish()
        assert len(e.get_crc_streams()) == 0
