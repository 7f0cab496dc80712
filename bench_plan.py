#!/usr/bin/env python
"""bench_plan.py -- cacheIDs of every step of a build plan, from real files on tmpfs.

  python bench_plan.py [--files 16384] [--file-kib 512] [--dirs 256] [--reps 3]

Plan: FROM scratch, COPY . /app/, one COPY dNNN /app/dNNN/ per directory, RUN true -- every file is hashed by two steps.
Legs (best of --reps after one warm-up each):
  a_per_step_s   one mkhost_context_crc32 per COPY step, chained by the caller (the path without a plan call)
  b_plan_cold_s  mkhost_plan_cache_ids without a cache: each file read and sent once
  c_plan_warm_s  the same call with a warm cache: no file bytes sent
  fold_ms        k_crc_fold alone over as many uses as the plan makes, host clock around fold + device synchronize
Gate before timing: the per-step IDs of (a), (b) and (c) are equal, and equal to the oracle on a two-directory sub-plan.
Prints one JSON line with the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def gpu_identity() -> dict:
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = [x.strip() for x in r.stdout.strip().split(",")]
        out.update(power_limit_w=float(pl), sm_max_mhz=int(mx))
    except Exception:  # noqa: BLE001  (informational)
        out.update(power_limit_w=None, sm_max_mhz=None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=16384)
    ap.add_argument("--file-kib", type=int, default=512)
    ap.add_argument("--dirs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--arena-mib", type=int, default=1024)
    ap.add_argument("--fs-dir", default="/dev/shm")
    args = ap.parse_args()

    from makisu_b200 import host
    from makisu_b200.abi import CrcUse, Engine, MKSNAP_U_VALUE
    from makisu_b200.host import PlanStep
    from oracle import ctx_crc
    from tests import plan_oracle

    fb, n_files, n_dirs = args.file_kib << 10, args.files, args.dirs
    base = os.path.join(args.fs_dir, "mkbench_plan_%d" % os.getpid())
    ctx = os.path.join(base, "ctx")
    threads = max(1, min(len(os.sched_getaffinity(0)), args.threads))
    arena = args.arena_mib << 20
    try:
        rng = np.random.default_rng(5)
        for d in range(n_dirs):
            os.makedirs(os.path.join(ctx, "d%03d" % d))
        for i in range(n_files):
            with open(os.path.join(ctx, "d%03d" % (i * n_dirs // n_files), "f%06d.bin" % i), "wb") as f:
                f.write(rng.bytes(fb))
        for d, _, _ in os.walk(ctx):
            os.utime(d, (1_500_000_000, 1_500_000_000))
        seed = ctx_crc.plan_seed(True, False)
        dirs = ["d%03d" % d for d in range(n_dirs)]
        steps = ([PlanStep.from_image("scratch"), PlanStep.copy("COPY", ". /app/", ["."])] +
                 [PlanStep.copy("COPY", "%s /app/%s/" % (d, d), [d]) for d in dirs] + [PlanStep.base("RUN", "true", True)])
        n_uses = sum(1 for s in steps if s.kind == host.MKHOST_STEP_COPY for _ in ctx_crc.context_segments(ctx, list(s.from_paths)))

        with Engine(device=0, device_arena_bytes=arena, n_host_arenas=max(4, (4 << 30) // arena), host_arena_bytes=arena,
                    n_device_slots=2, max_extents=1 << 16) as eng:
            def per_step():
                ids, sd = [], seed
                for s in steps:
                    if s.kind == host.MKHOST_STEP_COPY:
                        crc, _ = host.context_crc32(eng, (sd + s.directive + s.args).encode(), ctx, list(s.from_paths), threads)
                        cid = "%x" % crc
                    elif s.kind == host.MKHOST_STEP_FROM:
                        cid = ctx_crc.from_step_cache_id(sd, s.args)
                    else:
                        cid = ctx_crc.base_step_cache_id(sd, s.directive, s.args, s.commit)
                    ids.append(cid)
                    sd = cid
                return ids

            # gate: oracle on a two-directory sub-plan, then (a) == (b) == (c) on the whole plan
            sub = steps[:1] + [PlanStep.copy("COPY", "%s /app/%s/" % (d, d), [d]) for d in dirs[:2]] + steps[-1:]
            want_sub = plan_oracle.plan_cache_ids(seed, ctx, sub)
            got_sub, _ = host.plan_cache_ids(eng, seed, ctx, sub, threads)
            assert got_sub == want_sub, ("oracle gate", got_sub, want_sub)
            cache = host.CrcCache()
            ids_a = per_step()
            ids_b, st_b = host.plan_cache_ids(eng, seed, ctx, steps, threads)
            ids_c0, _ = host.plan_cache_ids(eng, seed, ctx, steps, threads, cache=cache)
            ids_c, st_c = host.plan_cache_ids(eng, seed, ctx, steps, threads, cache=cache)
            assert ids_a == ids_b == ids_c0 == ids_c, "per-step IDs differ between the legs"
            assert st_c["bytes_sent"] == 0, st_c

            def best(fn):
                fn()  # warm-up
                t = []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    fn()
                    t.append(time.perf_counter() - t0)
                return min(t), t

            a_s, a_all = best(per_step)
            b_s, b_all = best(lambda: host.plan_cache_ids(eng, seed, ctx, steps, threads))
            c_s, c_all = best(lambda: host.plan_cache_ids(eng, seed, ctx, steps, threads, cache=cache))

            # the fold alone: as many uses as the plan folds, immediate values, grouped by stream like the host emits them
            per = max(1, n_uses // (n_dirs + 1))
            uses = (CrcUse * n_uses)()
            for i in range(n_uses):
                uses[i].suffix, uses[i].src, uses[i].stream, uses[i].flags = i * 4096, i * 2654435761 & 0xFFFFFFFF, min(i // per, n_dirs), MKSNAP_U_VALUE

            def fold_timed():
                eng.begin()
                t0 = time.perf_counter()
                for u0 in range(0, n_uses, 1 << 16):
                    n = min(1 << 16, n_uses - u0)
                    eng.crc_fold((CrcUse * n).from_buffer(uses, 24 * u0))
                eng.sync()
                dt = time.perf_counter() - t0
                eng.finish()
                return dt

            fold_timed()
            fold_ms = 1e3 * min(fold_timed() for _ in range(5))

        total = n_files * fb
        out = {"bench": "plan_cache_ids", "gpu": gpu_identity(), "files": n_files, "file_kib": args.file_kib, "dirs": n_dirs,
               "steps": len(steps), "copy_steps": n_dirs + 1, "context_GiB": total / 2 ** 30, "host_threads": threads,
               "arena_MiB": args.arena_mib, "uses": n_uses,
               "gate": "per-step IDs of (a), (b), (c) equal; 2-directory sub-plan equals the oracle",
               "a_per_step_s": a_s, "b_plan_cold_s": b_s, "c_plan_warm_s": c_s,
               "a_runs_s": a_all, "b_runs_s": b_all, "c_runs_s": c_all,
               "a_bytes_read": 2 * total, "a_bytes_sent": 2 * total,
               "b_bytes_read": st_b["bytes_sent"], "b_bytes_sent": st_b["bytes_sent"],
               "c_bytes_read": st_c["bytes_sent"], "c_bytes_sent": st_c["bytes_sent"],
               "fold_ms": fold_ms, "fold_note": "k_crc_fold over %d immediate uses incl. the 24 B/use upload, host clock to sync" % n_uses,
               "last_cache_id": ids_b[-1]}
        print(json.dumps(out))
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
