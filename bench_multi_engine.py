#!/usr/bin/env python
"""bench_multi_engine.py -- libmkhost driving one engine against N engines: the bench_commit_layers.py workload
(--files x --file-kib on tmpfs as one `COPY dNNN /app/dNNN/` layer per directory, all layers in one batch, TarDigest on
the device, no tar_fd, no cache) through mkhost_memfs_commit_layers_multi, and the cacheID of the same context
(`COPY . /app/`, no cache) through mkhost_context_crc32_multi.

  python bench_multi_engine.py [--files 16384] [--file-kib 512] [--dirs 256] [--reps 3] [--engines N]

N engines sit one per device when the machine has N devices (N defaults to the device count, at least 2).  With fewer
devices than engines they share devices round robin: on one GPU that measures the cost of sharding (threads, sessions,
the table merge), not scaling, and the JSON says so.  Per operation, 1 engine and N engines run alternately, one
warm-up each, then best of --reps; the outputs of both must be equal (every layer's TarDigest, root, n_chunks,
n_unique; the cacheID and stream length).  Kernel time per device comes from one torch.profiler run of each leg.
Prints one JSON line with the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_plan import gpu_identity  # noqa: E402


def kernel_ms_per_device(fn) -> dict | None:
    """CUDA kernel time of one call of fn per device index, from torch.profiler (None if the profiler is unavailable)."""
    try:
        from torch.autograd import DeviceType
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        out = {}
        for e in prof.events():
            if e.device_type == DeviceType.CUDA:
                out[str(e.device_index)] = out.get(str(e.device_index), 0.0) + e.time_range.elapsed_us() / 1e3
        return out
    except Exception:  # noqa: BLE001  (informational)
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=16384)
    ap.add_argument("--file-kib", type=int, default=512)
    ap.add_argument("--dirs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--arena-mib", type=int, default=1024)
    ap.add_argument("--engines", type=int, default=0, help="N (default: the device count, at least 2)")
    ap.add_argument("--fs-dir", default="/dev/shm")
    args = ap.parse_args()

    import torch

    from makisu_b200 import host
    from makisu_b200.abi import Engine

    n_dev = torch.cuda.device_count()
    if n_dev < 1:
        raise SystemExit("no CUDA device")
    n_eng = args.engines or max(2, n_dev)
    fb, n_files, n_dirs = args.file_kib << 10, args.files, args.dirs
    base = os.path.join(args.fs_dir, "mkbench_multi_engine_%d" % os.getpid())
    ctx = os.path.join(base, "ctx")
    threads = max(1, min(len(os.sched_getaffinity(0)), args.threads))
    arena = args.arena_mib << 20
    total = n_files * fb
    rng = np.random.default_rng(5)
    try:
        for d in range(n_dirs):
            os.makedirs(os.path.join(ctx, "d%03d" % d))
        for i in range(n_files):
            with open(os.path.join(ctx, "d%03d" % (i * n_dirs // n_files), "f%06d.bin" % i), "wb") as f:
                f.write(rng.bytes(fb))
        for d, _, _ in os.walk(ctx):
            os.utime(d, (1_500_000_000, 1_500_000_000))
        layers = [[host.CopyOperation(["/d%03d" % d], ctx, "/", "/app/d%03d/" % d)] for d in range(n_dirs)]

        def engine(device):
            return Engine(device=device, device_arena_bytes=arena, n_host_arenas=4, host_arena_bytes=arena,
                          n_device_slots=2, max_extents=1 << 16, max_chunks=total // 4096 + n_files + (1 << 16))

        single = [engine(0)]
        multi = [engine(k % n_dev) for k in range(n_eng)]
        k = [0]

        def commit(engines):
            k[0] += 1
            root = os.path.join(base, "root%d" % k[0])
            os.mkdir(root)
            fs = host.MemFS(root)
            try:
                outs, _ = fs.commit_layers_multi(engines, None, 1_600_000_000, layers, threads)
                return [(o["tar_digest"], o["root"], o["n_chunks"], o["n_unique"]) for o in outs]
            finally:
                fs.close()
                os.rmdir(root)

        def cache_id(engines):
            crc, slen, _ = host.context_crc32_multi(engines, b"seedCOPY. /app/", ctx, ["."], threads)
            return crc, slen

        out = {"bench": "multi_engine", "gpu": gpu_identity(), "devices": n_dev, "engines": n_eng,
               "engine_devices": [k % n_dev for k in range(n_eng)], "files": n_files, "file_kib": args.file_kib,
               "layers": n_dirs, "context_GiB": total / 2 ** 30, "host_threads_per_engine": threads,
               "arena_MiB": args.arena_mib,
               "measures": "scaling over devices" if n_dev >= n_eng else
                           "overhead of sharding (engines share %d device(s)), not scaling" % n_dev}
        for op, fn in (("commit_layers_tar_digest", commit), ("cache_id", cache_id)):
            legs = {"1": single, str(n_eng): multi}
            want = fn(single)
            for name, engs in legs.items():  # gate and warm-up
                assert fn(engs) == want, (op, name)
            runs = {name: [] for name in legs}
            for _ in range(args.reps):  # alternating
                for name, engs in legs.items():
                    t0 = time.perf_counter()
                    got = fn(engs)
                    runs[name].append(time.perf_counter() - t0)
                    assert got == want, (op, name)
            res = {}
            for name, engs in legs.items():
                best = min(runs[name])
                res[name] = {"s": best, "runs_s": runs[name], "GiB_per_s": total / 2 ** 30 / best,
                             "kernel_ms_per_device": kernel_ms_per_device(lambda: fn(engs))}
            res["speedup"] = min(runs["1"]) / min(runs[str(n_eng)])
            out[op] = res
        out["gate"] = ("every layer's TarDigest, root, n_chunks, n_unique and the cacheID with its stream length equal "
                       "between 1 and N engines, in every timed run")
        print(json.dumps(out))
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
