#!/usr/bin/env python
"""bench_commit_cache.py -- incremental layer commit: one `COPY . /app/` layer from real files on tmpfs, with and without
remembered chunk digests (mkhost_memfs_commit_copy_ops_cached).

  python bench_commit_cache.py [--files 16384] [--file-kib 512] [--dirs 256] [--reps 3]

Modes (--modes, default all three):
  no_tar_digest  MKHOST_NO_TAR_DIGEST, the layer tar written to a pipe (drained by a thread): TarDigest left to the caller
  no_tar_digest_no_fd  the same without a tar_fd (the chunk table alone): a remembered file is not even read
  tar_digest     TarDigest on the device, no tar_fd, over the first --td-dirs directories only: the TarDigest of one layer
                 is one serial SHA-256 chain, far slower than the rest of the commit
Legs per mode (best of --reps after one warm-up each; every leg commits into a fresh MemFS):
  uncached  mkhost_memfs_commit_copy_ops                       (the path without a cache)
  cold      the cached entry point with an empty cache          (every file chunked and remembered)
  warm      the same cache, tree unchanged                      (nothing chunked)
  edited    one file rewritten (same size) before each run       (that file chunked)
Per leg: wall seconds, h2d_bytes of the commit (mksnap_stats delta) and device ms (sum of the engine's kernel times in
one profiled run, torch.profiler).  Gate before timing: root, n_chunks, n_unique and TarDigest of every cached leg equal
the uncached commit of the same tree.  Prints one JSON line with the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_plan import gpu_identity  # noqa: E402


def device_ms(fn) -> float | None:
    """Sum of the CUDA kernel times of one call of fn, from torch.profiler (None if the profiler is unavailable)."""
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        return sum(e.device_time_total for e in prof.key_averages()) / 1e3
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
    ap.add_argument("--td-dirs", type=int, default=2)
    ap.add_argument("--modes", default="no_tar_digest,no_tar_digest_no_fd,tar_digest")
    ap.add_argument("--fs-dir", default="/dev/shm")
    args = ap.parse_args()

    from makisu_b200 import host
    from makisu_b200.abi import Engine

    fb, n_files, n_dirs = args.file_kib << 10, args.files, args.dirs
    base = os.path.join(args.fs_dir, "mkbench_commit_cache_%d" % os.getpid())
    ctx = os.path.join(base, "ctx")
    threads = max(1, min(len(os.sched_getaffinity(0)), args.threads))
    arena = args.arena_mib << 20
    total = n_files * fb
    rng = np.random.default_rng(5)
    edited = os.path.join(ctx, "d%03d" % 0, "f%06d.bin" % 0)
    try:
        for d in range(n_dirs):
            os.makedirs(os.path.join(ctx, "d%03d" % d))
        for i in range(n_files):
            with open(os.path.join(ctx, "d%03d" % (i * n_dirs // n_files), "f%06d.bin" % i), "wb") as f:
                f.write(rng.bytes(fb))
        for d, _, _ in os.walk(ctx):
            os.utime(d, (1_500_000_000, 1_500_000_000))
        ops_all = [host.CopyOperation(["/"], ctx, "/", "/app/")]
        ops_td = [host.CopyOperation(["/d%03d" % d for d in range(args.td_dirs)], ctx, "/", "/app/")]

        with Engine(device=0, device_arena_bytes=arena, n_host_arenas=max(4, (4 << 30) // arena), host_arena_bytes=arena,
                    n_device_slots=2, max_extents=1 << 16, max_chunks=total // 4096 + n_files + (1 << 16)) as eng:
            k = [0]

            def commit(ops, flags, cache, pipe):
                k[0] += 1
                root = os.path.join(base, "root%d" % k[0])
                os.mkdir(root)
                fs = host.MemFS(root)
                fd, drain = -1, None
                if pipe:
                    r, fd = os.pipe()
                    drain = threading.Thread(target=lambda: [None for _ in iter(lambda: os.read(r, 1 << 20), b"")])
                    drain.start()
                try:
                    if cache is False:
                        lay, st = fs.commit_copy_ops(eng, 1_600_000_000, ops, threads, fd, flags), None
                    else:
                        lay, st = fs.commit_copy_ops_cached(eng, cache, 1_600_000_000, ops, threads, fd, flags)
                finally:
                    if pipe:
                        os.close(fd)
                        drain.join()
                        os.close(r)
                    fs.close()
                    os.rmdir(root)
                return lay, st

            def rewrite():
                with open(edited, "wb") as f:
                    f.write(rng.bytes(fb))

            def timed(fn):
                h0 = eng.stats().h2d_bytes
                t0 = time.perf_counter()
                out = fn()
                dt = time.perf_counter() - t0
                return dt, eng.stats().h2d_bytes - h0, out

            modes = {"no_tar_digest": (ops_all, host.MKHOST_NO_TAR_DIGEST, True),
                     "no_tar_digest_no_fd": (ops_all, host.MKHOST_NO_TAR_DIGEST, False), "tar_digest": (ops_td, 0, False)}
            modes = {m: modes[m] for m in args.modes.split(",")}
            out = {"bench": "commit_chunk_cache", "gpu": gpu_identity(), "files": n_files, "file_kib": args.file_kib,
                   "dirs": n_dirs, "context_GiB": total / 2 ** 30, "host_threads": threads, "arena_MiB": args.arena_mib}
            for mode, (ops, flags, pipe) in modes.items():
                key = lambda lay: (lay["root"], lay["n_chunks"], lay["n_unique"], lay["tar_digest"])  # noqa: E731
                ref, _ = commit(ops, flags, False, pipe)
                cache = host.ChunkCache()
                legs = {
                    "uncached": lambda: commit(ops, flags, False, pipe),
                    "cold": lambda: commit(ops, flags, host.ChunkCache(), pipe),
                    "warm": lambda: commit(ops, flags, cache, pipe),
                }
                # gate: cold and warm equal the uncached commit
                assert key(commit(ops, flags, cache, pipe)[0]) == key(ref), (mode, "cold")
                lay, st = commit(ops, flags, cache, pipe)
                assert key(lay) == key(ref) and st["bytes_chunked"] == 0, (mode, "warm", st)
                res = {}
                for leg, fn in legs.items():
                    fn()  # warm-up
                    runs = [timed(fn) for _ in range(args.reps)]
                    best = min(runs, key=lambda r: r[0])
                    res[leg] = {"s": best[0], "runs_s": [r[0] for r in runs], "h2d_bytes": best[1],
                                "device_ms": device_ms(fn), "stats": best[2][1]}

                def edited_run():
                    rewrite()
                    return commit(ops, flags, cache, pipe)

                runs = [timed(edited_run) for _ in range(args.reps + 1)][1:]
                best = min(runs, key=lambda r: r[0])
                rewrite()  # gate: one more edit, against the uncached commit of the edited tree
                want, _ = commit(ops, flags, False, pipe)
                assert key(commit(ops, flags, cache, pipe)[0]) == key(want), (mode, "edited")
                res["edited"] = {"s": best[0], "runs_s": [r[0] for r in runs], "h2d_bytes": best[1],
                                 "device_ms": device_ms(edited_run), "stats": best[2][1]}
                res["n_chunks"], res["n_unique"] = ref["n_chunks"], ref["n_unique"]
                res["layer_GiB"] = ref["tar_bytes"] / 2 ** 30
                out[mode] = res
            out["gate"] = "root, n_chunks, n_unique, TarDigest of cold / warm / edited equal the uncached commit of the same tree"
        print(json.dumps(out))
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
