#!/usr/bin/env python
"""bench_commit_layers.py -- batched incremental layer commit: real files on tmpfs committed as one `COPY dNNN /app/dNNN/`
layer per directory, all layers in one batch, with and without remembered chunk digests
(mkhost_memfs_commit_layers_cached).

  python bench_commit_layers.py [--files 16384] [--file-kib 512] [--dirs 256] [--reps 3]

Modes (--modes, default all four):
  tar_digest            TarDigest on the device (one chain per layer, all advancing together), no tar_fd
  tar_digest_files      the same with MKHOST_FILE_DIGESTS (one more SHA-256 stream per file)
  no_tar_digest         MKHOST_NO_TAR_DIGEST, no tar_fd: a remembered file is not even read
  no_tar_digest_files   the same with MKHOST_FILE_DIGESTS (every file is read and hashed again)
Legs per mode (best of --reps after one warm-up each; every leg commits into a fresh MemFS):
  uncached  mkhost_memfs_commit_layers                          (the batch without a cache)
  cold      the cached entry point with an empty cache          (every file chunked and remembered)
  warm      the same cache, tree unchanged                      (nothing chunked)
  edited    one file rewritten (same size) before each run       (that file chunked)
Per leg: wall seconds, h2d_bytes of the batch (mksnap_stats delta) and device ms (sum of the engine's kernel times in
one profiled run, torch.profiler).  Gate before timing: TarDigest of every layer, root, n_chunks and n_unique of every
cached leg equal the uncached batch of the same tree.  Prints one JSON line with the card's name and power limit."""
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

from bench_commit_cache import device_ms  # noqa: E402
from bench_plan import gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=16384)
    ap.add_argument("--file-kib", type=int, default=512)
    ap.add_argument("--dirs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--arena-mib", type=int, default=1024)
    ap.add_argument("--modes", default="tar_digest,tar_digest_files,no_tar_digest,no_tar_digest_files")
    ap.add_argument("--fs-dir", default="/dev/shm")
    args = ap.parse_args()

    from makisu_b200 import host
    from makisu_b200.abi import Engine

    fb, n_files, n_dirs = args.file_kib << 10, args.files, args.dirs
    base = os.path.join(args.fs_dir, "mkbench_commit_layers_%d" % os.getpid())
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
        layers = [[host.CopyOperation(["/d%03d" % d], ctx, "/", "/app/d%03d/" % d)] for d in range(n_dirs)]

        # max_extents: stream slots for every layer and, with file digests, every file
        with Engine(device=0, device_arena_bytes=arena, n_host_arenas=max(4, (4 << 30) // arena), host_arena_bytes=arena,
                    n_device_slots=2, max_extents=1 << 16, max_chunks=total // 4096 + n_files + (1 << 16)) as eng:
            k = [0]

            def commit(flags, cache):
                k[0] += 1
                root = os.path.join(base, "root%d" % k[0])
                os.mkdir(root)
                fs = host.MemFS(root)
                try:
                    if cache is False:
                        return fs.commit_layers(eng, 1_600_000_000, layers, threads, None, flags), None
                    return fs.commit_layers_cached(eng, cache, 1_600_000_000, layers, threads, None, flags)
                finally:
                    fs.close()
                    os.rmdir(root)

            def rewrite():
                with open(edited, "wb") as f:
                    f.write(rng.bytes(fb))

            def timed(fn):
                h0 = eng.stats().h2d_bytes
                t0 = time.perf_counter()
                out = fn()
                dt = time.perf_counter() - t0
                return dt, eng.stats().h2d_bytes - h0, out

            def key(outs):
                return [(o["tar_digest"], o["root"], o["n_chunks"], o["n_unique"]) for o in outs]

            NTD, FD = host.MKHOST_NO_TAR_DIGEST, host.MKHOST_FILE_DIGESTS
            modes = {"tar_digest": 0, "tar_digest_files": FD, "no_tar_digest": NTD, "no_tar_digest_files": NTD | FD}
            modes = {m: modes[m] for m in args.modes.split(",")}
            out = {"bench": "commit_layers_chunk_cache", "gpu": gpu_identity(), "files": n_files, "file_kib": args.file_kib,
                   "layers": n_dirs, "context_GiB": total / 2 ** 30, "host_threads": threads, "arena_MiB": args.arena_mib}
            for mode, flags in modes.items():
                ref, _ = commit(flags, False)
                cache = host.ChunkCache()
                legs = {
                    "uncached": lambda: commit(flags, False),
                    "cold": lambda: commit(flags, host.ChunkCache()),
                    "warm": lambda: commit(flags, cache),
                }
                # gate: cold and warm equal the uncached batch
                assert key(commit(flags, cache)[0]) == key(ref), (mode, "cold")
                lay, st = commit(flags, cache)
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
                    return commit(flags, cache)

                runs = [timed(edited_run) for _ in range(args.reps + 1)][1:]
                best = min(runs, key=lambda r: r[0])
                rewrite()  # gate: one more edit, against the uncached batch of the edited tree
                want, _ = commit(flags, False)
                assert key(commit(flags, cache)[0]) == key(want), (mode, "edited")
                res["edited"] = {"s": best[0], "runs_s": [r[0] for r in runs], "h2d_bytes": best[1],
                                 "device_ms": device_ms(edited_run), "stats": best[2][1]}
                res["n_chunks"], res["n_unique"] = ref[0]["n_chunks"], ref[0]["n_unique"]
                res["tar_GiB"] = sum(o["tar_bytes"] for o in ref) / 2 ** 30
                out[mode] = res
            out["gate"] = ("TarDigest of every layer, root, n_chunks, n_unique of cold / warm / edited equal the uncached "
                           "batch of the same tree")
        print(json.dumps(out))
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
