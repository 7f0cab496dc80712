#!/usr/bin/env python
"""bench_multi_ingest.py -- a run of layers ingested by one engine against N engines (mkhost_memfs_update_from_tars_multi,
no layer cache, so every layer is read, decoded, hashed and parsed).

Workloads:
  - plain / pgzip: the bench_apply_layers.py run, 16 layers whose tars cycle through 4, 16, 32 and 8 MiB, as plain tars
    and as pgzip blobs (1 MiB members, level 1, MKHOST_GUNZIP);
  - single_member_indexed: the bench_gunzip_index.py layers, 16 single-member level-6 gzip blobs of 64 MiB tars, with a
    gz index cache warmed by one run before anything is timed.

  python bench_multi_ingest.py [--layers 16] [--layer-mib 64] [--reps 3] [--engines N]

N engines sit one per device when the machine has N devices (N defaults to the device count, at least 2).  With fewer
devices than engines they share devices round robin: on one GPU that measures the overhead of sharding and the overlap
of several engines' sessions on one device, not scaling, and the JSON says so.  Per workload, 1 engine and N engines run
alternately, one warm-up each, then best of --reps; every timed run's outputs (DiffID, n_entries, tar_bytes, root,
n_chunks, n_unique of every layer) must equal the first run's.  Kernel time per device comes from one torch.profiler
run of each leg.  Prints one JSON line with the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_multi_engine import kernel_ms_per_device  # noqa: E402
from bench_plan import gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=16)
    ap.add_argument("--layer-mib", type=int, default=64, help="tar size of each single-member layer")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--engines", type=int, default=0, help="N (default: the device count, at least 2)")
    args = ap.parse_args()

    import torch

    import bench_apply_layers as bal
    import bench_gunzip as bgz
    from makisu_b200 import abi, host
    from tests import gzip_corpus as gc

    n_dev = torch.cuda.device_count()
    if n_dev < 1:
        raise SystemExit("no CUDA device")
    n_eng = args.engines or max(2, n_dev)
    tmp = tempfile.mkdtemp(prefix="mkbench_multi_ingest_")
    try:
        tars = [bal.layer_tar(i, bal.SIZES_MIB[i % len(bal.SIZES_MIB)] << 20) for i in range(args.layers)]
        single = [bgz.layer_tar(args.layer_mib << 20, seed=100 + i) for i in range(args.layers)]
        workloads = {
            "plain": ([t for t in tars], 0, False),
            "pgzip": ([gc.pgzip(t, block=1 << 20, level=1) for t in tars], host.MKHOST_GUNZIP, False),
            "single_member_indexed": ([gc.gzip_member(gc.deflate(t, 6), t) for t in single], host.MKHOST_GUNZIP, True),
        }
        tar_bytes = {"plain": sum(map(len, tars)), "pgzip": sum(map(len, tars)),
                     "single_member_indexed": sum(map(len, single))}
        del tars, single

        def engine(device):
            return abi.Engine(device=device, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=64 << 20,
                              max_extents=1 << 14)

        legs = {"1": [engine(0)], str(n_eng): [engine(k % n_dev) for k in range(n_eng)]}
        out = {"bench": "multi_ingest", "gpu": gpu_identity(), "devices": n_dev, "engines": n_eng,
               "engine_devices": [k % n_dev for k in range(n_eng)], "layers": args.layers,
               "measures": "scaling over devices" if n_dev >= n_eng else
                           "overhead of sharding and overlap of %d engines on %d device(s), not scaling" % (n_eng, n_dev)}
        for name, (blobs, g, indexed) in workloads.items():
            paths = []
            for i, b in enumerate(blobs):
                paths.append(os.path.join(tmp, "%s%02d" % (name, i)))
                with open(paths[-1], "wb") as f:
                    f.write(b)
            keys = ["%s%02d" % (name, i) for i in range(len(blobs))]
            gz = host.GzIndexCache() if indexed else None

            def ingest(engines):
                root = tempfile.mkdtemp(dir=tmp)
                fds = [os.open(p, os.O_RDONLY) for p in paths]
                fs = host.MemFS(root)
                try:
                    outs, _, gst = fs.update_from_tars_multi(engines, None, gz, keys, 1_600_000_000,
                                                             [(f, g) for f in fds], 0)
                    return [tuple(sorted(o.items())) for o in outs], gst
                finally:
                    for f in fds:
                        os.close(f)
                    fs.close()
                    shutil.rmtree(root)

            want, _ = ingest(legs["1"])  # fills the gz index cache of the indexed workload
            for engs in legs.values():   # warm-up and gate
                assert ingest(engs)[0] == want, name
            runs = {k: [] for k in legs}
            gz_stats = None
            for _ in range(args.reps):   # alternating
                for k, engs in legs.items():
                    t0 = time.perf_counter()
                    got, gz_stats = ingest(engs)
                    runs[k].append(time.perf_counter() - t0)
                    assert got == want, (name, k)
            res = {"tar_MiB": tar_bytes[name] / 2 ** 20, "blob_MiB": sum(map(len, blobs)) / 2 ** 20}
            if indexed:
                res["gz_stats_last_run"] = gz_stats
            for k, engs in legs.items():
                best = min(runs[k])
                res[k] = {"s": round(best, 4), "runs_s": [round(t, 4) for t in runs[k]],
                          "tar_GiB_per_s": round(tar_bytes[name] / 2 ** 30 / best, 3),
                          "kernel_ms_per_device": kernel_ms_per_device(lambda: ingest(engs))}
            res["speedup"] = round(min(runs["1"]) / min(runs[str(n_eng)]), 3)
            out[name] = res
            print(name, json.dumps(res), file=sys.stderr, flush=True)
        out["gate"] = "every layer's DiffID, n_entries, tar_bytes, root, n_chunks and n_unique equal in every timed run"
        print(json.dumps(out))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
