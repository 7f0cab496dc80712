"""ctypes binding of libmkhost.so (include/mkhost.h): the C++ host side above the mksnap C-ABI.

Mirrors the reference names: context_crc32 ~ addCopyStep.SetCacheID, commit_copy_ops ~ commitLayer over
MemFS.AddLayerByCopyOps, encode_tar_header ~ tario.WriteHeader.  No hashing happens here or in libmkhost.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Sequence

from . import abi

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libmkhost.so"


class TarHeader(C.Structure):
    _fields_ = [("name", C.c_char_p), ("linkname", C.c_char_p), ("mode", C.c_int64), ("uid", C.c_int64),
                ("gid", C.c_int64), ("size", C.c_int64), ("mtime_ns", C.c_int64), ("typeflag", C.c_char)]


class CopyOp(C.Structure):
    _fields_ = [("src_root", C.c_char_p), ("srcs", C.POINTER(C.c_char_p)), ("n_srcs", C.c_size_t),
                ("work_dir", C.c_char_p), ("dst", C.c_char_p), ("uid", C.c_int32), ("gid", C.c_int32)]


class CrcCacheStats(C.Structure):
    _fields_ = [("files_total", C.c_uint64), ("files_reused", C.c_uint64), ("bytes_total", C.c_uint64), ("bytes_sent", C.c_uint64)]


class ChunkCacheStats(C.Structure):
    _fields_ = [("files_total", C.c_uint64), ("files_reused", C.c_uint64), ("bytes_total", C.c_uint64),
                ("bytes_chunked", C.c_uint64), ("bytes_uploaded", C.c_uint64)]


class GzIndexStats(C.Structure):
    _fields_ = [("blobs", C.c_uint64), ("blobs_with_index", C.c_uint64), ("points_given", C.c_uint64),
                ("points_linked", C.c_uint64), ("points_recorded", C.c_uint64)]


class LayerCacheStats(C.Structure):
    _fields_ = [("layers", C.c_uint64), ("layers_replayed", C.c_uint64), ("layers_recorded", C.c_uint64),
                ("blob_bytes_read", C.c_uint64), ("chunks_appended", C.c_uint64)]


class LayerSpec(C.Structure):
    _fields_ = [("ops", C.POINTER(CopyOp)), ("n_ops", C.c_size_t), ("tar_fd", C.c_int)]


class LayerResult(C.Structure):
    _fields_ = [("tar_digest", C.c_uint8 * 32), ("root", C.c_uint8 * 32), ("n_entries", C.c_uint64),
                ("tar_bytes", C.c_uint64), ("n_chunks", C.c_uint64), ("n_unique", C.c_uint64)]


class TarSpec(C.Structure):
    _fields_ = [("tar_fd", C.c_int), ("flags", C.c_uint32)]


class _PlanStep(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("commit", C.c_int32), ("directive", C.c_char_p), ("args", C.c_char_p),
                ("from_stage", C.c_char_p), ("from_paths", C.POINTER(C.c_char_p)), ("n_paths", C.c_size_t)]


_P = C.c_void_p
SYMBOLS = [
    ("mkhost_encode_tar_header", C.c_size_t, [C.POINTER(TarHeader), _P, C.c_size_t]),
    ("mkhost_context_crc32", C.c_int, [_P, _P, C.c_size_t, C.c_char_p, C.POINTER(C.c_char_p), C.c_size_t, C.c_int,
                                       C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]),
    ("mkhost_crc_cache_new", _P, []),
    ("mkhost_crc_cache_free", None, [_P]),
    ("mkhost_crc_cache_size", C.c_uint64, [_P]),
    ("mkhost_crc_cache_save", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_crc_cache_load", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_context_crc32_cached", C.c_int, [_P, _P, _P, C.c_size_t, C.c_char_p, C.POINTER(C.c_char_p), C.c_size_t, C.c_int,
                                              C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(CrcCacheStats), C.c_char_p,
                                              C.c_size_t]),
    ("mkhost_plan_cache_ids", C.c_int, [_P, _P, C.c_char_p, C.c_char_p, C.POINTER(_PlanStep), C.c_size_t, C.c_int,
                                        C.POINTER(C.c_uint32), C.POINTER(CrcCacheStats), C.c_char_p, C.c_size_t]),
    ("mkhost_commit_copy_ops", C.c_int, [_P, C.c_char_p, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_int,
                                         C.POINTER(LayerResult), C.c_char_p, C.c_size_t]),
    ("mkhost_commit_copy_ops_to_fd", C.c_int, [_P, C.c_char_p, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_int, C.c_int,
                                               C.POINTER(LayerResult), C.c_char_p, C.c_size_t]),
    ("mkhost_commit_copy_ops_ex", C.c_int, [_P, C.c_char_p, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_int, C.c_int,
                                            C.c_uint32, C.POINTER(LayerResult), C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_new", _P, [C.c_char_p, C.POINTER(C.c_char_p), C.c_size_t, C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_free", None, [_P]),
    ("mkhost_memfs_file_digest", C.c_int, [_P, C.c_char_p, C.POINTER(C.c_uint8)]),
    ("mkhost_memfs_commit_copy_ops", C.c_int, [_P, _P, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_int, C.c_int, C.c_uint32,
                                               C.POINTER(LayerResult), C.c_char_p, C.c_size_t]),
    ("mkhost_chunk_cache_new", _P, []),
    ("mkhost_chunk_cache_free", None, [_P]),
    ("mkhost_chunk_cache_size", C.c_uint64, [_P]),
    ("mkhost_chunk_cache_save", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_chunk_cache_load", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_commit_copy_ops_cached", C.c_int, [_P, _P, _P, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_int, C.c_int,
                                                      C.c_uint32, C.POINTER(LayerResult), C.POINTER(ChunkCacheStats),
                                                      C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_commit_layers", C.c_int, [_P, _P, C.c_int64, C.POINTER(LayerSpec), C.c_size_t, C.c_int, C.c_uint32,
                                             C.POINTER(LayerResult), C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_commit_layers_cached", C.c_int, [_P, _P, _P, C.c_int64, C.POINTER(LayerSpec), C.c_size_t, C.c_int,
                                                    C.c_uint32, C.POINTER(LayerResult), C.POINTER(ChunkCacheStats),
                                                    C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_commit_scan", C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, C.c_uint32, C.POINTER(LayerResult),
                                           C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_describe_copy_ops", C.c_size_t, [_P, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_char_p, C.c_size_t,
                                                    C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_describe_scan", C.c_size_t, [_P, C.c_int64, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_update_from_tar", C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_uint32, C.POINTER(LayerResult), C.c_char_p,
                                               C.c_size_t]),
    ("mkhost_memfs_describe_update_from_tar_ex", C.c_size_t, [_P, C.c_int64, C.c_int, C.c_uint32, C.c_char_p, C.c_size_t,
                                                              C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_describe_update_from_tar", C.c_size_t, [_P, C.c_int64, C.c_int, C.c_char_p, C.c_size_t, C.c_char_p,
                                                           C.c_size_t]),
    ("mkhost_memfs_update_from_tars", C.c_int, [_P, _P, C.c_int64, C.POINTER(TarSpec), C.c_size_t, C.c_uint32,
                                                C.POINTER(LayerResult), C.c_char_p, C.c_size_t]),
    ("mkhost_gz_index_cache_new", _P, []),
    ("mkhost_gz_index_cache_free", None, [_P]),
    ("mkhost_gz_index_cache_size", C.c_uint64, [_P]),
    ("mkhost_gz_index_cache_save", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_gz_index_cache_load", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_update_from_tar_indexed", C.c_int, [_P, _P, _P, C.c_char_p, C.c_int64, C.c_int, C.c_uint32,
                                                       C.POINTER(LayerResult), C.POINTER(GzIndexStats), C.c_char_p,
                                                       C.c_size_t]),
    ("mkhost_memfs_update_from_tars_indexed", C.c_int, [_P, _P, _P, C.POINTER(C.c_char_p), C.c_int64,
                                                        C.POINTER(TarSpec), C.c_size_t, C.c_uint32,
                                                        C.POINTER(LayerResult), C.POINTER(GzIndexStats), C.c_char_p,
                                                        C.c_size_t]),
    ("mkhost_layer_cache_new", _P, []),
    ("mkhost_layer_cache_free", None, [_P]),
    ("mkhost_layer_cache_size", C.c_uint64, [_P]),
    ("mkhost_layer_cache_save", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_layer_cache_load", C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_memfs_update_from_tars_cached", C.c_int, [_P, _P, _P, _P, C.POINTER(C.c_char_p), C.c_int64,
                                                       C.POINTER(TarSpec), C.c_size_t, C.c_uint32, C.POINTER(LayerResult),
                                                       C.POINTER(LayerCacheStats), C.POINTER(GzIndexStats), C.c_char_p,
                                                       C.c_size_t]),
    ("mkhost_copy_op_execute", C.c_int, [C.POINTER(CopyOp), C.c_uint32, C.POINTER(C.c_char_p), C.c_size_t, C.c_char_p, C.c_size_t]),
    ("mkhost_eval_symlinks", C.c_size_t, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]),
    ("mkhost_cache_key", C.c_size_t, [C.c_char_p, C.c_int, C.c_char_p, C.c_size_t]),
    ("mkhost_cache_entry_create", C.c_size_t, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]),
    ("mkhost_cache_entry_parse", C.c_int, [C.c_char_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]),
    ("mkhost_cache_chunk_entry_create", C.c_size_t, [C.POINTER(C.c_uint8), C.c_uint64, C.c_char_p, C.c_size_t]),
    ("mkhost_cache_chunk_entry_parse", C.c_int, [C.c_char_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.c_char_p,
                                                 C.c_size_t]),
    ("mkhost_describe_context_stream", C.c_size_t, [C.c_char_p, C.POINTER(C.c_char_p), C.c_size_t, C.c_char_p,
                                                    C.c_size_t, C.c_char_p, C.c_size_t]),
    ("mkhost_describe_layer", C.c_size_t, [C.c_char_p, C.c_int64, C.POINTER(CopyOp), C.c_size_t, C.c_char_p,
                                           C.c_size_t, C.c_char_p, C.c_size_t]),
]

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        abi.load()  # libmksnap first (libmkhost links against it)
        if not LIB_PATH.exists():
            raise FileNotFoundError(f"{LIB_PATH} not found: run __graft_entry__.build()")
        lib = C.CDLL(str(LIB_PATH))
        for name, res, args in SYMBOLS:
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


class HostError(RuntimeError):
    pass


def _strs(items: Sequence[str]):
    arr = (C.c_char_p * max(1, len(items)))(*[os.fsencode(s) for s in items])
    return arr


@dataclass
class CopyOperation:
    """snapshot.NewCopyOperation(srcs, srcRoot, workDir, dst, chown...) (lib/snapshot/copy_op.go:45)."""
    srcs: List[str]
    src_root: str
    work_dir: str
    dst: str
    uid: int = 0
    gid: int = 0


def _ops(ops: Sequence[CopyOperation]):
    keep = []
    arr = (CopyOp * max(1, len(ops)))()
    for i, o in enumerate(ops):
        s = _strs(o.srcs)
        keep.append(s)
        arr[i].src_root = os.fsencode(o.src_root)
        arr[i].srcs = s
        arr[i].n_srcs = len(o.srcs)
        arr[i].work_dir = os.fsencode(o.work_dir)
        arr[i].dst = os.fsencode(o.dst)
        arr[i].uid, arr[i].gid = o.uid, o.gid
    return arr, keep


def encode_tar_header(name: str, mode: int, uid: int, gid: int, size: int, mtime_ns: int, typeflag: bytes,
                      linkname: str = "") -> bytes:
    h = TarHeader(os.fsencode(name), os.fsencode(linkname), mode, uid, gid, size, mtime_ns, typeflag)
    buf = C.create_string_buffer(8192)
    n = load().mkhost_encode_tar_header(C.byref(h), buf, len(buf))
    if n == 0:
        raise HostError("header not encodable")
    return buf.raw[:n]


def describe_context_stream(context_dir: str, from_paths: Sequence[str]) -> List[str]:
    err = C.create_string_buffer(1024)
    p = _strs(from_paths)
    n = load().mkhost_describe_context_stream(os.fsencode(context_dir), p, len(from_paths), None, 0, err, len(err))
    if n == 0:
        raise HostError(err.value.decode())
    buf = C.create_string_buffer(n)
    load().mkhost_describe_context_stream(os.fsencode(context_dir), p, len(from_paths), buf, n, err, len(err))
    return [l for l in os.fsdecode(buf.value).split("\n") if l]


def describe_layer(root_dir: str, now_unix: int, ops: Sequence[CopyOperation]) -> List[str]:
    err = C.create_string_buffer(1024)
    arr, keep = _ops(ops)
    n = load().mkhost_describe_layer(os.fsencode(root_dir), now_unix, arr, len(ops), None, 0, err, len(err))
    if n == 0:
        raise HostError(err.value.decode())
    buf = C.create_string_buffer(n)
    arr, keep = _ops(ops)
    load().mkhost_describe_layer(os.fsencode(root_dir), now_unix, arr, len(ops), buf, n, err, len(err))
    return [l for l in os.fsdecode(buf.value).split("\n") if l]


def context_crc32(eng: abi.Engine, prefix: bytes, context_dir: str, from_paths: Sequence[str], n_threads: int = 0):
    """-> (crc32 value as checksum.Sum32() would return it, stream length)."""
    err = C.create_string_buffer(1024)
    crc, slen = C.c_uint32(), C.c_uint64()
    rc = load().mkhost_context_crc32(eng.h, prefix, len(prefix), os.fsencode(context_dir), _strs(from_paths),
                                     len(from_paths), n_threads, C.byref(crc), C.byref(slen), err, len(err))
    if rc:
        raise HostError(err.value.decode())
    return crc.value, slen.value


def copy_step_cache_id(eng: abi.Engine, seed: str, directive: str, args: str, context_dir: str,
                       from_paths: Sequence[str]) -> str:
    crc, _ = context_crc32(eng, (seed + directive + args).encode(), context_dir, from_paths)
    return "%x" % crc  # add_copy_step.go:119


MKHOST_STEP_COPY, MKHOST_STEP_FROM, MKHOST_STEP_BASE, MKHOST_STEP_REMOTE_FROM = 1, 2, 3, 4


@dataclass
class PlanStep:
    """One step of a build plan for plan_cache_ids (include/mkhost.h, mkhost_plan_step).
    kind COPY: directive "COPY"/"ADD", from_paths its sources, from_stage set for COPY --from (no content);
    FROM / REMOTE_FROM: args = the image; BASE: any other directive, with its commit flag."""
    kind: int
    directive: str = ""
    args: str = ""
    from_paths: Sequence[str] = ()
    from_stage: str = ""
    commit: bool = False

    @classmethod
    def copy(cls, directive: str, args: str, from_paths: Sequence[str], from_stage: str = ""):
        return cls(MKHOST_STEP_COPY, directive, args, list(from_paths), from_stage)

    @classmethod
    def from_image(cls, image: str, remote: bool = False):
        return cls(MKHOST_STEP_REMOTE_FROM if remote else MKHOST_STEP_FROM, "FROM", image)

    @classmethod
    def base(cls, directive: str, args: str, commit: bool):
        return cls(MKHOST_STEP_BASE, directive, args, commit=commit)


def plan_cache_ids(eng: abi.Engine, seed: str, context_dir: str, steps: Sequence[PlanStep], n_threads: int = 0,
                   cache: Optional["CrcCache"] = None):
    """-> (cacheID of every step as "%x", stats dict): the whole plan in one pass over the context."""
    n = len(steps)
    arr, keep = (_PlanStep * max(1, n))(), []
    for i, s in enumerate(steps):
        paths = _strs(list(s.from_paths))
        keep.append(paths)
        arr[i].kind, arr[i].commit = s.kind, int(s.commit)
        arr[i].directive, arr[i].args = s.directive.encode(), s.args.encode()
        arr[i].from_stage = s.from_stage.encode()
        arr[i].from_paths, arr[i].n_paths = paths, len(s.from_paths)
    ids, st, err = (C.c_uint32 * max(1, n))(), CrcCacheStats(), C.create_string_buffer(1024)
    rc = load().mkhost_plan_cache_ids(eng.h, cache.h if cache is not None else None, seed.encode(), os.fsencode(context_dir),
                                      arr, n, n_threads, ids, C.byref(st), err, len(err))
    if rc:
        raise HostError(err.value.decode())
    return ["%x" % ids[i] for i in range(n)], {k: getattr(st, k) for k, _ in CrcCacheStats._fields_}


MKHOST_NO_TAR_DIGEST = 1
MKHOST_FILE_DIGESTS = 2   # remember per-file SHA-256 in the MemFS tree
MKHOST_SCAN_CONTENT = 4   # content-aware AddLayerByScan (implies FILE_DIGESTS)
MKHOST_MATERIALIZE = 8    # commit_copy_ops also performs the copy onto the file system, from the arena
MKHOST_MATERIALIZE_CHOWN = 16
MKHOST_UNTAR = 32         # UpdateFromTarReader(untar=true): also write the members under the root
MKHOST_GUNZIP = 64        # update_from_tar: tar_fd carries a gzip blob, decompressed on the GPU
MKHOST_COPY_CHOWN, MKHOST_COPY_INTERNAL, MKHOST_COPY_PRESERVE_OWNER, MKHOST_COPY_DEFERRED = 1, 2, 4, 8


def commit_copy_ops(eng: abi.Engine, root_dir: str, now_unix: int, ops: Sequence[CopyOperation], n_threads: int = 0,
                    tar_fd: int = -1, flags: int = 0):
    """commitLayer over AddLayerByCopyOps; tar_fd >= 0 also receives the uncompressed layer tar."""
    err = C.create_string_buffer(1024)
    arr, keep = _ops(ops)
    out = LayerResult()
    rc = load().mkhost_commit_copy_ops_ex(eng.h, os.fsencode(root_dir), now_unix, arr, len(ops), n_threads, tar_fd, flags,
                                          C.byref(out), err, len(err))
    if rc:
        raise HostError(err.value.decode())
    return {"tar_digest": "sha256:" + bytes(out.tar_digest).hex(), "root": bytes(out.root), "n_entries": out.n_entries,
            "tar_bytes": out.tar_bytes, "n_chunks": out.n_chunks, "n_unique": out.n_unique}


def _layer_dict(out: LayerResult):
    return {"tar_digest": "sha256:" + bytes(out.tar_digest).hex(), "root": bytes(out.root), "n_entries": out.n_entries,
            "tar_bytes": out.tar_bytes, "n_chunks": out.n_chunks, "n_unique": out.n_unique}


def _run_layers(layers: Sequence, keys: Sequence, call) -> List[dict]:
    """A run of layers through a C entry point: layers[i] is tar_fd or (tar_fd, per-layer flags such as MKHOST_GUNZIP),
    keys[i] a str or None.  call(specs, n, keys, outs, err) makes the C call.  -> one result dict per layer."""
    n = len(layers)
    specs, outs, err = (TarSpec * max(1, n))(), (LayerResult * max(1, n))(), C.create_string_buffer(1024)
    for i, l in enumerate(layers):
        specs[i].tar_fd, specs[i].flags = (l, 0) if isinstance(l, int) else l
    ks = (C.c_char_p * max(1, n))(*[k.encode() if k is not None else None for k in keys])
    if call(specs, n, ks, outs, err):
        raise HostError(err.value.decode())
    return [_layer_dict(outs[i]) for i in range(n)]


class MemFS:
    """snapshot.NewMemFS(clk, root, blacklist): layers accumulate; AddLayerByCopyOps / AddLayerByScan either
    described as text (no GPU) or committed through an Engine."""
    _BUF = 16 << 20

    def __init__(self, root: str, blacklist: Sequence[str] = ()):
        err = C.create_string_buffer(1024)
        self._bl = _strs(list(blacklist))
        self.h = load().mkhost_memfs_new(os.fsencode(root), self._bl, len(blacklist), err, len(err))
        if not self.h:
            raise HostError(err.value.decode())

    def close(self):
        if getattr(self, "h", None):
            load().mkhost_memfs_free(self.h)
            self.h = None

    __del__ = close

    def describe_copy_ops(self, now_unix: int, ops: Sequence[CopyOperation]) -> List[str]:
        err, buf = C.create_string_buffer(1024), C.create_string_buffer(self._BUF)
        arr, keep = _ops(ops)
        n = load().mkhost_memfs_describe_copy_ops(self.h, now_unix, arr, len(ops), buf, len(buf), err, len(err))
        if n == 0 or n > len(buf):
            raise HostError(err.value.decode() or "describe buffer too small")
        return [l for l in os.fsdecode(buf.value).split("\n") if l]

    def describe_scan(self, now_unix: int) -> List[str]:
        err, buf = C.create_string_buffer(1024), C.create_string_buffer(self._BUF)
        n = load().mkhost_memfs_describe_scan(self.h, now_unix, buf, len(buf), err, len(err))
        if n == 0 or n > len(buf):
            raise HostError(err.value.decode() or "describe buffer too small")
        return [l for l in os.fsdecode(buf.value).split("\n") if l]

    def commit_copy_ops(self, eng: abi.Engine, now_unix: int, ops: Sequence[CopyOperation], n_threads: int = 0,
                        tar_fd: int = -1, flags: int = 0):
        err, out = C.create_string_buffer(1024), LayerResult()
        arr, keep = _ops(ops)
        if load().mkhost_memfs_commit_copy_ops(self.h, eng.h, now_unix, arr, len(ops), n_threads, tar_fd, flags,
                                               C.byref(out), err, len(err)):
            raise HostError(err.value.decode())
        return _layer_dict(out)

    def commit_copy_ops_cached(self, eng: abi.Engine, cache: Optional["ChunkCache"], now_unix: int,
                               ops: Sequence[CopyOperation], n_threads: int = 0, tar_fd: int = -1, flags: int = 0):
        """commit_copy_ops with remembered chunk digests for unchanged files -> (layer dict, stats dict).  The layer is
        the one commit_copy_ops returns; cache None = no cache."""
        err, out, st = C.create_string_buffer(1024), LayerResult(), ChunkCacheStats()
        arr, keep = _ops(ops)
        if load().mkhost_memfs_commit_copy_ops_cached(self.h, eng.h, cache.h if cache is not None else None, now_unix, arr,
                                                      len(ops), n_threads, tar_fd, flags, C.byref(out), C.byref(st), err,
                                                      len(err)):
            raise HostError(err.value.decode())
        return _layer_dict(out), {k: getattr(st, k) for k, _ in ChunkCacheStats._fields_}

    def commit_layers(self, eng: abi.Engine, now_unix: int, layers: Sequence[Sequence[CopyOperation]], n_threads: int = 0,
                      tar_fds: Optional[Sequence[int]] = None, flags: int = 0):
        """Consecutive layers of one build in ONE engine session (all TarDigest chains advance together).
        flags: MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS."""
        return self._commit_layers(layers, tar_fds, lambda specs, n, outs, err: load().mkhost_memfs_commit_layers(
            self.h, eng.h, now_unix, specs, n, n_threads, flags, outs, err, len(err)))

    def commit_layers_cached(self, eng: abi.Engine, cache: Optional["ChunkCache"], now_unix: int,
                             layers: Sequence[Sequence[CopyOperation]], n_threads: int = 0,
                             tar_fds: Optional[Sequence[int]] = None, flags: int = 0):
        """commit_layers with remembered chunk digests for unchanged files -> (layer dicts, stats dict summed over the
        batch).  Equals commit_copy_ops_cached once per layer, except root / n_chunks / n_unique (the whole batch's) and
        the cache lookups, which all see the cache as it was when the call started.  cache None = no cache."""
        st = ChunkCacheStats()
        res = self._commit_layers(layers, tar_fds, lambda specs, n, outs, err: load().mkhost_memfs_commit_layers_cached(
            self.h, eng.h, cache.h if cache is not None else None, now_unix, specs, n, n_threads, flags, outs, C.byref(st),
            err, len(err)))
        return res, {k: getattr(st, k) for k, _ in ChunkCacheStats._fields_}

    @staticmethod
    def _commit_layers(layers: Sequence[Sequence[CopyOperation]], tar_fds: Optional[Sequence[int]], call) -> List[dict]:
        """call(specs, n, outs, err) makes the C call -> one result dict per layer."""
        err = C.create_string_buffer(1024)
        n = len(layers)
        specs, keep, outs = (LayerSpec * max(1, n))(), [], (LayerResult * max(1, n))()
        for i, ops in enumerate(layers):
            arr, k = _ops(ops)
            keep.append((arr, k))
            specs[i].ops, specs[i].n_ops = arr, len(ops)
            specs[i].tar_fd = tar_fds[i] if tar_fds is not None else -1
        if call(specs, n, outs, err):
            raise HostError(err.value.decode())
        return [_layer_dict(outs[i]) for i in range(n)]

    def file_digest(self, dst: str) -> Optional[bytes]:
        """SHA-256 the tree remembers for the regular file at dst, or None."""
        out = (C.c_uint8 * 32)()
        return bytes(out) if load().mkhost_memfs_file_digest(self.h, os.fsencode(dst), out) == 0 else None

    def describe_update_from_tar(self, now_unix: int, tar_fd: int, flags: int = 0) -> List[str]:
        """UpdateFromTarReader without a GPU: the merged layer as text (flags: MKHOST_UNTAR writes the members)."""
        err, buf = C.create_string_buffer(1024), C.create_string_buffer(self._BUF)
        n = load().mkhost_memfs_describe_update_from_tar_ex(self.h, now_unix, tar_fd, flags, buf, len(buf), err, len(err))
        if n == 0 or n > len(buf):
            raise HostError(err.value.decode() or "describe buffer too small")
        return [l for l in os.fsdecode(buf.value).split("\n") if l]

    def update_from_tar(self, eng: abi.Engine, now_unix: int, tar_fd: int, flags: int = 0):
        """UpdateFromTarReader(untar=false) through the GPU: DiffID of the blob + chunk table of its files."""
        err, out = C.create_string_buffer(1024), LayerResult()
        if load().mkhost_memfs_update_from_tar(self.h, eng.h, now_unix, tar_fd, flags, C.byref(out), err, len(err)):
            raise HostError(err.value.decode())
        return _layer_dict(out)

    def update_from_tars(self, eng: abi.Engine, now_unix: int, layers: Sequence, flags: int = 0):
        """A run of layers applied in order in ONE engine session, their DiffID chains hashed together.  layers: tar_fd
        or (tar_fd, per-layer flags such as MKHOST_GUNZIP) per layer.  -> one dict per layer, as update_from_tar gives;
        root / n_chunks / n_unique are those of the whole run."""
        return _run_layers(layers, (), lambda specs, n, ks, outs, err: load().mkhost_memfs_update_from_tars(
            self.h, eng.h, now_unix, specs, n, flags, outs, err, len(err)))

    def update_from_tar_indexed(self, eng: abi.Engine, cache: Optional["GzIndexCache"], key: Optional[str],
                                now_unix: int, tar_fd: int, flags: int = 0):
        """update_from_tar whose MKHOST_GUNZIP blob is opened with the block index cached under `key` (the image
        store's digest hex), and leaves the index it returns there.  -> (result dict, stats dict)."""
        err, out, st = C.create_string_buffer(1024), LayerResult(), GzIndexStats()
        if load().mkhost_memfs_update_from_tar_indexed(self.h, eng.h, cache.h if cache is not None else None,
                                                       key.encode() if key is not None else None, now_unix, tar_fd,
                                                       flags, C.byref(out), C.byref(st), err, len(err)):
            raise HostError(err.value.decode())
        return _layer_dict(out), {k: getattr(st, k) for k, _ in GzIndexStats._fields_}

    def update_from_tars_indexed(self, eng: abi.Engine, cache: Optional["GzIndexCache"], keys: Sequence,
                                 now_unix: int, layers: Sequence, flags: int = 0):
        """update_from_tars with a block-index cache: keys[i] (or None) for layer i.  -> (dicts, stats dict)."""
        st = GzIndexStats()
        res = _run_layers(layers, keys, lambda specs, n, ks, outs, err: load().mkhost_memfs_update_from_tars_indexed(
            self.h, eng.h, cache.h if cache is not None else None, ks, now_unix, specs, n, flags, outs, C.byref(st), err,
            len(err)))
        return res, {k: getattr(st, k) for k, _ in GzIndexStats._fields_}

    def update_from_tars_cached(self, eng: abi.Engine, cache: Optional["LayerCache"], gz: Optional["GzIndexCache"],
                                keys: Sequence, now_unix: int, layers: Sequence, flags: int = 0):
        """update_from_tars_indexed that replays the layers `cache` remembers under keys[i] for an unchanged store file,
        and remembers the others.  -> (dicts, layer-cache stats dict, gz-index stats dict)."""
        st, gst = LayerCacheStats(), GzIndexStats()
        res = _run_layers(layers, keys, lambda specs, n, ks, outs, err: load().mkhost_memfs_update_from_tars_cached(
            self.h, eng.h, cache.h if cache is not None else None, gz.h if gz is not None else None, ks, now_unix, specs, n,
            flags, outs, C.byref(st), C.byref(gst), err, len(err)))
        return (res, {k: getattr(st, k) for k, _ in LayerCacheStats._fields_},
                {k: getattr(gst, k) for k, _ in GzIndexStats._fields_})

    def commit_scan(self, eng: abi.Engine, now_unix: int, n_threads: int = 0, tar_fd: int = -1, flags: int = 0):
        err, out = C.create_string_buffer(1024), LayerResult()
        if load().mkhost_memfs_commit_scan(self.h, eng.h, now_unix, n_threads, tar_fd, flags, C.byref(out), err, len(err)):
            raise HostError(err.value.decode())
        return _layer_dict(out)


# ---- cache.Manager wire format (lib/cache/cache_manager.go:34-35,239-252) --------------------------
def cache_key(cache_id: str, chunk_table: bool = False) -> str:
    buf = C.create_string_buffer(len(cache_id) + 64)
    load().mkhost_cache_key(cache_id.encode(), int(chunk_table), buf, len(buf))
    return buf.value.decode()


def cache_entry_create(tar_hex: Optional[str], gzip_hex: str = "") -> str:
    buf = C.create_string_buffer(len(tar_hex or "") + len(gzip_hex) + 32)
    load().mkhost_cache_entry_create(None if tar_hex is None else tar_hex.encode(), gzip_hex.encode(), buf, len(buf))
    return buf.value.decode()


def cache_entry_parse(entry: str):
    t, g, err = C.create_string_buffer(len(entry) + 16), C.create_string_buffer(len(entry) + 16), C.create_string_buffer(512)
    if load().mkhost_cache_entry_parse(entry.encode(), t, len(t), g, len(g), err, len(err)):
        raise HostError(err.value.decode())
    return t.value.decode(), g.value.decode()


def cache_chunk_entry_create(root: bytes, n_unique: int) -> str:
    buf = C.create_string_buffer(128)
    load().mkhost_cache_chunk_entry_create((C.c_uint8 * 32).from_buffer_copy(root), n_unique, buf, len(buf))
    return buf.value.decode()


def cache_chunk_entry_parse(entry: str):
    root, n, err = (C.c_uint8 * 32)(), C.c_uint64(), C.create_string_buffer(512)
    if load().mkhost_cache_chunk_entry_parse(entry.encode(), root, C.byref(n), err, len(err)):
        raise HostError(err.value.decode())
    return bytes(root), n.value


def copy_op_execute(op: "CopyOperation", mode: int = 0, blacklist: Sequence[str] = ()) -> None:
    """CopyOperation.Execute (lib/snapshot/copy_op.go:82-147) through fileio.Copier's rules."""
    err = C.create_string_buffer(1024)
    arr, keep = _ops([op])
    bl = _strs(list(blacklist))
    if load().mkhost_copy_op_execute(arr, mode, bl, len(blacklist), err, len(err)):
        raise HostError(err.value.decode())


def eval_symlinks(path: str, src_root: str) -> str:
    """evalSymlinks(p, srcRoot) (lib/snapshot/utils.go:249-324)."""
    err, buf = C.create_string_buffer(1024), C.create_string_buffer(8192)
    n = load().mkhost_eval_symlinks(os.fsencode(path), os.fsencode(src_root), buf, len(buf), err, len(err))
    if n == 0 or n > len(buf):
        raise HostError(err.value.decode() or "path too long")
    return os.fsdecode(buf.value)


class _Cache:
    """A libmkhost cache object (mkhost_<prefix>_cache_*), owned by the caller and kept between builds through its file:
    a file that does not parse fails the load and leaves the cache as it was."""
    _prefix = ""

    def __init__(self, path: Optional[str] = None):
        self.h = self._fn("new")()
        if path is not None and os.path.exists(path):
            self.load(path)

    @classmethod
    def _fn(cls, op: str):
        return getattr(load(), "mkhost_%s_cache_%s" % (cls._prefix, op))

    def __len__(self):
        return int(self._fn("size")(self.h))

    def load(self, path: str):
        err = C.create_string_buffer(512)
        if self._fn("load")(self.h, os.fsencode(path), err, len(err)):
            raise HostError(err.value.decode())

    def save(self, path: str):
        err = C.create_string_buffer(512)
        if self._fn("save")(self.h, os.fsencode(path), err, len(err)):
            raise HostError(err.value.decode())

    def close(self):
        if getattr(self, "h", None):
            self._fn("free")(self.h)
            self.h = None

    __del__ = close


class CrcCache(_Cache):
    """pure(file content) per context file, remembered between builds: unchanged files are folded into the cacheID on
    the host, only changed files travel to the device (include/mkhost.h, "Incremental cacheID")."""
    _prefix = "crc"

    def context_crc32(self, eng: abi.Engine, prefix: bytes, context_dir: str, from_paths: Sequence[str], n_threads: int = 0):
        """-> (crc32 as checksum.Sum32() returns it, stream length, stats dict)."""
        err = C.create_string_buffer(1024)
        crc, slen, st = C.c_uint32(), C.c_uint64(), CrcCacheStats()
        rc = load().mkhost_context_crc32_cached(eng.h, self.h, prefix, len(prefix), os.fsencode(context_dir), _strs(from_paths),
                                                len(from_paths), n_threads, C.byref(crc), C.byref(slen), C.byref(st), err, len(err))
        if rc:
            raise HostError(err.value.decode())
        return crc.value, slen.value, {k: getattr(st, k) for k, _ in CrcCacheStats._fields_}


class ChunkCache(_Cache):
    """Chunk digests per source file, remembered between builds: a layer commit takes an unchanged file's digests from
    here instead of chunking it again (include/mkhost.h, "Incremental layer commit"; MemFS.commit_copy_ops_cached)."""
    _prefix = "chunk"


class GzIndexCache(_Cache):
    """Block indexes of single-member gzip layers, per image-store digest, remembered between builds: a later ingest
    of the same blob decodes it in parallel on the device (include/mkhost.h; MemFS.update_from_tar(s)_indexed)."""
    _prefix = "gz_index"


class LayerCache(_Cache):
    """What a run of layers took from each blob, per image-store digest, remembered between builds: a later run replays
    an unchanged store file instead of reading, decompressing and hashing it (include/mkhost.h, "Incremental layer
    ingest"; MemFS.update_from_tars_cached)."""
    _prefix = "layer"
