// +build mksnap

// Package mksnap binds libmksnap.so (include/mksnap.h: the H100 snapshot+hash engine) and libmkhost.so
// (include/mkhost.h: walker, tar headers and arena packers above it) into makisu.
//
// Drop this directory into the reference tree as lib/mksnap, apply integration/patches/*.patch and build with
//   CGO_ENABLED=1 go build -tags mksnap ./bin/makisu
// Without the tag the stock pure-Go files are compiled unchanged.  The engine has no CPU fallback: New fails when no
// sm_90 device is usable, and so does the build that asked for it.
//
// NOTE: the image this repository is built in has no Go toolchain, so these files have been reviewed against
// include/*.h but never compiled; the same C entry points are exercised from Python (makisu_b200/abi.py, host.py).
package mksnap

/*
#cgo LDFLAGS: -lmkhost -lmksnap
#include <stdlib.h>
#include "mksnap.h"
#include "mkhost.h"
*/
import "C"

import (
	"bytes"
	"compress/gzip"
	"encoding/hex"
	"fmt"
	"io"
	"os"
	"runtime"
	"unsafe"
)

// Engine owns one GPU: streams, pinned host arenas, device slots.  One session at a time; the reference drives the
// seams from the plan goroutine (lib/builder/build_plan.go:174), which is what the C side expects.
type Engine struct{ h *C.mksnap_t }

// New creates an engine on `device` with nArenas pinned host arenas of arenaBytes each (1 GiB and 3 are good
// defaults: one being filled, one in flight, one on the device).
func New(device int, arenaBytes uint64, nArenas int) (*Engine, error) {
	cfg := C.mksnap_config{
		device:             C.int32_t(device),
		n_host_arenas:      C.uint32_t(nArenas),
		host_arena_bytes:   C.uint64_t(arenaBytes),
		device_arena_bytes: C.uint64_t(arenaBytes),
		max_extents:        1 << 20,
	}
	e := &Engine{}
	if rc := C.mksnap_create(&cfg, &e.h); rc != 0 {
		return nil, fmt.Errorf("mksnap create: %s", C.GoString(C.mksnap_last_error(nil)))
	}
	runtime.SetFinalizer(e, func(e *Engine) { e.Close() })
	return e, nil
}

// Close releases the device.
func (e *Engine) Close() {
	if e.h != nil {
		C.mksnap_destroy(e.h)
		e.h = nil
	}
}

const errLen = 1024

func cStrings(ss []string) (**C.char, func()) {
	arr := C.malloc(C.size_t(len(ss)+1) * C.size_t(unsafe.Sizeof(uintptr(0))))
	view := (*[1 << 28]*C.char)(arr)[: len(ss)+1 : len(ss)+1]
	for i, s := range ss {
		view[i] = C.CString(s)
	}
	view[len(ss)] = nil
	return (**C.char)(arr), func() {
		for i := range ss {
			C.free(unsafe.Pointer(view[i]))
		}
		C.free(arr)
	}
}

// ContextCRC32 replaces the crc32.NewIEEE() / filepath.Walk / io.Copy chain of
// addCopyStep.SetCacheID (lib/builder/step/add_copy_step.go:102-122,153-238): prefix is seed+directive+args,
// fromPaths are the directive's sources exactly as resolveFromPaths receives them.  The result is what
// checksum.Sum32() returns; format it with "%x".
func (e *Engine) ContextCRC32(prefix []byte, contextDir string, fromPaths []string, threads int) (uint32, error) {
	var crc C.uint32_t
	var n C.uint64_t
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cdir := C.CString(contextDir)
	defer C.free(unsafe.Pointer(cdir))
	paths, free := cStrings(fromPaths)
	defer free()
	var p unsafe.Pointer
	if len(prefix) > 0 {
		p = C.CBytes(prefix)
		defer C.free(p)
	}
	if rc := C.mkhost_context_crc32(e.h, p, C.size_t(len(prefix)), cdir, paths, C.size_t(len(fromPaths)),
		C.int(threads), &crc, &n, errBuf, errLen); rc != 0 {
		return 0, fmt.Errorf("%s", C.GoString(errBuf)) // already "hash context sources: ..." like add_copy_step.go:116
	}
	return uint32(crc), nil
}

// CopyOp mirrors snapshot.CopyOperation (lib/snapshot/copy_op.go:29-80).
type CopyOp struct {
	SrcRoot, WorkDir, Dst string
	Srcs                  []string
	UID, GID              int
}

// LayerResult carries what commitLayer needs (lib/builder/step/common.go:86-110) plus the chunk-table address.
type LayerResult struct {
	TarDigest        string // "sha256:<hex>" == image.DigestPair.TarDigest
	ChunkRoot        [32]byte
	Entries, TarSize uint64
	Chunks, Unique   uint64
}

func toResult(r *C.mkhost_layer_result) LayerResult {
	out := LayerResult{Entries: uint64(r.n_entries), TarSize: uint64(r.tar_bytes), Chunks: uint64(r.n_chunks), Unique: uint64(r.n_unique)}
	out.TarDigest = "sha256:" + hex.EncodeToString(C.GoBytes(unsafe.Pointer(&r.tar_digest[0]), 32))
	copy(out.ChunkRoot[:], C.GoBytes(unsafe.Pointer(&r.root[0]), 32))
	return out
}

// MemFS is the C++ mirror of snapshot.MemFS (lib/snapshot/mem_fs.go:60-83): the merged tree lives on the C side, so
// the entry order, the headers and the tar bytes are produced next to the arenas they are packed into.
type MemFS struct{ m *C.mkhost_memfs }

// NewMemFS = snapshot.NewMemFS(clk, root, blacklist); the clock is passed per call (now) instead.
func NewMemFS(root string, blacklist []string) (*MemFS, error) {
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	croot := C.CString(root)
	defer C.free(unsafe.Pointer(croot))
	bl, free := cStrings(blacklist)
	defer free()
	m := C.mkhost_memfs_new(croot, bl, C.size_t(len(blacklist)), errBuf, errLen)
	if m == nil {
		return nil, fmt.Errorf("new memfs: %s", C.GoString(errBuf))
	}
	fs := &MemFS{m: m}
	runtime.SetFinalizer(fs, func(fs *MemFS) { C.mkhost_memfs_free(fs.m) })
	return fs, nil
}

type cOps struct {
	arr   *C.mkhost_copy_op
	n     int
	frees []func()
}

func newCOps(ops []CopyOp) *cOps {
	c := &cOps{n: len(ops)}
	c.arr = (*C.mkhost_copy_op)(C.calloc(C.size_t(len(ops)+1), C.size_t(unsafe.Sizeof(C.mkhost_copy_op{}))))
	view := (*[1 << 20]C.mkhost_copy_op)(unsafe.Pointer(c.arr))[:len(ops):len(ops)]
	for i, o := range ops {
		srcs, free := cStrings(o.Srcs)
		c.frees = append(c.frees, free)
		view[i].src_root, view[i].work_dir, view[i].dst = C.CString(o.SrcRoot), C.CString(o.WorkDir), C.CString(o.Dst)
		view[i].srcs, view[i].n_srcs = srcs, C.size_t(len(o.Srcs))
		view[i].uid, view[i].gid = C.int32_t(o.UID), C.int32_t(o.GID)
	}
	return c
}

func (c *cOps) free() {
	view := (*[1 << 20]C.mkhost_copy_op)(unsafe.Pointer(c.arr))[:c.n:c.n]
	for i := range view {
		C.free(unsafe.Pointer(view[i].src_root))
		C.free(unsafe.Pointer(view[i].work_dir))
		C.free(unsafe.Pointer(view[i].dst))
	}
	for _, f := range c.frees {
		f()
	}
	C.free(unsafe.Pointer(c.arr))
}

// Flags of the commit calls (include/mkhost.h).
const (
	NoTarDigest uint32 = 1 // leave TarDigest to the caller (keep sha256.New() on the host for a single huge layer)
	FileDigests uint32 = 2
	ScanContent uint32 = 4
	Materialize uint32 = 8
	Gunzip      uint32 = 64 // UpdateFromTar: tarIn is the gzip blob as the image store holds it, decompressed on the GPU
)

// CommitCopyOps = MemFS.AddLayerByCopyOps + commitLayer's tar/SHA-256 half (mem_fs.go:276-289, common.go:35-63).
// The uncompressed layer tar is written to tarOut (feed it to pgzip); TarDigest comes back from the GPU.
func (fs *MemFS) CommitCopyOps(e *Engine, now int64, ops []CopyOp, tarOut *os.File, threads int, flags uint32) (LayerResult, error) {
	c := newCOps(ops)
	defer c.free()
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	fd := C.int(-1)
	if tarOut != nil {
		fd = C.int(tarOut.Fd())
	}
	var r C.mkhost_layer_result
	if rc := C.mkhost_memfs_commit_copy_ops(fs.m, e.h, C.int64_t(now), c.arr, C.size_t(c.n), C.int(threads), fd,
		C.uint32_t(flags), &r, errBuf, errLen); rc != 0 {
		return LayerResult{}, fmt.Errorf("%s", C.GoString(errBuf)) // "failed to generate diff layer: ..." (common.go:82)
	}
	return toResult(&r), nil
}

// CommitScan = MemFS.AddLayerByScan + the same digest half (mem_fs.go:260-270).
func (fs *MemFS) CommitScan(e *Engine, now int64, tarOut *os.File, threads int, flags uint32) (LayerResult, error) {
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	fd := C.int(-1)
	if tarOut != nil {
		fd = C.int(tarOut.Fd())
	}
	var r C.mkhost_layer_result
	if rc := C.mkhost_memfs_commit_scan(fs.m, e.h, C.int64_t(now), C.int(threads), fd, C.uint32_t(flags), &r, errBuf, errLen); rc != 0 {
		return LayerResult{}, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return toResult(&r), nil
}

// CommitLayers commits consecutive COPY/ADD layers of one build in ONE engine session: every TarDigest chain
// advances together on the device (on an H100 one chain runs at ~0.06 GB/s, 256 chains at ~15 GB/s).  tarOuts[i] may be nil.
// flags: NoTarDigest, FileDigests.
func (fs *MemFS) CommitLayers(e *Engine, now int64, layers [][]CopyOp, tarOuts []*os.File, threads int, flags uint32) ([]LayerResult, error) {
	res, _, err := fs.CommitLayersCached(e, nil, now, layers, tarOuts, threads, flags)
	return res, err
}

// ChunkCache remembers the chunk digests of every source file a layer commit chunked (include/mkhost.h, "Incremental
// layer commit"): an unchanged file (same device, inode, size, mtime, ctime) is not chunked again, and under
// NoTarDigest its bytes do not travel to the device.  One cache per build context; Save/Load keep it between makisu
// invocations.
type ChunkCache struct{ c *C.mkhost_chunk_cache }

// NewChunkCache loads `path` when it exists ("" = start cold).
func NewChunkCache(path string) (*ChunkCache, error) {
	cc := &ChunkCache{c: C.mkhost_chunk_cache_new()}
	runtime.SetFinalizer(cc, func(cc *ChunkCache) { C.mkhost_chunk_cache_free(cc.c) })
	if path == "" {
		return cc, nil
	}
	if _, err := os.Stat(path); err != nil {
		return cc, nil
	}
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_chunk_cache_load(cc.c, cpath, errBuf, errLen) != 0 {
		return nil, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return cc, nil
}

// Save writes the cache next to the build context (or into makisu's storage dir).
func (cc *ChunkCache) Save(path string) error {
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_chunk_cache_save(cc.c, cpath, errBuf, errLen) != 0 {
		return fmt.Errorf("%s", C.GoString(errBuf))
	}
	return nil
}

// ChunkCacheStats adds up over a call: regular files and their bytes, files taken from the cache, bytes chunked on
// the device, file bytes copied to the device.
type ChunkCacheStats struct {
	FilesTotal, FilesReused                 uint64
	BytesTotal, BytesChunked, BytesUploaded uint64
}

// CommitLayersCached is CommitLayers with the chunk cache in the loop (cc == nil: no cache).  The result equals one
// cached commit per layer in order -- tree, file digests, tar bytes, TarDigest per layer, the cache afterwards --
// except that every lookup sees the cache as it was when the call started.
func (fs *MemFS) CommitLayersCached(e *Engine, cc *ChunkCache, now int64, layers [][]CopyOp, tarOuts []*os.File, threads int,
	flags uint32) ([]LayerResult, ChunkCacheStats, error) {
	return fs.CommitLayersMulti([]*Engine{e}, cc, now, layers, tarOuts, threads, flags)
}

// engineArray is the mksnap_t * of every engine in C memory; free it with C.free.
func engineArray(engines []*Engine) **C.mksnap_t {
	n := len(engines)
	arr := (**C.mksnap_t)(C.calloc(C.size_t(n+1), C.size_t(unsafe.Sizeof((*C.mksnap_t)(nil)))))
	view := (*[1 << 20]*C.mksnap_t)(unsafe.Pointer(arr))[:n:n]
	for i, e := range engines {
		view[i] = e.h
	}
	return arr
}

// CommitLayersMulti is CommitLayersCached with the layers shared out over several engines -- one per GPU of the build
// host, or several on one -- each driven by libmkhost from a thread of its own (mkhost_memfs_commit_layers_multi).  The
// result is that of CommitLayersCached on engines[0], bit for bit.  The engines must not be used by anything else
// during the call.
func (fs *MemFS) CommitLayersMulti(engines []*Engine, cc *ChunkCache, now int64, layers [][]CopyOp, tarOuts []*os.File,
	threads int, flags uint32) ([]LayerResult, ChunkCacheStats, error) {
	n := len(layers)
	specs := (*C.mkhost_layer_spec)(C.calloc(C.size_t(n+1), C.size_t(unsafe.Sizeof(C.mkhost_layer_spec{}))))
	defer C.free(unsafe.Pointer(specs))
	sview := (*[1 << 20]C.mkhost_layer_spec)(unsafe.Pointer(specs))[:n:n]
	for i, ops := range layers {
		c := newCOps(ops)
		defer c.free()
		sview[i].ops, sview[i].n_ops, sview[i].tar_fd = c.arr, C.size_t(c.n), -1
		if tarOuts != nil && tarOuts[i] != nil {
			sview[i].tar_fd = C.int(tarOuts[i].Fd())
		}
	}
	outs := (*C.mkhost_layer_result)(C.calloc(C.size_t(n+1), C.size_t(unsafe.Sizeof(C.mkhost_layer_result{}))))
	defer C.free(unsafe.Pointer(outs))
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	var cache *C.mkhost_chunk_cache
	if cc != nil {
		cache = cc.c
	}
	hs := engineArray(engines)
	defer C.free(unsafe.Pointer(hs))
	var st C.mkhost_chunk_cache_stats
	if rc := C.mkhost_memfs_commit_layers_multi(fs.m, hs, C.size_t(len(engines)), cache, C.int64_t(now), specs, C.size_t(n),
		C.int(threads), C.uint32_t(flags), outs, &st, errBuf, errLen); rc != 0 {
		return nil, ChunkCacheStats{}, fmt.Errorf("%s", C.GoString(errBuf))
	}
	oview := (*[1 << 20]C.mkhost_layer_result)(unsafe.Pointer(outs))[:n:n]
	res := make([]LayerResult, n)
	for i := range res {
		res[i] = toResult(&oview[i])
	}
	return res, ChunkCacheStats{uint64(st.files_total), uint64(st.files_reused), uint64(st.bytes_total),
		uint64(st.bytes_chunked), uint64(st.bytes_uploaded)}, nil
}

// DecodesInParallel reports whether the gzip blob in f has, in its first 2 MiB, segment starts that let the device
// decode it in parallel (UpdateFromTar with Gunzip): a flush marker (00 00 FF FF, the empty stored block pgzip ends
// every 1 MiB block with: the layers makisu writes itself, tario.NewGzipWriter), or a second member right after the
// first one's trailer (bgzip / BGZF, eStargz layers, pigz --independent, concatenated gzip files).  A single member
// without flush points (the gzip CLI, compress/gzip, most registry layers) reports false: it is one GPU thread's work.
// The first member is inflated on the CPU to find its end, reading at most the 2 MiB.  f is left at offset 0.
func DecodesInParallel(f *os.File) (bool, error) {
	buf := make([]byte, 2<<20)
	n, err := f.ReadAt(buf, 0)
	if err != nil && err != io.EOF {
		return false, err
	}
	buf = buf[:n]
	if bytes.Contains(buf, []byte{0, 0, 0xFF, 0xFF}) {
		return true, nil
	}
	br := bytes.NewReader(buf) // an io.ByteReader: the gzip reader takes no byte past the first member's trailer
	zr, err := gzip.NewReader(br)
	if err != nil {
		return false, nil
	}
	zr.Multistream(false)
	if _, err := io.Copy(io.Discard, zr); err != nil {
		return false, nil // the first member runs past 2 MiB, or is malformed
	}
	rest := buf[n-br.Len():]
	return len(rest) >= 3 && rest[0] == 0x1f && rest[1] == 0x8b && rest[2] == 8, nil
}

// UpdateFromTar = MemFS.UpdateFromTarReader (mem_fs.go:165-255) on a tar stream, uncompressed or, with Gunzip, the
// gzip blob itself (no tario.NewGzipReader): the DiffID of the tar and the chunk table come back; untar also writes the
// members under the root from the arena.
func (fs *MemFS) UpdateFromTar(e *Engine, now int64, tarIn *os.File, untar bool, flags uint32) (LayerResult, error) {
	if untar {
		flags |= 32 // MKHOST_UNTAR
	}
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	var r C.mkhost_layer_result
	if rc := C.mkhost_memfs_update_from_tar(fs.m, e.h, C.int64_t(now), C.int(tarIn.Fd()), C.uint32_t(flags), &r, errBuf, errLen); rc != 0 {
		return LayerResult{}, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return toResult(&r), nil
}

// CrcCache remembers pure(file content) per context file between builds (include/mkhost.h, "Incremental cacheID"):
// unchanged files (same device, inode, size, mtime, ctime) are folded into the cacheID on the host, only changed files
// travel to the device.  One cache per build context; Save/Load keep it between makisu invocations.
type CrcCache struct{ c *C.mkhost_crc_cache }

// NewCrcCache loads `path` when it exists ("" = start cold).
func NewCrcCache(path string) (*CrcCache, error) {
	cc := &CrcCache{c: C.mkhost_crc_cache_new()}
	runtime.SetFinalizer(cc, func(cc *CrcCache) { C.mkhost_crc_cache_free(cc.c) })
	if path == "" {
		return cc, nil
	}
	if _, err := os.Stat(path); err != nil {
		return cc, nil
	}
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_crc_cache_load(cc.c, cpath, errBuf, errLen) != 0 {
		return nil, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return cc, nil
}

// Save writes the cache next to the build context (or into makisu's storage dir).
func (cc *CrcCache) Save(path string) error {
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_crc_cache_save(cc.c, cpath, errBuf, errLen) != 0 {
		return fmt.Errorf("%s", C.GoString(errBuf))
	}
	return nil
}

// ContextCRC32Cached is ContextCRC32 with the cache in the loop; sent = file bytes that travelled to the device.
func (e *Engine) ContextCRC32Cached(cc *CrcCache, prefix []byte, contextDir string, fromPaths []string, threads int) (crc uint32, sent uint64, err error) {
	var c C.uint32_t
	var n C.uint64_t
	var st C.mkhost_crc_cache_stats
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cdir := C.CString(contextDir)
	defer C.free(unsafe.Pointer(cdir))
	paths, free := cStrings(fromPaths)
	defer free()
	var p unsafe.Pointer
	if len(prefix) > 0 {
		p = C.CBytes(prefix)
		defer C.free(p)
	}
	if rc := C.mkhost_context_crc32_cached(e.h, cc.c, p, C.size_t(len(prefix)), cdir, paths, C.size_t(len(fromPaths)),
		C.int(threads), &c, &n, &st, errBuf, errLen); rc != 0 {
		return 0, 0, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return uint32(c), uint64(st.bytes_sent), nil
}

// ContextCRC32Multi is ContextCRC32Cached with the context's files shared out over several engines, each driven by
// libmkhost from a thread of its own (mkhost_context_crc32_multi); cc may be nil.  The cacheID is that of one engine,
// bit for bit.
func ContextCRC32Multi(engines []*Engine, cc *CrcCache, prefix []byte, contextDir string, fromPaths []string,
	threads int) (crc uint32, sent uint64, err error) {
	var c C.uint32_t
	var n C.uint64_t
	var st C.mkhost_crc_cache_stats
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cdir := C.CString(contextDir)
	defer C.free(unsafe.Pointer(cdir))
	paths, free := cStrings(fromPaths)
	defer free()
	var p unsafe.Pointer
	if len(prefix) > 0 {
		p = C.CBytes(prefix)
		defer C.free(p)
	}
	var cache *C.mkhost_crc_cache
	if cc != nil {
		cache = cc.c
	}
	hs := engineArray(engines)
	defer C.free(unsafe.Pointer(hs))
	if rc := C.mkhost_context_crc32_multi(hs, C.size_t(len(engines)), cache, p, C.size_t(len(prefix)), cdir, paths,
		C.size_t(len(fromPaths)), C.int(threads), &c, &n, &st, errBuf, errLen); rc != 0 {
		return 0, 0, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return uint32(c), uint64(st.bytes_sent), nil
}

// GzIndexCache remembers where the DEFLATE blocks of single-member gzip layers start, per image-store digest
// (include/mkhost.h, "Block indexes of single-member gzip layers"): the first ingest of a base-image layer records the
// index, later ingests of the same blob decode it in parallel on the GPU.  One cache per image store; Save/Load keep it
// between makisu invocations.  A stale or foreign entry costs speed only, never output.
type GzIndexCache struct{ c *C.mkhost_gz_index_cache }

// NewGzIndexCache loads `path` when it exists ("" = start cold).
func NewGzIndexCache(path string) (*GzIndexCache, error) {
	gc := &GzIndexCache{c: C.mkhost_gz_index_cache_new()}
	runtime.SetFinalizer(gc, func(gc *GzIndexCache) { C.mkhost_gz_index_cache_free(gc.c) })
	if path == "" {
		return gc, nil
	}
	if _, err := os.Stat(path); err != nil {
		return gc, nil
	}
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_gz_index_cache_load(gc.c, cpath, errBuf, errLen) != 0 {
		return nil, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return gc, nil
}

// Save writes the cache (next to the image store).
func (gc *GzIndexCache) Save(path string) error {
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_gz_index_cache_save(gc.c, cpath, errBuf, errLen) != 0 {
		return fmt.Errorf("%s", C.GoString(errBuf))
	}
	return nil
}

// TarLayer is one layer of a run: the store file and its per-layer flags (Gunzip), and the key of its block index in
// a GzIndexCache (descriptor.Digest.Hex(); "" = none).
type TarLayer struct {
	File  *os.File
	Flags uint32
	Key   string
}

// UpdateFromTarsIndexed applies a run of layers in order in one engine session (FromStep.Execute, buildNode.applyLayer),
// each Gunzip layer with a key opened with the block index cached under it; gc == nil is the same run without an index.
func (fs *MemFS) UpdateFromTarsIndexed(e *Engine, gc *GzIndexCache, now int64, layers []TarLayer, untar bool, flags uint32) ([]LayerResult, error) {
	if untar {
		flags |= 32 // MKHOST_UNTAR
	}
	n := len(layers)
	if n == 0 {
		return nil, nil
	}
	specs := make([]C.mkhost_tar_spec, n)
	keys := make([]string, n)
	for i, l := range layers {
		specs[i].tar_fd = C.int(l.File.Fd())
		specs[i].flags = C.uint32_t(l.Flags)
		keys[i] = l.Key
	}
	ckeys, freeKeys := cStrings(keys)
	defer freeKeys()
	view := (*[1 << 28]*C.char)(unsafe.Pointer(ckeys))[:n:n]
	for i := range keys {
		if keys[i] == "" { // NULL key: this layer is opened without an index
			C.free(unsafe.Pointer(view[i]))
			view[i] = nil
		}
	}
	var cache *C.mkhost_gz_index_cache
	if gc != nil {
		cache = gc.c
	}
	outs := make([]C.mkhost_layer_result, n)
	var st C.mkhost_gz_index_stats
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	if rc := C.mkhost_memfs_update_from_tars_indexed(fs.m, e.h, cache, (**C.char)(unsafe.Pointer(ckeys)), C.int64_t(now),
		&specs[0], C.size_t(n), C.uint32_t(flags), &outs[0], &st, errBuf, errLen); rc != 0 {
		return nil, fmt.Errorf("%s", C.GoString(errBuf))
	}
	res := make([]LayerResult, n)
	for i := range outs {
		res[i] = toResult(&outs[i])
	}
	return res, nil
}

// LayerCache remembers what a run of layers took from each blob, per image-store digest (include/mkhost.h,
// "Incremental layer ingest"): a later run replays an unchanged store file -- its remembered headers merged, its chunk
// digests appended, its DiffID taken from the record -- instead of reading, decompressing and hashing it.  One cache
// per image store, beside gz-index.cache; Save/Load keep it between makisu invocations.
type LayerCache struct{ c *C.mkhost_layer_cache }

// NewLayerCache loads `path` when it exists ("" = start cold).
func NewLayerCache(path string) (*LayerCache, error) {
	lc := &LayerCache{c: C.mkhost_layer_cache_new()}
	runtime.SetFinalizer(lc, func(lc *LayerCache) { C.mkhost_layer_cache_free(lc.c) })
	if path == "" {
		return lc, nil
	}
	if _, err := os.Stat(path); err != nil {
		return lc, nil
	}
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_layer_cache_load(lc.c, cpath, errBuf, errLen) != 0 {
		return nil, fmt.Errorf("%s", C.GoString(errBuf))
	}
	return lc, nil
}

// Save writes the cache (next to the image store).
func (lc *LayerCache) Save(path string) error {
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	cpath := C.CString(path)
	defer C.free(unsafe.Pointer(cpath))
	if C.mkhost_layer_cache_save(lc.c, cpath, errBuf, errLen) != 0 {
		return fmt.Errorf("%s", C.GoString(errBuf))
	}
	return nil
}

// UpdateFromTarsCached is UpdateFromTarsIndexed that replays every layer lc remembers under its Key for an unchanged
// store file and records the others; lc == nil is UpdateFromTarsIndexed.  Results are those of the uncached run.
func (fs *MemFS) UpdateFromTarsCached(e *Engine, lc *LayerCache, gc *GzIndexCache, now int64, layers []TarLayer, untar bool, flags uint32) ([]LayerResult, error) {
	return fs.UpdateFromTarsMulti([]*Engine{e}, lc, gc, now, layers, untar, flags)
}

// UpdateFromTarsMulti is UpdateFromTarsCached with the layers shared out over several engines -- one per GPU of the
// build host, or several on one -- each driven by libmkhost from a thread of its own (mkhost_memfs_update_from_tars_multi).
// The result is that of UpdateFromTarsCached on engines[0], bit for bit.  Every layer needs a File of its own, and untar
// (--modifyfs) takes one engine.  The engines must not be used by anything else during the call.
func (fs *MemFS) UpdateFromTarsMulti(engines []*Engine, lc *LayerCache, gc *GzIndexCache, now int64, layers []TarLayer, untar bool, flags uint32) ([]LayerResult, error) {
	if untar {
		flags |= 32 // MKHOST_UNTAR
	}
	n := len(layers)
	if n == 0 {
		return nil, nil
	}
	specs := make([]C.mkhost_tar_spec, n)
	keys := make([]string, n)
	for i, l := range layers {
		specs[i].tar_fd = C.int(l.File.Fd())
		specs[i].flags = C.uint32_t(l.Flags)
		keys[i] = l.Key
	}
	ckeys, freeKeys := cStrings(keys)
	defer freeKeys()
	view := (*[1 << 28]*C.char)(unsafe.Pointer(ckeys))[:n:n]
	for i := range keys {
		if keys[i] == "" { // NULL key: no cache for this layer
			C.free(unsafe.Pointer(view[i]))
			view[i] = nil
		}
	}
	var cache *C.mkhost_layer_cache
	if lc != nil {
		cache = lc.c
	}
	var gz *C.mkhost_gz_index_cache
	if gc != nil {
		gz = gc.c
	}
	outs := make([]C.mkhost_layer_result, n)
	var st C.mkhost_layer_cache_stats
	var gst C.mkhost_gz_index_stats
	errBuf := (*C.char)(C.malloc(errLen))
	defer C.free(unsafe.Pointer(errBuf))
	hs := engineArray(engines)
	defer C.free(unsafe.Pointer(hs))
	if rc := C.mkhost_memfs_update_from_tars_multi(fs.m, hs, C.size_t(len(engines)), cache, gz, (**C.char)(unsafe.Pointer(ckeys)),
		C.int64_t(now), &specs[0], C.size_t(n), C.uint32_t(flags), &outs[0], &st, &gst, errBuf, errLen); rc != 0 {
		return nil, fmt.Errorf("%s", C.GoString(errBuf))
	}
	res := make([]LayerResult, n)
	for i := range outs {
		res[i] = toResult(&outs[i])
	}
	return res, nil
}
