/*
 * mkhost.h — host side ABOVE the mksnap C-ABI, in C++ (libmkhost.so), C interface.
 *
 * The reference's host code on this path is Go; no Go toolchain exists in the build image, so the
 * packer / walker / tar-header logic a cgo build would keep in Go is implemented here in C++ with the
 * reference's names, argument meaning and error behaviour, and is what the tests drive.  It contains NO
 * hashing: every digest comes from libmksnap (the GPU); without a device these calls fail.
 *
 *   mkhost_context_crc32      = addCopyStep.SetCacheID + calculateContextChecksum + checksumPathContents
 *                               reference lib/builder/step/add_copy_step.go:102-122,153-184,194-238
 *   mkhost_commit_copy_ops    = MemFS.AddLayerByCopyOps + commitLayer + tario.WriteEntry, digested on the GPU
 *                               reference lib/snapshot/mem_fs.go:276-289,353-433,509-569, mem_layer.go:152-244,
 *                               lib/tario/write.go:28-68, lib/builder/step/common.go:35-111
 *   mkhost_memfs_update_from_tar = MemFS.UpdateFromTarReader (untar=false) + go1.14 archive/tar Reader, with blob
 *                               verification (DiffID) and the chunk table on the GPU
 *                               reference lib/snapshot/mem_fs.go:165-255
 *   mkhost_encode_tar_header  = tario.WriteHeader + go1.14 archive/tar Writer.WriteHeader (USTAR / PAX)
 *   mkhost_describe_*         = the same host logic without a GPU (entry order / stream order as text), so the
 *                               CPU test-suite can diff it against the oracle.
 */
#ifndef MKHOST_H
#define MKHOST_H

#include <stddef.h>
#include <stdint.h>

#include "mksnap.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    const char *name;     /* as stored in tar.Header.Name (WriteHeader strips leading '/') */
    const char *linkname;
    int64_t mode;         /* perm | 04000 | 02000 | 01000, no type bits (FileInfoHeader) */
    int64_t uid, gid;
    int64_t size;
    int64_t mtime_ns;     /* truncated to the second by tario.WriteHeader (write.go:61) */
    char typeflag;        /* '0' reg, '1' link, '2' symlink, '5' dir, ... */
} mkhost_tar_header;

/* Returns the number of bytes written (512 for USTAR, 1536+ for PAX), 0 on error (cap too small /
 * field not encodable). */
size_t mkhost_encode_tar_header(const mkhost_tar_header *h, uint8_t *out, size_t cap);

/* snapshot.CopyOperation (lib/snapshot/copy_op.go:29-80).  srcs are relative to src_root (leading '/'
 * allowed, as TrimRoot produces them); dst is absolute or relative to work_dir. */
typedef struct {
    const char *src_root;
    const char *const *srcs;
    size_t n_srcs;
    const char *work_dir;
    const char *dst;
    int32_t uid, gid;
} mkhost_copy_op;

typedef struct {
    uint8_t tar_digest[32]; /* DigestPair.TarDigest bytes */
    uint8_t root[32];       /* chunk-table content address */
    uint64_t n_entries;     /* tar entries */
    uint64_t tar_bytes;     /* length of the uncompressed tar stream */
    uint64_t n_chunks, n_unique;
} mkhost_layer_result;

/* cacheID arithmetic of a COPY/ADD step from the build context.  prefix = seed+directive+args.
 * from_paths are the directive's sources (globbed and joined like resolveFromPaths).  *crc_out is what
 * checksum.Sum32() returns; format it with "%x" for the cacheID.  n_threads: file readers (0 = default). */
int mkhost_context_crc32(mksnap_t *eng, const void *prefix, size_t prefix_len, const char *context_dir,
                         const char *const *from_paths, size_t n_paths, int n_threads, uint32_t *crc_out,
                         uint64_t *stream_len_out, char *err, size_t errlen);

/* Incremental cacheID.  CRC-32 is linear: the context value is the XOR over its segments of pure(segment) shifted to
 * the segment's place, so pure(file content) -- 32 bits -- remembered from an earlier build lets an UNCHANGED file be
 * folded in on the host (mksnap_crc_add): no read, no copy to the device, no kernel.  "Unchanged" = same device, inode,
 * size, mtime and ctime (nanoseconds) as when the value was remembered -- stricter than the reference's own notion of an
 * unchanged file (tario.IsSimilarHeader: mtime to the second + size, lib/tario/compare.go:104-120).  Path strings,
 * link targets and the prefix are always streamed (tiny).  The result is bit-identical to mkhost_context_crc32 /
 * addCopyStep.SetCacheID whenever the remembered values are current; a cold cache degrades to the full computation and
 * fills itself.  The cache object belongs to the caller (one per build context); save/load keep it between processes (a
 * file that does not parse fails the load and leaves the cache as it was; a loaded file merges into the cache). */
typedef struct mkhost_crc_cache mkhost_crc_cache;
typedef struct {
    uint64_t files_total, files_reused; /* regular files in the stream / folded from the cache */
    uint64_t bytes_total, bytes_sent;   /* file bytes in the stream / file bytes that travelled to the device */
} mkhost_crc_cache_stats;
mkhost_crc_cache *mkhost_crc_cache_new(void);
void mkhost_crc_cache_free(mkhost_crc_cache *c);
uint64_t mkhost_crc_cache_size(const mkhost_crc_cache *c);
int mkhost_crc_cache_save(const mkhost_crc_cache *c, const char *path, char *err, size_t errlen);
int mkhost_crc_cache_load(mkhost_crc_cache *c, const char *path, char *err, size_t errlen);
int mkhost_context_crc32_cached(mksnap_t *eng, mkhost_crc_cache *cache, const void *prefix, size_t prefix_len,
                                const char *context_dir, const char *const *from_paths, size_t n_paths, int n_threads,
                                uint32_t *crc_out, uint64_t *stream_len_out, mkhost_crc_cache_stats *stats, char *err,
                                size_t errlen);

/* cacheID of every step of a build plan (processStagesAndAliases + createDockerfileSteps, lib/builder/build_plan.go:93-160,
 * build_stage.go:153-165: each step is seeded with the cacheID of the step before it), with the context read once for
 * the whole plan.  The sources of every COPY/ADD step are walked like mkhost_context_crc32 walks them; a file that
 * several steps cover (same path, device, inode, size, mtime and ctime) travels to the device once, and so does each
 * distinct path string and link target.  The device then folds every step's stream out of those values (mksnap_crc_fold)
 * and the host prepends seed + directive + args step by step (mksnap_crc_prepend).  ids_out[i] is what
 * checksum.Sum32() returns for step i; "%x" of it is the step's cacheID and the next step's seed.  A plan with more
 * COPY/ADD steps than the engine has stream slots runs as consecutive sessions; a file read in one is not read again.
 * With a cache, files it vouches for are not read at all and every file that travelled is remembered, like
 * mkhost_context_crc32_cached.  stats: files_total / bytes_total count every occurrence over all steps, files_reused
 * the occurrences folded from the cache, bytes_sent each file that travelled once.  Steps come in plan order, the
 * stages in order, with the stage of a remote image that a COPY --from names (build_plan.go:142-152) in front of the
 * stage that names it. */
#define MKHOST_STEP_COPY 1        /* addCopyStep.SetCacheID (add_copy_step.go:102-122): directive "COPY"/"ADD"; a
                                     non-empty from_stage (COPY --from) hashes no content (add_copy_step.go:109-113) */
#define MKHOST_STEP_FROM 2        /* FromStep.SetCacheID: crc32(seed + "FROM" + args), args = image (from_step.go:79-83) */
#define MKHOST_STEP_BASE 3        /* baseStep.SetCacheID: crc32(seed + directive + args + "true"/"false" of commit)
                                     (base_step.go:62-67): RUN, ENV, CMD, ... */
#define MKHOST_STEP_REMOTE_FROM 4 /* the FROM step of a remote-image stage (newRemoteImageStage, build_stage.go:78-108).
                                     The stage that names the image was seeded before it was inserted: a run of these
                                     chains from the seed of the step in front of them, and the step after the run takes
                                     that same seed again. */
typedef struct {
    uint32_t kind;
    int32_t commit;             /* MKHOST_STEP_BASE */
    const char *directive;      /* COPY / BASE */
    const char *args;           /* as the reference prints them; the image of a FROM */
    const char *from_stage;     /* COPY: NULL or "" = sources from the context */
    const char *const *from_paths;
    size_t n_paths;
} mkhost_plan_step;
int mkhost_plan_cache_ids(mksnap_t *eng, mkhost_crc_cache *cache, const char *seed, const char *context_dir,
                          const mkhost_plan_step *steps, size_t n_steps, int n_threads, uint32_t *ids_out,
                          mkhost_crc_cache_stats *stats, char *err, size_t errlen);

/* Commit one layer from copy operations against an EMPTY MemFS rooted at root_dir (FROM scratch): packs
 * the sorted entries as a tar stream into one arena, digests it (TarDigest) and chunks every regular
 * file (chunk table).  now_unix = clk.Now() for synthesized ancestors (mem_fs.go:562). */
int mkhost_commit_copy_ops(mksnap_t *eng, const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops,
                           size_t n_ops, int n_threads, mkhost_layer_result *out, char *err, size_t errlen);
/* Same, and additionally writes the uncompressed layer tar (the packed arenas, byte for byte what
 * tar.Writer would have produced) to tar_fd -- the stream the Go side feeds to pgzip (common.go:47-55,
 * SURVEY section 8f-1).  SHA-256 of those bytes == out->tar_digest. */
int mkhost_commit_copy_ops_to_fd(mksnap_t *eng, const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops,
                                 size_t n_ops, int n_threads, int tar_fd, mkhost_layer_result *out, char *err,
                                 size_t errlen);
/* flags for mkhost_commit_copy_ops_ex */
#define MKHOST_NO_TAR_DIGEST 1u /* leave TarDigest to the caller (Go's sha256.New() fed from the same bytes, see
                                   INTEGRATION.md section 3): out->tar_digest is zeroed, no serial stream is submitted */
/* MemFS entry points only (they need a tree to remember into):
 * MKHOST_FILE_DIGESTS  also hash every regular file of the layer (one serial SHA-256 stream per file, stream slots
 *                      1..n; the engine needs max_extents > n) and remember the digest in the tree.
 * MKHOST_SCAN_CONTENT  mkhost_memfs_commit_scan: content-aware change detection (SURVEY section 8f-3).  Files the
 *                      reference's IsSimilarHeader calls unchanged (same mtime second, size, mode, owner) are
 *                      re-hashed on the GPU and compared with the remembered digest; a difference puts the file into
 *                      the layer.  Removes the need for the sync() + 1 s sleep of mem_fs.go:291-311.  Implies
 *                      MKHOST_FILE_DIGESTS.  No reference counterpart: with the flag clear the scan is the reference's. */
#define MKHOST_FILE_DIGESTS 2u
#define MKHOST_SCAN_CONTENT 4u
int mkhost_commit_copy_ops_ex(mksnap_t *eng, const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops,
                              size_t n_ops, int n_threads, int tar_fd, uint32_t flags, mkhost_layer_result *out,
                              char *err, size_t errlen);

/* Persistent mirror of snapshot.MemFS (lib/snapshot/mem_fs.go:60-83): layers accumulate in the merged tree, later
 * layers contain only entries whose header is not "similar" (lib/tario/compare.go) to what the tree holds, scans
 * emit whiteouts for children that vanished (mem_fs.go:459-480), `blacklist` as in NewMemFS(clk, root, blacklist). */
typedef struct mkhost_memfs mkhost_memfs;
mkhost_memfs *mkhost_memfs_new(const char *root_dir, const char *const *blacklist, size_t n_blacklist, char *err,
                               size_t errlen);
void mkhost_memfs_free(mkhost_memfs *m);
/* SHA-256 of the content the tree remembers for the regular file at dst (MKHOST_FILE_DIGESTS / MKHOST_SCAN_CONTENT
 * commits and ingests); returns 0 and fills out, or 1 when nothing is remembered for that path. */
int mkhost_memfs_file_digest(mkhost_memfs *m, const char *dst, uint8_t out[32]);
/* AddLayerByCopyOps / AddLayerByScan followed by commitLayer on the GPU (flags: MKHOST_NO_TAR_DIGEST). */
int mkhost_memfs_commit_copy_ops(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops,
                                 int n_threads, int tar_fd, uint32_t flags, mkhost_layer_result *out, char *err,
                                 size_t errlen);
/* Incremental layer commit.  Chunks never span files, so a file's chunk digests depend on its bytes (and the CDC
 * parameters) alone, and the chunk table is the sorted-unique multiset of all of them: the digests of an UNCHANGED file,
 * remembered from an earlier commit, can join the table (mksnap_chunks_add) instead of the file being chunked again.
 * "Unchanged" is what it is for the incremental cacheID: same device, inode, size, mtime and ctime (nanoseconds) as when
 * the file was read.  The result -- entries, tar bytes to tar_fd, TarDigest, root, n_chunks, n_unique -- is that of
 * mkhost_memfs_commit_copy_ops with the same flags, bit for bit, whenever the remembered digests are current; with
 * cache == NULL this IS mkhost_memfs_commit_copy_ops.  What is saved depends on the mode: TarDigest is one serial SHA-256
 * chain over every byte, so by default an unchanged file still travels to the device (the chain reads it) and only the
 * scan and chunk SHA-256 skip it; under MKHOST_NO_TAR_DIGEST nothing on the device needs it, so its bytes do not cross
 * PCIe (mksnap_arena_submit_spans), and without tar_fd and MKHOST_MATERIALIZE it is not even read.  Every file chunked
 * by the commit is remembered.  The cache records the CDC parameters (mksnap_get_cdc); used with an engine cut under
 * others it starts over, nothing is an error.  One cache per build context, owned by the caller; save/load keep it
 * between processes (a file that does not parse fails the load and leaves the cache as it was; a loaded file merges
 * into the cache, or replaces it when it was saved under other CDC parameters).  stats: regular files of the layer and
 * their bytes, files taken from the cache, bytes chunked on the device, file bytes copied to the device. */
typedef struct mkhost_chunk_cache mkhost_chunk_cache;
typedef struct {
    uint64_t files_total, files_reused;
    uint64_t bytes_total, bytes_chunked, bytes_uploaded;
} mkhost_chunk_cache_stats;
mkhost_chunk_cache *mkhost_chunk_cache_new(void);
void mkhost_chunk_cache_free(mkhost_chunk_cache *c);
uint64_t mkhost_chunk_cache_size(const mkhost_chunk_cache *c);
int mkhost_chunk_cache_save(const mkhost_chunk_cache *c, const char *path, char *err, size_t errlen);
int mkhost_chunk_cache_load(mkhost_chunk_cache *c, const char *path, char *err, size_t errlen);
int mkhost_memfs_commit_copy_ops_cached(mkhost_memfs *m, mksnap_t *eng, mkhost_chunk_cache *cache, int64_t now_unix,
                                        const mkhost_copy_op *ops, size_t n_ops, int n_threads, int tar_fd, uint32_t flags,
                                        mkhost_layer_result *out, mkhost_chunk_cache_stats *stats, char *err, size_t errlen);
int mkhost_memfs_commit_scan(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, int n_threads, int tar_fd, uint32_t flags,
                             mkhost_layer_result *out, char *err, size_t errlen);
/* Several consecutive layers of ONE build committed in one engine session.  Equivalent to calling
 * mkhost_memfs_commit_copy_ops once per layer, in order (same entries, same tar bytes to each layer's tar_fd, same
 * TarDigest per layer) -- but every pinned arena carries a piece of EVERY unfinished layer, so the serial SHA-256
 * chains (one per layer, lib/builder/step/common.go:44-55) advance together on the device instead of one after the
 * other.  This is what makes TarDigest on the GPU worthwhile: on an H100 one chain runs at ~0.06 GB/s, 256 chains at ~15 GB/s.
 * The reference commits layer by layer (build_node.go:102-107); COPY/ADD steps that do not modify the file system
 * (no RUN in between) can be deferred and committed together, which is what a cgo caller would do (INTEGRATION.md).
 * outs[i].tar_digest / tar_bytes / n_entries are per layer; root / n_chunks / n_unique describe the chunk table of the
 * whole batch (one session).  flags: MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS.  tar_fd < 0: that layer's tar is not
 * emitted.  This is mkhost_memfs_commit_layers_cached with cache == NULL. */
typedef struct {
    const mkhost_copy_op *ops;
    size_t n_ops;
    int tar_fd;
} mkhost_layer_spec;
int mkhost_memfs_commit_layers(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_layer_spec *layers,
                               size_t n_layers, int n_threads, uint32_t flags, mkhost_layer_result *outs, char *err,
                               size_t errlen);
/* Batched incremental layer commit.  The result equals calling mkhost_memfs_commit_copy_ops_cached once per layer, in
 * order, with the same cache and flags: the same tree and the same remembered file digests (a destination written by
 * two layers keeps the later layer's digest), the same bytes to each layer's tar_fd, the same outs[i].tar_digest,
 * n_entries and tar_bytes, and the same cache contents afterwards (mkhost_chunk_cache_save writes the same bytes).  Two
 * things differ by design: outs[i].root / n_chunks / n_unique describe the chunk table of the whole batch, as for
 * mkhost_memfs_commit_layers; and every lookup uses the cache as it stood when the call started, so a source that two
 * layers copy and the cache does not yet hold is chunked in both (the table is sorted and unique: the root is the
 * same).  stats adds up over the batch and counts every occurrence of a file (files_reused included).  cache == NULL:
 * no cache.  flags: MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS; any other flag is refused.
 * Stream slots: layer i's TarDigest chain is slot i; under MKHOST_FILE_DIGESTS every regular file with content in the
 * batch takes one slot from n_layers on.  A batch whose layers plus such files exceed mksnap_limits.max_streams is
 * refused before anything is read or submitted.
 * Deliberately not supported: an entry larger than one arena is refused ("exceeds the arena"), since it would have to
 * stay open across submits next to the other layers' pieces; and MKHOST_MATERIALIZE, since the copier mode (--chown or
 * not) belongs to each step and mkhost_layer_spec has no field for it. */
int mkhost_memfs_commit_layers_cached(mkhost_memfs *m, mksnap_t *eng, mkhost_chunk_cache *cache, int64_t now_unix,
                                      const mkhost_layer_spec *layers, size_t n_layers, int n_threads, uint32_t flags,
                                      mkhost_layer_result *outs, mkhost_chunk_cache_stats *stats, char *err, size_t errlen);
/* the same two without a GPU: entry list as text (format below); they DO merge the layer into the tree */
size_t mkhost_memfs_describe_copy_ops(mkhost_memfs *m, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops, char *out,
                                      size_t cap, char *err, size_t errlen);
size_t mkhost_memfs_describe_scan(mkhost_memfs *m, int64_t now_unix, char *out, size_t cap, char *err, size_t errlen);

/* UpdateFromTarReader(r, untar=false) (lib/snapshot/mem_fs.go:165-255; FROM / cache-hit path, from_step.go:118-134):
 * merge a layer tar read from tar_fd (file or pipe; uncompressed, or gzip with MKHOST_GUNZIP below) into the tree,
 * hard links in a second pass, nothing written to disk.  The stream goes through the pinned arenas once:
 * out->tar_digest = SHA-256 of every byte read up to EOF (the layer's DiffID: compare with the image config to
 * verify the pulled blob, lib/docker/image/digest.go:42-50), out->root / n_chunks / n_unique = chunk table of the
 * regular-file members (so base layers join the chunk-granular dedup), out->n_entries = headers merged (the
 * count the reference logs).  flags: MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS, MKHOST_UNTAR, MKHOST_GUNZIP.  A regular-file member
 * larger than one arena travels in pieces (MKSNAP_X_MORE / MKSNAP_X_CONT); only MKHOST_UNTAR, which writes a member
 * from one contiguous body, still needs every member to fit an arena. */
int mkhost_memfs_update_from_tar(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, int tar_fd, uint32_t flags,
                                 mkhost_layer_result *out, char *err, size_t errlen);
/* the same merge without a GPU: merged layer as text (format below) */
size_t mkhost_memfs_describe_update_from_tar(mkhost_memfs *m, int64_t now_unix, int tar_fd, char *out, size_t cap,
                                             char *err, size_t errlen);
/* MKHOST_UNTAR (flag of mkhost_memfs_update_from_tar and of the _ex describe): UpdateFromTarReader(r, untar=true) --
 * every member is also written under the root (untarOneItem, lib/snapshot/mem_fs.go:574-716: whiteouts delete,
 * existing directories are updated in place, similar entries are left alone, anything else is replaced; hard links
 * last; tario.ApplyHeader sets owner, mode and mtime; parent directory mtimes are restored).  On the GPU path the file
 * bodies are written straight from the arena that is being digested. */
#define MKHOST_UNTAR 32u
/* MKHOST_GUNZIP (flag of mkhost_memfs_update_from_tar): tar_fd carries the blob as the image store holds it, gzip
 * (tario.NewGzipReader + UpdateFromTarReader, from_step.go:118-134, build_node.go:131-148).  The blob is read whole and
 * decompressed on the device (mksnap_gunzip_open / _read, one window at a time); everything downstream is that of the
 * uncompressed stream: the DiffID is the SHA-256 of the decompressed tar.  Combines with every other flag.  Malformed
 * gzip data fails the call.  The describe functions read uncompressed tars only. */
#define MKHOST_GUNZIP 64u
size_t mkhost_memfs_describe_update_from_tar_ex(mkhost_memfs *m, int64_t now_unix, int tar_fd, uint32_t flags, char *out,
                                                size_t cap, char *err, size_t errlen);

/* A run of layers applied back to back in ONE engine session (FromStep.Execute merging the layers of the base image,
 * from_step.go:118-134; buildNode.Build applying the layers of cached steps, build_node.go:72-79,133-148).  The result
 * equals n_layers calls of mkhost_memfs_update_from_tar in order: the same tree, the same files on disk under
 * MKHOST_UNTAR, the same remembered file digests, and per layer the same outs[i].tar_digest, n_entries and tar_bytes;
 * outs[i].root / n_chunks / n_unique describe the chunk table of the whole run (one session).  The layers are read and
 * merged strictly in order, but their DiffID chains are hashed together: layer i's tar stream is stream slot i, a
 * MKSNAP_R_DEFER stream, so its bytes wait in the engine's stream log and every chain of the run advances in the same
 * K4 launches (one chain on an H100 runs at ~0.06 GB/s).  The call reserves the stream log itself (1 GiB) and leaves it
 * reserved on the handle.  flags: MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS (per-file streams take the slots after
 * n_layers and stay inline; the engine needs max_extents > n_layers), MKHOST_UNTAR.  layers[i].flags: MKHOST_GUNZIP
 * for a gzip blob.  The chunks of the whole run share one session's table (mksnap_limits.max_chunks).  A run with
 * more layers than stream slots fails before anything is read.  If layer k fails, layers
 * before k stay merged in the tree and on disk, as after separate calls; the call returns -1 and outs is unspecified. */
typedef struct {
    int tar_fd;
    uint32_t flags; /* MKHOST_GUNZIP: this blob is gzip */
} mkhost_tar_spec;
int mkhost_memfs_update_from_tars(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_tar_spec *layers,
                                  size_t n_layers, uint32_t flags, mkhost_layer_result *outs, char *err, size_t errlen);

/* Block indexes of single-member gzip layers, remembered between builds.  A registry layer is one gzip member without
 * flush points, which mksnap_gunzip_open decodes on one GPU thread; mksnap_gunzip_open_indexed records where its DEFLATE
 * blocks start on the first decode, and later opens of the same blob take those points and decode in parallel.  The
 * cache maps a caller key (makisu: the image store's file name, descriptor.Digest.Hex()) to the blob length and its
 * points; an entry whose length differs from the blob's, or whose points are not ascending and inside the blob, is
 * ignored.  A point the engine cannot link costs speed only, never output or an error, so a stale or foreign entry is
 * harmless.  One cache per image store, owned by the caller; save/load keep it between processes (a file that does not
 * parse fails the load and leaves the cache as it was).
 * The _indexed calls equal mkhost_memfs_update_from_tar / _tars, except that each layer flagged MKHOST_GUNZIP that has a
 * key (key, keys[i]; NULL = none) is opened by mksnap_gunzip_open_indexed with the cached points, and after the open
 * succeeds its entry is replaced with what mksnap_gunzip_get_index returns.  With cache == NULL they are the plain
 * calls.  stats (may be NULL) adds up over the call: blobs opened indexed, of them with a cached index, and the engine's
 * points_given / points_linked / points_recorded. */
typedef struct mkhost_gz_index_cache mkhost_gz_index_cache;
typedef struct {
    uint64_t blobs, blobs_with_index;
    uint64_t points_given, points_linked, points_recorded;
} mkhost_gz_index_stats;
mkhost_gz_index_cache *mkhost_gz_index_cache_new(void);
void mkhost_gz_index_cache_free(mkhost_gz_index_cache *c);
uint64_t mkhost_gz_index_cache_size(const mkhost_gz_index_cache *c);
int mkhost_gz_index_cache_save(const mkhost_gz_index_cache *c, const char *path, char *err, size_t errlen);
int mkhost_gz_index_cache_load(mkhost_gz_index_cache *c, const char *path, char *err, size_t errlen);
int mkhost_memfs_update_from_tar_indexed(mkhost_memfs *m, mksnap_t *eng, mkhost_gz_index_cache *cache, const char *key,
                                         int64_t now_unix, int tar_fd, uint32_t flags, mkhost_layer_result *out,
                                         mkhost_gz_index_stats *stats, char *err, size_t errlen);
int mkhost_memfs_update_from_tars_indexed(mkhost_memfs *m, mksnap_t *eng, mkhost_gz_index_cache *cache,
                                          const char *const *keys, int64_t now_unix, const mkhost_tar_spec *layers,
                                          size_t n_layers, uint32_t flags, mkhost_layer_result *outs,
                                          mkhost_gz_index_stats *stats, char *err, size_t errlen);

/* Incremental layer ingest.  What a run of layers takes from a blob -- the member headers the merge reads, the DiffID,
 * the tar length, the per-file SHA-256 values and the chunk digests of its files -- depends only on the blob's bytes
 * and the CDC parameters, and the store files of base-image and cache-hit layers are content-addressed and almost
 * never change between builds.  The layer cache remembers those values per caller key (makisu: the image store's file
 * name, descriptor.Digest.Hex()), so an unchanged blob is REPLAYED: its remembered members go through the same merge
 * (and, under MKHOST_FILE_DIGESTS, leave their remembered digests in the tree), its chunk digests join the session's
 * table through mksnap_chunks_add and its DiffID comes from the record.  No byte of it is read, decompressed, uploaded
 * or hashed; a replayed gzip layer also leaves its gz entry as it was.
 * mkhost_memfs_update_from_tars_cached equals mkhost_memfs_update_from_tars_indexed(m, eng, gz, keys, ...) with the same
 * arguments -- tree, remembered file digests, outs (DiffID, n_entries, tar_bytes per layer; root, n_chunks, n_unique of
 * the run), refusals, and the state a failing layer leaves -- and with lc == NULL it is that call.  keys[i] == NULL:
 * no cache for layer i.  An entry is replayed only when tar_fd is a regular file read from offset 0 whose device, inode,
 * size, mtime and ctime (nanoseconds) are those it was recorded from, its MKHOST_GUNZIP flag is the recorded one, and
 * it holds what the call needs (a DiffID unless MKHOST_NO_TAR_DIGEST, file digests under MKHOST_FILE_DIGESTS); under
 * MKHOST_UNTAR nothing is replayed, since the files must be written.  Every other layer with a key and a regular file
 * read from offset 0 is ingested as usual and recorded (replacing the entry under its key) once the whole run has
 * finished; a call that fails records nothing.  A pipe is never replayed nor recorded.  The cache records the CDC
 * parameters (mksnap_get_cdc); used with an engine cut under others it starts over.  One cache per image store, owned
 * by the caller; save/load keep it between processes (a file that does not parse fails the load and leaves the cache
 * as it was).  stats (may be NULL): layers of the call, of them replayed and recorded, bytes read from the layers' fds,
 * chunk rows appended for replayed layers. */
typedef struct mkhost_layer_cache mkhost_layer_cache;
typedef struct {
    uint64_t layers, layers_replayed, layers_recorded;
    uint64_t blob_bytes_read; /* bytes read from the layers' fds by this call */
    uint64_t chunks_appended; /* rows added through mksnap_chunks_add */
} mkhost_layer_cache_stats;
mkhost_layer_cache *mkhost_layer_cache_new(void);
void mkhost_layer_cache_free(mkhost_layer_cache *c);
uint64_t mkhost_layer_cache_size(const mkhost_layer_cache *c);
int mkhost_layer_cache_save(const mkhost_layer_cache *c, const char *path, char *err, size_t errlen);
int mkhost_layer_cache_load(mkhost_layer_cache *c, const char *path, char *err, size_t errlen);
int mkhost_memfs_update_from_tars_cached(mkhost_memfs *m, mksnap_t *eng, mkhost_layer_cache *lc, mkhost_gz_index_cache *gz,
                                         const char *const *keys, int64_t now_unix, const mkhost_tar_spec *layers,
                                         size_t n_layers, uint32_t flags, mkhost_layer_result *outs,
                                         mkhost_layer_cache_stats *stats, mkhost_gz_index_stats *gz_stats, char *err,
                                         size_t errlen);

/* CopyOperation.Execute (lib/snapshot/copy_op.go:82-147) with fileio.Copier (lib/fileio/copy.go): what a COPY/ADD step
 * does to the file system when it runs with --modifyfs.  op->dst is used as the on-disk destination exactly like the
 * reference does (resolved against op->work_dir when relative).  mode selects the Copier of copy_op.go:98-124:
 * MKHOST_COPY_CHOWN (--chown: op->uid/gid), MKHOST_COPY_INTERNAL (--from=<stage>: no blacklist, owners preserved),
 * MKHOST_COPY_PRESERVE_OWNER (--from --archive).  mode 0 = copy from the build context (owner root).
 * MKHOST_COPY_DEFERRED runs the traversal (directories, symlinks, chmod of existing targets) first and writes the
 * regular files afterwards from buffers read once -- the path mkhost_memfs_commit_copy_ops(…, MKHOST_MATERIALIZE)
 * takes with its arena; here the buffers are plain reads, so the deferred machinery can be exercised without a GPU. */
#define MKHOST_COPY_CHOWN 1u
#define MKHOST_COPY_INTERNAL 2u
#define MKHOST_COPY_PRESERVE_OWNER 4u
#define MKHOST_COPY_DEFERRED 8u
int mkhost_copy_op_execute(const mkhost_copy_op *op, uint32_t mode, const char *const *blacklist, size_t n_blacklist,
                           char *err, size_t errlen);
/* evalSymlinks(p, srcRoot) (lib/snapshot/utils.go:249-324): the root-relative path after following every symlink on
 * it, links confined to src_root (absolute targets must carry the root prefix, which is trimmed), at most 255 links.
 * Both CopyOperation.Execute (copy_op.go:86) and MemFS.addToLayer (mem_fs.go:380) resolve each source through it.
 * Returns the number of bytes needed including NUL (nothing written if > cap), 0 on error. */
size_t mkhost_eval_symlinks(const char *path, const char *src_root, char *out, size_t cap, char *err, size_t errlen);
/* flag for mkhost_memfs_commit_copy_ops: also perform the copy (as mkhost_copy_op_execute with `copy_mode` 0 / CHOWN
 * decided by MKHOST_MATERIALIZE_CHOWN), writing regular files from the arena the layer is packed in: the context is
 * read once for the copy, the layer, its digest and its chunk table (SURVEY section 8f-4). */
#define MKHOST_MATERIALIZE 8u
#define MKHOST_MATERIALIZE_CHOWN 16u

/* cache.Manager wire format (lib/cache/cache_manager.go:34-35,239-252).  key = "makisu_builder_cache_" + cacheID;
 * entry = "<tarHex>,<gzipHex>" (createEntry), or "MAKISU_CACHE_EMPTY" for a nil pair (tar_hex == NULL).
 * parse = parseEntry: error when there is no ',', otherwise SplitN(entry, ",", 2) -- no hex validation, like
 * the reference.  Because old readers keep everything after the first ',' as the gzip digest, the chunk-table
 * root cannot ride in the same value: it is stored under its own key "<key>_chunks" = "<rootHex>,<n_unique>",
 * which readers that do not know it never fetch (SURVEY section 8f-1: "old readers must still parse").
 * All return the number of bytes needed including NUL (nothing written if > cap), 0 on error. */
size_t mkhost_cache_key(const char *cache_id, int chunk_table, char *out, size_t cap);
size_t mkhost_cache_entry_create(const char *tar_hex, const char *gzip_hex, char *out, size_t cap);
int mkhost_cache_entry_parse(const char *entry, char *tar_digest, size_t tar_cap, char *gzip_digest, size_t gzip_cap,
                             char *err, size_t errlen);
size_t mkhost_cache_chunk_entry_create(const uint8_t root[32], uint64_t n_unique, char *out, size_t cap);
int mkhost_cache_chunk_entry_parse(const char *entry, uint8_t root[32], uint64_t *n_unique, char *err, size_t errlen);

/* No-GPU introspection for the CPU tests: one line per item, '\n' separated, NUL terminated.
 *   stream : "P <relpath>" | "L <target>" | "F <size> <abs path>"   in CRC stream order
 *   layer  : "<typeflag> <mode octal> <uid> <gid> <size> <mtime> <dst> <hdr.Name> <src>"  in tar order
 * Return the number of bytes needed (including NUL); if > cap nothing is written. */
size_t mkhost_describe_context_stream(const char *context_dir, const char *const *from_paths, size_t n_paths,
                                      char *out, size_t cap, char *err, size_t errlen);
size_t mkhost_describe_layer(const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops,
                             char *out, size_t cap, char *err, size_t errlen);

#ifdef __cplusplus
}
#endif
#endif
