/*
 * mksnap.h — C-ABI of libmksnap.so: the H100-native snapshot+hash engine that
 * replaces the CPU arithmetic on makisu's build-context fingerprint and layer
 * digest path.  Plain C, plain pointers and sizes; no torch / C++ types.
 *
 * The reference (uber/makisu @5fdc8f4) has NO FFI on this path: it is direct Go
 * calls inside a CGO_ENABLED=0 binary (reference Makefile:46-49).  The entry
 * points below are what a cgo shim would bind at the three seams SURVEY.md
 * section 8(b) identifies; each one cites the reference code it replaces.  The Go-side
 * stubs are shown in INTEGRATION.md.
 *
 * Model: a handle owns one CUDA device, its streams, a ring of pinned host
 * arenas and device arena slots.  A *session* (begin ... finish) digests one
 * build context / layer: the host packs file bytes into an arena in layer-tar
 * order (512-byte aligned, zero padded -- i.e. the arena *is* the tar stream),
 * describes what to hash with extent / range tables, and submits.  All
 * arithmetic runs on the device; there is no CPU fallback: every call fails
 * with MKSNAP_E_CUDA if no device is usable.
 *
 * Threading: one session per handle at a time, calls on a handle must be
 * serialised by the caller (the reference calls these seams from one goroutine
 * per build: lib/builder/build_plan.go:174, lib/stream/multi_writer.go:60);
 * different handles may be used concurrently.  Every entry point does its own
 * cudaSetDevice, so a goroutine may migrate between OS threads.
 *
 * Errors: 0 = ok, negative = MKSNAP_E_*; text via mksnap_last_error().  A Go
 * wrapper maps them to fmt.Errorf("...: %s", err) like lib/builder/step/common.go:59.
 */
#ifndef MKSNAP_H
#define MKSNAP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MKSNAP_ABI_VERSION 1

enum {
    MKSNAP_OK = 0,
    MKSNAP_E_INVAL = -1,    /* bad argument / misuse */
    MKSNAP_E_CUDA = -2,     /* CUDA runtime / driver failure, or no device */
    MKSNAP_E_NOMEM = -3,    /* allocation failed */
    MKSNAP_E_CAPACITY = -4, /* batch / table exceeds a configured capacity */
    MKSNAP_E_STATE = -5,    /* call out of sequence */
    MKSNAP_E_NCCL = -6,     /* NCCL unavailable or failed */
    MKSNAP_E_DATA = -7      /* malformed compressed data */
};

typedef struct mksnap mksnap_t;

/* Content-defined chunking parameters (DESIGN.md section 3; no reference counterpart). */
/* Largest max_size mksnap_create accepts: the big-file cut selection works in 16 MiB windows of 32-bit offsets and
 * computes (offset <= 16 MiB) + max_size, which must not wrap. */
#define MKSNAP_CDC_MAX_SIZE_LIMIT 0xFEFFFFFFu /* 2^32 - 2^24 - 1 */
typedef struct {
    uint32_t min_size;    /* default 4096   (must be >= 64)                     */
    uint32_t normal_size; /* default 16384  (strict mask below, loose at/after) */
    uint32_t max_size;    /* default 131072 (at most MKSNAP_CDC_MAX_SIZE_LIMIT)  */
    uint32_t strict_bits; /* default 16: candidate iff the top bits of roll32 are all ones */
    uint32_t loose_bits;  /* default 12                                         */
} mksnap_cdc_params;

typedef struct {
    int32_t device;              /* CUDA ordinal                                      */
    uint32_t n_host_arenas;      /* pinned staging arenas; 0 = device-resident use    */
    uint64_t host_arena_bytes;   /* capacity of each pinned arena                     */
    uint64_t device_arena_bytes; /* capacity of each device arena slot                */
    uint32_t n_device_slots;     /* 0 = auto (2 if host arenas are used, else 1)      */
    uint32_t reserved0;
    uint64_t max_extents;        /* per submit                                        */
    uint64_t max_chunks;         /* per session; 0 = device_arena_bytes/min_size + 3*max_extents + 64 */
    mksnap_cdc_params cdc;       /* all-zero = defaults                               */
} mksnap_config;

/* One contiguous piece of an arena.  Offsets are relative to the arena that is
 * being submitted and must be multiples of 16. */
#define MKSNAP_X_CRC 1u /* part of the CRC-32 context stream */
#define MKSNAP_X_CDC 2u /* chunk + digest this extent as one file */
/* A file larger than one arena (tario.WriteEntry copies any size, lib/tario/write.go:45): its pieces travel in
 * consecutive submits.  Every piece but the last carries MKSNAP_X_MORE, must be the LAST CDC extent of its submit and
 * states in `reserved` how many bytes of the file follow in later submits (saturate at 0xFFFFFFFF); every piece but
 * the first carries MKSNAP_X_CONT, must be the FIRST CDC extent of the next submit and start at arena offset >=
 * mksnap_limits.carry_bytes (the engine copies the chunk left open at the end of the previous piece in front of it).
 * Chunks and digests are exactly those of the undivided file.  CRC extents need none of this: they split anywhere. */
#define MKSNAP_X_MORE 4u
#define MKSNAP_X_CONT 8u
typedef struct {
    uint64_t arena_off;
    uint64_t len;
    /* MKSNAP_X_CRC: number of context-stream bytes that FOLLOW this extent's last
     * byte (over the whole session, across submits).  The stream is the byte
     * sequence the reference feeds to crc32 in lib/builder/step/add_copy_step.go:104-119,
     * 194-238: seed+directive+args, then relpath / link target / file content
     * per walked path, no separators. */
    uint64_t crc_suffix;
    uint32_t flags;
    uint32_t reserved; /* MKSNAP_X_MORE: bytes of this file in later submits (saturated); otherwise 0 */
} mksnap_extent;

/* A piece of a serial SHA-256 stream (replaces the tarDigester sha256.New() sink of
 * lib/builder/step/common.go:44-55: every tar.Writer write lands in one stream).  arena_off multiple of 16.
 * `stream` is a caller-chosen slot in [0, max_extents): the digest of the stream lands in row `stream` of the
 * stream-digest table.  A stream may span several submits (a layer tar larger than one arena): every piece but
 * the last carries MKSNAP_R_MORE and a length that is a non-empty multiple of 64; the device keeps the SHA-256
 * midstate between submits.  The last piece may be empty (every byte went out in earlier pieces).  At most one piece
 * per stream per submit.  mksnap_finish refuses a session whose stream is still open (its last piece carried
 * MKSNAP_R_MORE) with MKSNAP_E_STATE; the session stays open, so the final piece can still be submitted.  A slot may
 * carry a new stream once its previous stream has finished. */
#define MKSNAP_R_MORE 1u
/* A piece of a DEFERRED stream: its bytes are copied on the device from the arena slot into the handle's stream log
 * (mksnap_reserve_stream_log) before the slot is recycled, and hashed later, together with the deferred pieces of every
 * other stream, so that many chains advance in the same K4 launch even when the caller fills arenas one stream after
 * the other (layers applied in order).  The log is hashed ("flushed") at mksnap_finish at the latest, and earlier when
 * a deferred piece does not fit in the room left: the pending pieces are grouped by stream in log order, adjacent
 * pieces of one stream merged, and K4 runs once per round (the r-th remaining piece of every stream).  A deferred piece
 * larger than the whole log, and every deferred piece of a handle without a log, is hashed in its own submit.
 * Every other rule of this table is unchanged and digests are bit-identical to the inline path.  All pieces of one
 * stream carry the flag or none does (MKSNAP_E_INVAL otherwise); deferred and inline streams may share a session.
 * The row of a deferred stream is readable after mksnap_finish only. */
#define MKSNAP_R_DEFER 2u
typedef struct {
    uint64_t arena_off;
    uint64_t len;
    uint32_t stream;
    uint32_t flags;
} mksnap_range;

typedef struct {
    uint32_t crc_pure;      /* GF(2)-linear accumulator; use mksnap_ctx_crc32() */
    uint32_t reserved;
    uint64_t crc_bytes;     /* context-stream bytes seen */
    uint64_t cdc_bytes;     /* bytes chunked             */
    uint64_t n_files;       /* MKSNAP_X_CDC extents      */
    uint64_t n_chunks;
    uint64_t n_unique;      /* rows of the sorted-unique table */
    uint8_t root[32];       /* fan-out-256 Merkle root of the table = layer content address */
    uint64_t n_streams;     /* rows of the stream-digest table (highest finished stream slot + 1) */
} mksnap_result;

typedef struct {
    /* device time of the most recent submit, CUDA events on the compute stream */
    float ms_total;
    float ms_crc;     /* K0  crc32 extents          */
    float ms_scan;    /* K1  rolling-hash candidate scan */
    float ms_select;  /* K1b cut selection          */
    float ms_sha;     /* K2  per-chunk SHA-256      */
    float ms_stream;  /* K4  serial-stream SHA-256  */
    float ms_h2d;     /* host->device copy (copy stream) */
    /* device time of the most recent finish */
    float ms_sort;    /* K3  radix sort + unique    */
    float ms_root;    /* Merkle root                */
    float ms_gather;  /* NCCL all-gather + merge    */
    uint64_t kernel_launches; /* kernels launched by this handle since create */
    uint64_t h2d_bytes;       /* since create */
    uint64_t d2h_bytes;       /* since create */
    float ms_flush;           /* K4 rounds of the most recent stream-log flush (MKSNAP_R_DEFER) */
} mksnap_stats_t;

/* ---- lifetime --------------------------------------------------------- */
int mksnap_abi_version(void);
int mksnap_create(const mksnap_config *cfg, mksnap_t **out);
void mksnap_destroy(mksnap_t *h);
const char *mksnap_last_error(const mksnap_t *h); /* h may be NULL: create() errors */

/* ---- session ---------------------------------------------------------- */
/* Start digesting a new context/layer: clears the CRC accumulator and the
 * chunk table.  Replaces crc32.NewIEEE() (add_copy_step.go:104) +
 * sha256.New() (common.go:44-45). */
int mksnap_begin(mksnap_t *h);

/* Borrow a C-owned pinned host arena (cudaHostAlloc).  Blocks until one is
 * free.  The caller writes file bytes into it (the Go side through
 * unsafe.Slice; no Go-heap pointer crosses the boundary) and hands it back
 * with mksnap_arena_submit. */
int mksnap_arena_acquire(mksnap_t *h, void **host_ptr, uint64_t *capacity, int32_t *arena_id);

/* Give an acquired arena back without submitting it (error unwinding in a packer: a file vanished, a damaged
 * archive).  mksnap_begin() also reclaims every arena that was acquired and never submitted. */
int mksnap_arena_release(mksnap_t *h, int32_t arena_id);

/* Capacities of this handle, so that a packer can flush an arena BEFORE a table limit is hit (a context of 500k tiny
 * files fills max_extents long before it fills a 1 GiB arena; the reference handles any file count,
 * add_copy_step.go:153-169). */
typedef struct {
    uint64_t max_extents;        /* extents, and ranges, per submit */
    uint64_t max_streams;        /* serial-stream slots per session */
    uint64_t max_chunks;         /* chunk-table rows per session */
    uint64_t host_arena_bytes;
    uint64_t device_arena_bytes;
    uint32_t n_host_arenas;
    uint32_t n_device_slots;
    uint64_t carry_bytes;        /* earliest arena offset of a MKSNAP_X_CONT extent (max chunk size, 512-aligned) */
} mksnap_limits;
int mksnap_get_limits(const mksnap_t *h, mksnap_limits *out);

/* Device memory for the stream log of MKSNAP_R_DEFER pieces: allocate it, resize it to `bytes` (rounded up to 64), or
 * free it (bytes == 0).  Refused with MKSNAP_E_STATE while deferred pieces wait in the log (a session between its
 * first deferred piece and finish); callable outside a session and right after begin.  Each deferred piece takes its
 * length rounded up to 16 bytes of the log.  The log stays allocated until resized, freed or the handle is destroyed. */
int mksnap_reserve_stream_log(mksnap_t *h, uint64_t bytes);

/* Async: copy arena[0,used) host->device, then run CRC over MKSNAP_X_CRC
 * extents, CDC + per-chunk SHA-256 over MKSNAP_X_CDC extents and one serial
 * SHA-256 per range.  Returns once everything is enqueued; the arena becomes
 * acquirable again when its copy has completed.  Replaces the io.Copy(checksum, fh)
 * loop of add_copy_step.go:230-237 and the tario.WriteEntry -> ConcurrentMultiWriter
 * fan-out of lib/tario/write.go:28-52 / lib/stream/multi_writer.go:35-66. */
int mksnap_arena_submit(mksnap_t *h, int32_t arena_id, uint64_t used,
                        const mksnap_extent *extents, uint64_t n_extents,
                        const mksnap_range *ranges, uint64_t n_ranges);

/* Device-resident variant: the bytes are already in device slot `slot`
 * (written by mksnap_synth_fill, a previous upload, or a GPUDirect producer). */
int mksnap_device_arena(mksnap_t *h, uint32_t slot, void **device_ptr, uint64_t *capacity);
int mksnap_device_upload(mksnap_t *h, uint32_t slot, uint64_t dst_off, const void *src, uint64_t n);
int mksnap_device_submit(mksnap_t *h, uint32_t slot, uint64_t used,
                         const mksnap_extent *extents, uint64_t n_extents,
                         const mksnap_range *ranges, uint64_t n_ranges);

/* Finish the session: sort + unique the chunk digests, Merkle root, wait for
 * the device, fill *out.  On a handle that is one rank of SEVERAL (mksnap_comm_init with n_ranks > 1) out->root is
 * left zeroed: the content address is the root of the global table, which mksnap_exchange_tables /
 * mksnap_allgather_tables return. */
int mksnap_finish(mksnap_t *h, mksnap_result *out);

/* cacheID arithmetic: the value checksum.Sum32() returns at
 * add_copy_step.go:119 for a context stream of stream_len bytes whose pure
 * accumulator is res->crc_pure. */
uint32_t mksnap_ctx_crc32(const mksnap_result *res);

/* ---- incremental cacheID: CRC-32 is linear, so a file's contribution can be reused without its bytes ----
 * With pure(M) = M(x) * x^32 mod P (what the engine accumulates), the context stream's value is the XOR over its
 * segments of pure(segment) * x^(8 * bytes after the segment).  mksnap_get_extent_crcs returns pure(extent) for every
 * MKSNAP_X_CRC extent of the finished session, in submission order; a caller that remembers pure(file content) per
 * file (keyed like MemFS keys a file: size + mtime, lib/tario/compare.go:104-120) folds an UNCHANGED file into a later
 * session with mksnap_crc_add -- no read, no H2D copy, no kernel -- and only changed files travel.  The cacheID is
 * bit-identical to the full computation (add_copy_step.go:102-122) as long as the remembered values are current.
 * mksnap_crc_concat joins the values of two adjacent pieces: pure(A||B) from pure(A), pure(B), len(B). */
int mksnap_crc_add(mksnap_t *h, uint32_t pure, uint64_t len, uint64_t crc_suffix); /* between begin and finish */
uint32_t mksnap_crc_concat(uint32_t pure_a, uint32_t pure_b, uint64_t len_b);
int mksnap_get_extent_crcs(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out);

/* ---- plan-level cacheIDs: many CRC streams from one session's extent values ----
 * Every COPY/ADD step of a build plan hashes its own stream (add_copy_step.go:102-122), and the steps share segments:
 * `COPY requirements.txt .` then `COPY . .`.  Each unique segment travels once as a MKSNAP_X_CRC extent; then
 * mksnap_crc_fold XORs, per use, value * x^(8 * suffix) into stream slot `stream` of this session on the device
 * (k_crc_fold), where suffix = bytes of that stream after the use.  The value is pure(extent) of the CRC extent `src`
 * (mksnap_get_extent_crcs numbering; it must already be submitted) or, with MKSNAP_U_VALUE, the low 32 bits of src (a
 * value the caller remembered).  Stream slots are [0, max_streams) and start at zero in every session.  Call between
 * begin and finish, at most max_extents uses per call; `uses` may be reused when the call returns.  A session whose CRC
 * extents outran the engine's per-extent table fails the fold (MKSNAP_E_CAPACITY) rather than fold a value it did not
 * keep.  The prefix seed + directive + args is not part of a stream: mksnap_crc_prepend adds it on the host. */
#define MKSNAP_U_VALUE 1u
typedef struct {
    uint64_t suffix;
    uint64_t src;
    uint32_t stream;
    uint32_t flags;
} mksnap_crc_use;
int mksnap_crc_fold(mksnap_t *h, const mksnap_crc_use *uses, uint64_t n);
/* after finish: pure value of the streams [0, *n_out), n_out = highest stream slot folded + 1 */
int mksnap_get_crc_streams(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out);
/* host arithmetic, no device: checksum.Sum32() of prefix || rest, given pure(rest) and len(rest) */
uint32_t mksnap_crc_prepend(const void *prefix, uint64_t n, uint32_t pure_rest, uint64_t len_rest);

/* ---- incremental layer commit: chunk digests remembered from an earlier session ----
 * Chunks never span files (DESIGN.md section 3), so a file's chunk digests depend on its own bytes only, and the table
 * is the sorted-unique multiset of all of them.  A caller that remembers a file's digests (keyed by file identity, under
 * the CDC parameters mksnap_get_cdc reports) appends them for an UNCHANGED file with mksnap_chunks_add instead of
 * submitting the file as a MKSNAP_X_CDC extent; finish sorts, uniques and roots the union, so root, n_chunks and
 * n_unique equal those of the full pass.  Appended rows join the table in call order behind the chunks of the submits
 * enqueued before the call (k_chunks_append, stream-ordered); mksnap_get_chunks returns them with end == UINT64_MAX.  At
 * most MKSNAP_CHUNKS_ADD_MAX rows (32 bytes each) per call: they travel through one pinned staging buffer of that size in
 * one copy; `digests` may be reused when the call returns.  Rows past max_chunks fail finish with MKSNAP_E_CAPACITY,
 * like computed chunks.  Call between begin and finish. */
#define MKSNAP_CHUNKS_ADD_MAX 65536u
int mksnap_chunks_add(mksnap_t *h, const uint8_t *digests, uint64_t n);
/* mksnap_arena_submit that copies only the listed spans of arena[0, used) host->device: the bytes the device reads
 * (MKSNAP_X_CDC / MKSNAP_X_CRC extents, ranges).  A file whose digests are appended and whose bytes are in the arena only
 * for the host (the layer tar to a file descriptor) then does not cross PCIe.  Spans are ascending, non-overlapping, off
 * and len multiples of 16, inside [0, used); every extent and range must lie inside one span (MKSNAP_E_INVAL
 * otherwise).  Device bytes of [0, used) outside the spans are zeroed on the copy stream, so the scan, which still reads
 * the whole arena, never sees bytes of an earlier submit.  stats.h2d_bytes counts the spans.  mksnap_arena_submit is
 * the single span [0, used). */
typedef struct {
    uint64_t off;
    uint64_t len;
} mksnap_span;
int mksnap_arena_submit_spans(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_span *spans, uint64_t n_spans,
                              const mksnap_extent *extents, uint64_t n_extents, const mksnap_range *ranges,
                              uint64_t n_ranges);
/* the handle's effective CDC parameters (defaults filled in): remembered chunk digests are valid only under these */
int mksnap_get_cdc(const mksnap_t *h, mksnap_cdc_params *out);

/* ---- gunzip: decompress a gzip blob on the device (replaces tario.NewGzipReader in FromStep.Execute,
 * lib/builder/step/from_step.go:118-134, and buildNode.applyLayer, lib/builder/build_node.go:131-148) ----
 * mksnap_gunzip_open copies the whole blob to the device, finds every candidate segment start (the byte after each
 * `00 00 FF FF`, the empty stored block of a sync / full flush, and each member body start), decodes from all of them
 * in parallel without output, links the true chain of segments member by member (trailers, next header) and fills
 * *info.  mksnap_gunzip_read then hands out the decompressed stream in order: `got` < `cap` only at the end (0 once
 * everything was read).  The output is produced one window of whole segments at a time: decode to 16-bit symbols,
 * resolve back-references across segments, CRC-32 each member piece with the K0 kernel, copy to `dst`.
 * Independent of begin / finish: a gunzip may be open while an ingest session on the same handle is, so the host can
 * feed the decompressed stream into arenas; calls are serialised by the caller as everywhere else.  One gunzip per
 * handle at a time (open on an open one: MKSNAP_E_STATE).
 * Every member body start is a scanned candidate, found on the device at each `1f 8b 08` whose header parses, so the
 * members of a bgzip / BGZF, eStargz or concatenated blob decode in parallel like the blocks of a pgzip blob.
 * Device memory is allocated at open and freed at close / destroy: the blob and its candidate tables (at most
 * gz_len / 4 + gz_len / 3 + 1 candidates at 40 bytes each, <= 25 * gz_len with the blob; a gz_len / 8 bitmap during
 * the scan only), plus one output window of max(256 MiB, largest segment) at 3 bytes per output byte, and a pinned host
 * copy of the window (reads are host copies; one D2H per window).  A single member without flush points is one
 * segment, so there the window is as large as the member, and it decodes on one GPU thread.  Blobs of 16 GiB or more,
 * and blobs whose candidates do not fit the 32-bit candidate scan, are refused (MKSNAP_E_CAPACITY); candidate tables
 * that do not fit in device memory fail with MKSNAP_E_NOMEM.  The gunzip runs on a stream of its own, so window
 * decodes do not wait behind the work of an open session.
 * Acceptance is that of Go's compress/gzip in multistream mode: zlib's inflate for the DEFLATE data; FNAME / FCOMMENT
 * at most 511 bytes; FHCRC checked; whatever follows a member must be another member header (trailing garbage and zero
 * padding are errors).  Malformed headers or DEFLATE data fail open with MKSNAP_E_DATA; a distance before the start of
 * its member, or a CRC-32 / ISIZE mismatch, fails the read that reaches the end of that member (bytes before it are
 * delivered).  After any error the handle stays usable: close, then open again. */
typedef struct {
    uint64_t gz_bytes, out_bytes;   /* blob length, decompressed length over all members */
    uint64_t n_members, n_segments; /* gzip members; independently decoded pieces (>= n_members) */
} mksnap_gunzip_info;
int mksnap_gunzip_open(mksnap_t *h, const void *gz, uint64_t gz_len, mksnap_gunzip_info *info);
int mksnap_gunzip_read(mksnap_t *h, void *dst, uint64_t cap, uint64_t *got); /* next bytes of the decompressed stream; 0 at the end */
int mksnap_gunzip_close(mksnap_t *h);
/* device time of the open gunzip so far (CUDA events on the compute stream): candidate scan, count decodes (including
 * the re-decodes of starts on the chain, counted in extra_decodes), write decodes, resolve + narrow, member CRC-32 */
typedef struct {
    float ms_scan, ms_count, ms_write, ms_resolve, ms_crc;
    uint32_t extra_decodes;
} mksnap_gunzip_times;
int mksnap_gunzip_get_times(mksnap_t *h, mksnap_gunzip_times *out);

/* ---- result tables (valid after mksnap_finish, until the next begin) ---- */
/* chunk END offsets (exclusive; position in the concatenation of all submitted
 * arenas) and digests, in (submit, extent, position) order; rows of mksnap_chunks_add
 * in their place in that order, with end = UINT64_MAX. */
int mksnap_get_chunks(mksnap_t *h, uint64_t *ends, uint8_t *digests, uint64_t capacity);
/* sorted-unique 32-byte digest table */
int mksnap_get_table(mksnap_t *h, uint8_t *table, uint64_t capacity_rows);
/* rows the handle's table currently holds: result.n_unique after finish / allgather, this rank's range after exchange */
uint64_t mksnap_table_rows(mksnap_t *h);
/* stream digests, row = stream slot: the TarDigest bytes of
 * lib/builder/step/common.go:86 (hex-encode and prefix "sha256:" on the host).  Rows [0, result.n_streams); the row of
 * a slot on which no stream finished in the session is unspecified (it may hold an earlier session's digest).  Inside a
 * session the call waits for the submits enqueued so far; the row of a stream that finished inline (not MKSNAP_R_DEFER)
 * in one of them is then final, and the slot may carry a new stream afterwards. */
int mksnap_get_stream_digests(mksnap_t *h, uint8_t *digests, uint64_t capacity);

/* ---- multi-GPU: one process per GPU, files sharded, one exchange step ---- */
/* NCCL is dlopen()ed (libnccl.so.2); rank 0 creates the id, the host side
 * distributes it (any out-of-band channel), every rank calls comm_init. */
int mksnap_comm_unique_id(uint8_t id[128]);
int mksnap_comm_init(mksnap_t *h, const uint8_t id[128], int32_t n_ranks, int32_t rank);
/* After mksnap_finish on every rank: all-gather the per-rank sorted-unique
 * tables (ncclAllGather of counts, then of padded rows), merge + unique on the
 * device, XOR-combine the CRC partials.  *out is identical on every rank and
 * equal to what a single GPU would produce for the whole context. */
int mksnap_allgather_tables(mksnap_t *h, mksnap_result *out);
/* The scalable form of the same step: the global table stays RANGE-PARTITIONED.  Rank r ends up owning the digests
 * whose big-endian 64-bit prefix p has floor(p * n_ranks / 2^64) == r: slices of the per-rank tables travel once
 * (ncclSend/ncclRecv all-to-all over NVLink), every rank sorts only its range, Merkle level 0 is computed where the
 * rows are (a group of 256 consecutive global rows by the rank owning its first row, the missing rows of a group
 * that straddles a range end come from an all-gather of every rank's first 255 rows), level-1 digests are
 * all-gathered and the upper levels run everywhere.  *out (root, CRC, counters, n_unique = GLOBAL unique rows) is
 * identical on every rank and equal to the single-GPU result; afterwards mksnap_get_table returns THIS rank's range
 * (ascending; the ranges of ranks 0..n-1 concatenated are the global table).  Work per rank stays ~constant as
 * n_ranks grows, where mksnap_allgather_tables sorts n_ranks times more rows on every rank. */
int mksnap_exchange_tables(mksnap_t *h, mksnap_result *out);
/* The same exchange between n handles of ONE process on ONE device (device copies instead of NCCL; no comm_init):
 * handle i plays rank i, outs[i] receives its result.  Used to run the exchange logic for any n on a single GPU. */
int mksnap_exchange_tables_local(mksnap_t **handles, int32_t n, mksnap_result *outs);
/* Host arithmetic of the exchange, no device needed: given the rows every rank holds after the all-to-all, which
 * groups of 256 global rows does `rank` hash?  out = {U total rows, g0 first global row of the rank, lead rows that
 * belong to a predecessor's group, full groups, own rows in the tail group, rows borrowed from successors, groups}. */
int mksnap_exchange_plan(const uint64_t *rows_per_rank, int32_t n_ranks, int32_t rank, uint64_t out[7]);

/* ---- utilities --------------------------------------------------------- */
/* Deterministic synthetic content, generated on the device into slot bytes
 * [byte_off, byte_off+n) (multiples of 16): little-endian u64 word i (absolute
 * word index in the slot) = mix64(seed + (i+1)*0x9E3779B97F4A7C15). */
int mksnap_synth_fill(mksnap_t *h, uint32_t slot, uint64_t byte_off, uint64_t n, uint64_t seed);
int mksnap_memset(mksnap_t *h, uint32_t slot, uint64_t byte_off, uint64_t n, int value);
int mksnap_device_download(mksnap_t *h, uint32_t slot, uint64_t src_off, void *dst, uint64_t n);
int mksnap_sync(mksnap_t *h);
int mksnap_stats(mksnap_t *h, mksnap_stats_t *out);
void mksnap_default_cdc(mksnap_cdc_params *p);
/* the multiplier M of the frozen rolling hash h_i = h_{i-1}*M + (LE word ending at byte i) (for cross-checking against
 * the oracle) */
uint32_t mksnap_roll_multiplier(void);

#ifdef __cplusplus
}
#endif
#endif
