// mksnap.cu — C-ABI implementation of include/mksnap.h (libmksnap.so).
//
// Host-side orchestration only: arena ring, extent tables, stream/event
// plumbing, result tables.  All arithmetic happens in the kernels of
// mksnap_kernels.cuh; there is deliberately no CPU fallback.
#include "../../include/mksnap.h"
#include "mksnap_kernels.cuh"

#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

using namespace mk;

struct Id128 {
    char b[128];
};

namespace {

// Owner of n elements of T, in device memory (cudaMalloc) or pinned host memory (cudaHostAlloc).  alloc() frees the
// old block before it allocates, so a growth never holds both, and records n only when the allocation succeeds: after
// a failed growth size() is 0, and a capacity check against it grows again or refuses rather than use a null pointer.
template <typename T, bool Pinned> class Buf {
public:
    Buf() = default;
    Buf(Buf &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    Buf &operator=(Buf &&o) noexcept
    {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        return *this;
    }
    ~Buf() { reset(); }

    cudaError_t alloc(uint64_t n)
    {
        reset();
        void *q = nullptr;
        cudaError_t e;
        if constexpr (Pinned)
            e = cudaHostAlloc(&q, n * sizeof(T), cudaHostAllocDefault);
        else
            e = cudaMalloc(&q, n * sizeof(T));
        if (e == cudaSuccess) {
            p_ = static_cast<T *>(q);
            n_ = n;
        }
        return e;
    }
    void reset()
    {
        if (!p_)
            return;
        if constexpr (Pinned)
            cudaFreeHost(p_);
        else
            cudaFree(p_);
        p_ = nullptr;
        n_ = 0;
    }
    uint64_t size() const { return n_; }
    T *get() const { return p_; }
    operator T *() const { return p_; }
    T *operator->() const { return p_; }

private:
    T *p_ = nullptr;
    uint64_t n_ = 0;
};
template <typename T> using DevBuf = Buf<T, false>;
template <typename T> using PinnedBuf = Buf<T, true>;

// Owner of one CUDA event or stream.  put() destroys what it holds and returns the slot a create call writes.
template <typename H, cudaError_t (*Destroy)(H)> class Handle {
public:
    Handle() = default;
    Handle(Handle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Handle &operator=(Handle &&o) noexcept
    {
        std::swap(h_, o.h_);
        return *this;
    }
    ~Handle()
    {
        if (h_)
            Destroy(h_);
    }

    H *put()
    {
        if (h_)
            Destroy(h_);
        h_ = nullptr;
        return &h_;
    }
    operator H() const { return h_; }

private:
    H h_ = nullptr;
};
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;

thread_local std::string g_create_error;

constexpr uint64_t SLOT_SLACK = 8192;
constexpr int N_EV = 8; // timing marks per submit
constexpr uint32_t MAX_SLOTS = 4;
constexpr int GH_WORDS = 8; // u64 words per rank in the all-gather header

struct MetaSet {
    // pinned host staging
    PinnedBuf<CrcExtent> h_crc;
    PinnedBuf<uint32_t> h_piece_base;
    PinnedBuf<CdcFile> h_files;
    PinnedBuf<uint64_t> h_rstart, h_rlen;
    PinnedBuf<uint32_t> h_rstream, h_rflags;
    // device mirrors
    DevBuf<CrcExtent> d_crc;
    DevBuf<uint32_t> d_piece_base;
    DevBuf<uint32_t> d_ext_pure; // pure(extent) of this submit's CRC extents
    DevBuf<CdcFile> d_files;
    DevBuf<uint64_t> d_rstart, d_rlen;
    DevBuf<uint32_t> d_rstream, d_rflags;
    Event ev_done; // kernels that read this set have finished
    bool in_flight = false;
};

struct HostArena {
    PinnedBuf<uint8_t> ptr;
    Event ev_h2d;
    bool in_flight = false;
    bool acquired = false;
};

// NCCL via dlopen: only the handful of entry points we need
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(void *) = nullptr;
    int (*CommInitRank)(void **, int, /* ncclUniqueId by value */ Id128, int) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    int (*Send)(const void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*Recv)(void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
};

} // namespace

struct mksnap_gunzip_state; // mksnap_inflate.cuh

struct mksnap {
    mksnap_config cfg;
    CdcParamsDev prm;
    std::string err;
    int sm_count = 132;
    Stream s_comp, s_copy; // declared first, so destroyed after the buffers and events used on them

    uint32_t n_slots = 0;
    DevBuf<uint8_t> d_slot[MAX_SLOTS];
    Event ev_slot_free[MAX_SLOTS];
    bool slot_used[MAX_SLOTS] = {false, false, false, false};

    std::vector<HostArena> arenas;
    uint32_t next_arena = 0;

    std::vector<MetaSet> meta;
    uint64_t submit_idx = 0;

    DevBuf<CrcConsts> d_consts;
    DevBuf<SessionCounters> d_sc;
    PinnedBuf<SessionCounters> h_sc;

    DevBuf<TileRec> d_tiles;
    CUtensorMap tm_main[MAX_SLOTS]; // per slot: arena viewed as [rows][128 B]
    CUtensorMap tm_crc[MAX_SLOTS];  // the same with the box of the CRC variant's tiles
    DevBuf<uint32_t> d_part;        // CRC of every 128-byte arena row, written by the CRC variant of the scan
    int scan_cfg = 0; // index into SCAN_SHAPES
    bool sha_fma = true; // chunk SHA-256: additions on the FMA pipe
    DevBuf<uint32_t> d_pool;
    uint32_t pool_cap = 0;
    DevBuf<uint32_t> d_pool_count;
    DevBuf<uint32_t> d_counts, d_bases;
    DevBuf<uint32_t> d_scan_tmp; // block sums for the generic scan (several levels)

    // session tables
    uint64_t max_chunks = 0;
    DevBuf<uint64_t> d_chunk_start, d_chunk_len, d_chunk_end;
    DevBuf<uint32_t> d_order; // K2 work order of the current batch (batch-relative chunk indices)
    bool sha_order = true;
    DevBuf<uint8_t> d_digests;
    uint64_t max_streams = 0;
    DevBuf<uint8_t> d_stream_digests;
    DevBuf<StreamState> d_stream_state;
    std::vector<uint32_t> stream_stamp; // submit epoch that last used the stream slot (one piece per stream per submit)
    uint32_t stamp_epoch = 0;
    std::vector<uint8_t> stream_open; // per slot: the last piece carried MKSNAP_R_MORE (finish refuses the session)
    uint64_t n_open = 0;              // slots with stream_open set
    uint64_t n_streams = 0;
    uint64_t stream_base = 0; // bytes of arenas submitted before the current one
    // MKSNAP_R_DEFER: the stream log and the pieces waiting in it (log order)
    std::vector<uint8_t> stream_defer; // per slot: the open stream is a deferred one
    std::vector<uint32_t> log_count;   // per slot: pieces waiting in the log
    struct LogPiece {
        uint64_t off, len;
        uint32_t stream, more;
    };
    std::vector<LogPiece> log_pending;
    DevBuf<uint8_t> d_log;
    uint64_t log_used = 0;
    PinnedBuf<uint64_t> h_flush; // K4 tables of a flush, 3 words per row: start, len (u64), stream, flags (u32)
    DevBuf<uint64_t> d_flush;
    Event ev_flush;              // the last flush's table copy has left h_flush
    bool have_flush_time = false;
    uint64_t crc_bytes = 0;
    DevBuf<uint32_t> d_crc_session; // pure(extent) of every CRC extent of the session, submission order
    uint64_t crc_session_n = 0;
    uint32_t crc_host_acc = 0;         // contributions folded on the host (mksnap_crc_add)
    uint64_t crc_host_bytes = 0;
    DevBuf<CrcUse> d_uses;             // mksnap_crc_fold: use table (max_extents rows) and stream values (max_streams),
    DevBuf<uint32_t> d_stream_pure;    //   allocated by the first fold
    uint64_t fold_streams = 0;         // highest stream slot folded in this session + 1
    PinnedBuf<uint8_t> h_add;          // mksnap_chunks_add: pinned staging of MKSNAP_CHUNKS_ADD_MAX rows, its device
    DevBuf<uint8_t> d_add;             //   twin and the end of the last copy out of it; allocated by the first call
    Event ev_add;
    bool open_file = false;      // the last submit ended with a MKSNAP_X_MORE extent: the next must start with its continuation
    DevBuf<uint8_t> d_carry;     // open chunk of that file (k_carry_out -> k_carry_in)

    // sort / table
    DevBuf<uint64_t> d_keys[2];
    DevBuf<uint32_t> d_idx[2];
    DevBuf<uint8_t> d_sorted, d_table;
    DevBuf<uint32_t> d_flags, d_pos, d_hist;
    DevBuf<uint8_t> d_merkle[2];
    uint64_t table_cap = 0; // rows the sort buffers can hold
    uint64_t n_unique = 0;
    uint8_t root[32];
    bool finished = false;
    bool in_session = false;
    mksnap_result last_result;

    // multi-GPU
    NcclApi nccl;
    void *comm = nullptr;
    int n_ranks = 1, rank = 0;
    DevBuf<uint8_t> d_gather;                // n_ranks * pad_rows * 32
    DevBuf<unsigned long long> d_gcount;     // n_ranks * GH_WORDS header words
    DevBuf<uint8_t> d_concat;                // dense concatenation of all ranks' tables
    // range-partitioned exchange (mksnap_exchange_tables): small fixed-size scratch
    DevBuf<unsigned long long> d_xbounds;    // R+1 slice boundaries of my table
    DevBuf<unsigned long long> d_xhdr;       // R * (GH_WORDS + R) header words
    DevBuf<uint8_t> d_xrec;                  // R records of XREC_BYTES: u64 rows-in-range, then the first 255 rows
    DevBuf<uint8_t> d_xtail;                 // 256 rows: the Merkle group that straddles the end of my range
    int x_ranks = 0;                         // ranks the four buffers above hold

    // timing
    Event ev[N_EV];
    Event ev_copy0, ev_copy1, ev_copy_done;
    Event ev_fin[4];
    bool have_submit_times = false, have_h2d_time = false, have_fin_times = false, have_gather_time = false;
    mksnap_stats_t stats;

    mksnap_gunzip_state *gz = nullptr; // open gunzip (mksnap_gunzip_open .. close), independent of the session
};

namespace {

void gz_free(mksnap *h); // mksnap_inflate.cuh

int fail(mksnap *h, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h)
        h->err = buf;
    else
        g_create_error = buf;
    return code;
}

#define CK(h, call)                                                                                   \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess)                                                                       \
            return fail((h), e__ == cudaErrorMemoryAllocation ? MKSNAP_E_NOMEM : MKSNAP_E_CUDA,       \
                        "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));          \
    } while (0)

#define LAUNCH_OK(h)                                                                                  \
    do {                                                                                              \
        cudaError_t e__ = cudaGetLastError();                                                         \
        if (e__ != cudaSuccess)                                                                       \
            return fail((h), MKSNAP_E_CUDA, "%s:%d kernel launch: %s", __FILE__, __LINE__,            \
                        cudaGetErrorString(e__));                                                     \
        (h)->stats.kernel_launches++;                                                                 \
    } while (0)

uint32_t xpow_bits(uint64_t bits) // x^bits mod P, reflected
{
    uint32_t result = 0x80000000u, sq = 0x40000000u; // x^0, x^1
    while (bits) {
        if (bits & 1)
            result = crc_mulmod(result, sq);
        sq = crc_mulmod(sq, sq);
        bits >>= 1;
    }
    return result;
}

void build_crc_consts(CrcConsts *c)
{
    const uint32_t x4096 = xpow_bits(4096);
    for (int t = 0; t < 4; t++)
        for (uint32_t v = 0; v < 256; v++)
            c->mulk[t][v] = crc_mulmod(v << (8 * t), x4096);
    for (int l = 0; l < 32; l++)
        for (int k = 0; k < 4; k++)
            c->lane_c[l * 4 + k] = xpow_bits(32 + 8 * (508 - 16 * l - 4 * k));
    for (int t = 0; t < 4; t++)
        for (uint32_t v = 0; v < 256; v++)
            c->xe[t][v] = xpow_bits((uint64_t)v << (8 * t));
    const uint32_t xg = xpow_bits(8ull * CRC_GRANULE * 128), x32 = xpow_bits(32);
    for (int t = 0; t < 4; t++)
        for (uint32_t v = 0; v < 256; v++) {
            c->mulk_g[t][v] = crc_mulmod(v << (8 * t), xg);
            c->mulk_w[t][v] = crc_mulmod(v << (8 * t), x32);
        }
    for (int l = 0; l < 32; l++)
        for (int k = 0; k < 4; k++)
            c->lane_g[l * 4 + k] = xpow_bits(32 + 8ull * CRC_GRANULE * (127 - 4 * l - k));
    for (int j = 0; j < 32; j++)
        c->word_g[j] = xpow_bits(32ull * (31 - j));
}

// generic device exclusive scan (u32), in -> out (may alias), n elements
int scan_u32(mksnap *h, const uint32_t *in, uint32_t *out, uint64_t n, cudaStream_t s)
{
    if (n == 0)
        return 0;
    // level sizes
    std::vector<uint64_t> sizes;
    sizes.push_back(n);
    while (sizes.back() > SCAN_ITEMS)
        sizes.push_back((sizes.back() + SCAN_ITEMS - 1) / SCAN_ITEMS);
    // temp layout: level l (l>=1) sums at offset
    std::vector<uint64_t> off(sizes.size(), 0);
    uint64_t total = 0;
    for (size_t l = 1; l < sizes.size(); l++) {
        off[l] = total;
        total += sizes[l];
    }
    if (total > h->d_scan_tmp.size())
        return fail(h, MKSNAP_E_CAPACITY, "scan temp too small (%llu > %llu)", (unsigned long long)total,
                    (unsigned long long)h->d_scan_tmp.size());
    // up-sweep: reduce each level into the next
    for (size_t l = 0; l + 1 < sizes.size(); l++) {
        const uint32_t *src = l == 0 ? in : h->d_scan_tmp + off[l];
        uint32_t nb = (uint32_t)sizes[l + 1];
        k_scan_reduce<<<nb, 256, 0, s>>>(src, sizes[l], h->d_scan_tmp + off[l + 1]);
        LAUNCH_OK(h);
    }
    // top level fits one block: scan in place
    for (size_t l = sizes.size(); l-- > 0;) {
        const uint32_t *src = l == 0 ? in : h->d_scan_tmp + off[l];
        uint32_t *dst = l == 0 ? out : h->d_scan_tmp + off[l];
        const uint32_t *boff = (l + 1 < sizes.size()) ? h->d_scan_tmp + off[l + 1] : nullptr;
        uint32_t nb = (uint32_t)((sizes[l] + SCAN_ITEMS - 1) / SCAN_ITEMS);
        k_scan_apply<<<nb, 256, 0, s>>>(src, sizes[l], boff, dst);
        LAUNCH_OK(h);
    }
    return 0;
}

int sha_grid(const mksnap *h) { return h->sm_count * 8; }

// sort n digests at `src` -> sorted unique table at h->d_table; sets h->n_unique, root
int sort_unique_root(mksnap *h, const uint8_t *src, uint64_t n, cudaStream_t s)
{
    if (n > h->table_cap)
        return fail(h, MKSNAP_E_CAPACITY, "table of %llu rows exceeds capacity %llu", (unsigned long long)n,
                    (unsigned long long)h->table_cap);
    h->n_unique = 0;
    if (n) {
        const uint32_t tb = 256;
        k_make_keys<<<(uint32_t)((n + tb - 1) / tb), tb, 0, s>>>(src, n, h->d_keys[0], h->d_idx[0]);
        LAUNCH_OK(h);
        const uint32_t nblocks = (uint32_t)((n + SORT_TILE - 1) / SORT_TILE);
        int cur = 0;
        for (int pass = 0; pass < SORT_KEY_BITS / 8; pass++) {
            const int shift = 64 - SORT_KEY_BITS + pass * 8;
            k_radix_hist<<<nblocks, SORT_THREADS, 0, s>>>(h->d_keys[cur], n, shift, h->d_hist, nblocks);
            LAUNCH_OK(h);
            int rc = scan_u32(h, h->d_hist, h->d_hist, (uint64_t)256 * nblocks, s);
            if (rc)
                return rc;
            k_radix_scatter<<<nblocks, SORT_THREADS, 0, s>>>(h->d_keys[cur], h->d_idx[cur], n, shift, h->d_hist,
                                                             nblocks, h->d_keys[cur ^ 1], h->d_idx[cur ^ 1]);
            LAUNCH_OK(h);
            cur ^= 1;
        }
        k_gather_digests<<<(uint32_t)((2 * n + tb - 1) / tb), tb, 0, s>>>(src, h->d_idx[cur], n, h->d_sorted);
        LAUNCH_OK(h);
        // long runs (duplicates) are listed in the idle flag buffer and handled by whole CTAs
        uint2 *long_runs = reinterpret_cast<uint2 *>(h->d_hist.get()); // sized for FIX_LONG_CAP entries in alloc_table_buffers
        uint32_t *n_long = h->d_pos;
        CK(h, cudaMemsetAsync(n_long, 0, 4, s));
        k_fix_ties<<<(uint32_t)((n + tb - 1) / tb), tb, 0, s>>>(h->d_keys[cur], n, h->d_sorted, 64 - SORT_KEY_BITS, long_runs, n_long);
        LAUNCH_OK(h);
        k_fix_long_runs<<<h->sm_count, 256, 0, s>>>(h->d_sorted, long_runs, n_long);
        LAUNCH_OK(h);
        k_unique_flags<<<(uint32_t)((n + tb - 1) / tb), tb, 0, s>>>(h->d_sorted, n, h->d_flags);
        LAUNCH_OK(h);
        int rc = scan_u32(h, h->d_flags, h->d_pos, n, s);
        if (rc)
            return rc;
        k_compact_digests<<<(uint32_t)((2 * n + tb - 1) / tb), tb, 0, s>>>(h->d_sorted, h->d_flags, h->d_pos, n,
                                                                            h->d_table);
        LAUNCH_OK(h);
        uint32_t last_pos = 0, last_flag = 0;
        CK(h, cudaMemcpyAsync(&last_pos, h->d_pos + (n - 1), 4, cudaMemcpyDeviceToHost, s));
        CK(h, cudaMemcpyAsync(&last_flag, h->d_flags + (n - 1), 4, cudaMemcpyDeviceToHost, s));
        CK(h, cudaStreamSynchronize(s));
        h->n_unique = (uint64_t)last_pos + last_flag;
    }
    return 0;
}

// hash level after level (groups of 256 digests = 8 KiB) starting from `cur_n` digests at `cur`; always at least once
int merkle_from(mksnap *h, const uint8_t *cur, uint64_t cur_n, cudaStream_t s)
{
    int which = 0;
    for (;;) {
        const uint64_t next_n = cur_n == 0 ? 1 : (cur_n + 255) / 256;
        // a Merkle group is one 8 KiB serial SHA-256: the warp-pair stream kernel (next block prefetched, rounds and
        // schedule on separate warps) suits a level better than one lane per group of the chunk kernel, which waits
        // for its un-prefetched loads with only a handful of warps per SM
        CK(h, cudaMemsetAsync(&h->d_sc->work, 0, 4, s));
        k_sha256_streams<<<(uint32_t)std::min<uint64_t>((next_n + 31) / 32, (uint64_t)h->sm_count * 4), SS_THREADS, 0, s>>>(
            cur, nullptr, nullptr, (uint32_t)next_n, nullptr, nullptr, nullptr, h->d_merkle[which], &h->d_sc->work, 32u, 1u, 8192,
            cur_n * 32);
        LAUNCH_OK(h);
        cur = h->d_merkle[which];
        cur_n = next_n;
        which ^= 1;
        if (cur_n == 1)
            break;
    }
    CK(h, cudaMemcpyAsync(h->root, cur, 32, cudaMemcpyDeviceToHost, s));
    h->stats.d2h_bytes += 32;
    return 0;
}
int merkle_root(mksnap *h, cudaStream_t s) { return merkle_from(h, h->d_table, h->n_unique, s); } // level 0 = table

} // namespace

// ---------------------------------------------------------------------------
extern "C" {

int mksnap_abi_version(void) { return MKSNAP_ABI_VERSION; }

void mksnap_default_cdc(mksnap_cdc_params *p)
{
    p->min_size = 4096;
    p->normal_size = 16384;
    p->max_size = 131072;
    p->strict_bits = 16;
    p->loose_bits = 12;
}

uint32_t mksnap_roll_multiplier(void) { return ROLL_MULT; }

const char *mksnap_last_error(const mksnap_t *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

} // extern "C" (helpers below are C++)

// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda link dependency)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int make_row_map(mksnap *h, EncodeTiledFn enc, CUtensorMap *out, void *base, uint64_t n_rows, uint32_t box_rows)
{
    const cuuint64_t dims[2] = {128, n_rows};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {128, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(h, MKSNAP_E_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%llu box=%u", (int)r,
                    (unsigned long long)n_rows, box_rows);
    return 0;
}

// (re)allocate everything whose size follows the number of table rows: radix keys/payload, sorted and unique
// tables, flags/positions, histograms, Merkle levels, scan temporaries.  Called at create (rows = max_chunks)
// and again by mksnap_comm_init (rows = max_chunks x ranks: every rank merges the union of all tables).
static int alloc_table_buffers(mksnap *h, uint64_t rows)
{
    h->table_cap = 0;
    for (int k = 0; k < 2; k++) {
        CK(h, h->d_keys[k].alloc(rows));
        CK(h, h->d_idx[k].alloc(rows));
    }
    CK(h, h->d_sorted.alloc(rows * 32));
    CK(h, h->d_table.alloc(rows * 32));
    CK(h, h->d_flags.alloc(rows));
    CK(h, h->d_pos.alloc(rows));
    const uint64_t hist_words = std::max<uint64_t>(256ull * ((rows + SORT_TILE - 1) / SORT_TILE + 1), 2ull * FIX_LONG_CAP + 64); // also holds k_fix_ties' long-run list
    CK(h, h->d_hist.alloc(hist_words));
    const uint64_t merkle_rows = rows / 256 + 2;
    CK(h, h->d_merkle[0].alloc(merkle_rows * 32));
    CK(h, h->d_merkle[1].alloc((merkle_rows / 256 + 2) * 32));
    CK(h, h->d_scan_tmp.alloc(std::max(rows, std::max<uint64_t>(hist_words, h->cfg.max_extents)) / SCAN_ITEMS * 2 + 4096));
    h->table_cap = rows;
    return 0;
}

template <int GROUPS, int TW, int ST, int REP = 0>
static int launch_scan(mksnap *h, uint32_t slot, uint32_t n_regions, cudaStream_t sk)
{
    using Cfg = ScanCfg<GROUPS, TW, ST, REP>;
    const uint32_t n_tiles = (n_regions + Cfg::TILE_WARPS - 1) / Cfg::TILE_WARPS;
    const uint32_t grid = std::min<uint32_t>(n_tiles, (uint32_t)h->sm_count);
    k_roll_scan<GROUPS, TW, ST, REP><<<grid, Cfg::THREADS, Cfg::SMEM, sk>>>(
        REP ? h->tm_crc[slot] : h->tm_main[slot], n_tiles, h->prm.strict_lim, h->prm.loose_lim, h->d_tiles, h->d_pool,
        h->pool_cap, h->d_pool_count, &h->d_sc->err, &h->d_consts->mulk_w[0][0], h->d_part);
    LAUNCH_OK(h);
    return 0;
}

// the k_roll_scan shapes that are compiled in: {groups, warps per tile, stages}; MKSNAP_SCAN_CFG picks one (0 = default)
struct ScanShape {
    int groups, tile_warps, stages;
};
#define MK_SCAN_SHAPES(X) X(0, 4, 6, 8) X(1, 2, 6, 8) X(2, 4, 4, 12) X(3, 3, 4, 12) X(4, 2, 4, 12) X(5, 4, 3, 16) X(6, 6, 4, 12)
#define MK_SHAPE_ROW(I, G, T, S) {G, T, S},
static const ScanShape SCAN_SHAPES[] = {MK_SCAN_SHAPES(MK_SHAPE_ROW)};
#undef MK_SHAPE_ROW
constexpr int N_SCAN_SHAPES = (int)(sizeof(SCAN_SHAPES) / sizeof(SCAN_SHAPES[0]));

static int launch_scan_cfg(mksnap *h, uint32_t slot, uint32_t n_regions, cudaStream_t sk)
{
    switch (h->scan_cfg) {
#define MK_SHAPE_CASE(I, G, T, S) \
    case I: return launch_scan<G, T, S>(h, slot, n_regions, sk);
        MK_SCAN_SHAPES(MK_SHAPE_CASE)
#undef MK_SHAPE_CASE
    default: return launch_scan<4, 6, 8>(h, slot, n_regions, sk);
    }
}

// The CRC variant of the scan (submits with CRC extents and CDC files): 3 groups x 6 warps per tile, 6 stages, tables in 16 copies
// (64 KiB: lanes l and l+16 share one, at most a 2-way conflict).  Fastest of the shapes measured on an H100 (DESIGN.md
// section 5); full replication (128 KiB) leaves too little room for stages.
#define MK_CRC_SCAN_SHAPE 3, 6, 6, 16

extern "C" {

static int create_impl(mksnap *h)
{
    const mksnap_config &c = h->cfg;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(h, MKSNAP_E_CUDA, "no CUDA device usable (%s); libmksnap has no CPU fallback",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (c.device < 0 || c.device >= ndev)
        return fail(h, MKSNAP_E_INVAL, "device %d out of range [0,%d)", c.device, ndev);
    CK(h, cudaSetDevice(c.device));
    cudaDeviceProp prop;
    CK(h, cudaGetDeviceProperties(&prop, c.device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(h, MKSNAP_E_CUDA, "device %d is sm_%d%d; libmksnap is built for sm_90a only", c.device,
                    prop.major, prop.minor);
    h->sm_count = prop.multiProcessorCount;
    CK(h, cudaStreamCreateWithFlags(h->s_comp.put(), cudaStreamNonBlocking));
    CK(h, cudaStreamCreateWithFlags(h->s_copy.put(), cudaStreamNonBlocking));

    h->n_slots = c.n_device_slots ? c.n_device_slots : (c.n_host_arenas ? 2u : 1u);
    if (h->n_slots > MAX_SLOTS)
        return fail(h, MKSNAP_E_INVAL, "n_device_slots > %u", MAX_SLOTS);
    for (uint32_t s = 0; s < h->n_slots; s++) {
        CK(h, h->d_slot[s].alloc(c.device_arena_bytes + SLOT_SLACK));
        CK(h, cudaMemsetAsync(h->d_slot[s] + c.device_arena_bytes, 0, SLOT_SLACK, h->s_comp));
        CK(h, cudaEventCreateWithFlags(h->ev_slot_free[s].put(), cudaEventDisableTiming));
    }
    h->arenas.resize(c.n_host_arenas);
    for (auto &a : h->arenas) {
        CK(h, a.ptr.alloc(c.host_arena_bytes));
        CK(h, cudaEventCreateWithFlags(a.ev_h2d.put(), cudaEventDisableTiming));
    }
    const uint64_t mx = c.max_extents;
    h->meta.resize(std::max<uint32_t>(2, h->n_slots));
    for (auto &m : h->meta) {
        CK(h, m.h_crc.alloc(mx));
        CK(h, m.h_piece_base.alloc(mx + 1));
        CK(h, m.h_files.alloc(mx));
        CK(h, m.h_rstart.alloc(mx));
        CK(h, m.h_rlen.alloc(mx));
        CK(h, m.h_rstream.alloc(mx));
        CK(h, m.h_rflags.alloc(mx));
        CK(h, m.d_crc.alloc(mx));
        CK(h, m.d_piece_base.alloc(mx + 1));
        CK(h, m.d_ext_pure.alloc(mx));
        CK(h, m.d_files.alloc(mx));
        CK(h, m.d_rstart.alloc(mx));
        CK(h, m.d_rlen.alloc(mx));
        CK(h, m.d_rstream.alloc(mx));
        CK(h, m.d_rflags.alloc(mx));
        CK(h, cudaEventCreateWithFlags(m.ev_done.put(), cudaEventDisableTiming));
    }

    CrcConsts *hc = new CrcConsts;
    build_crc_consts(hc);
    CK(h, h->d_consts.alloc(1));
    CK(h, cudaMemcpy(h->d_consts, hc, sizeof(CrcConsts), cudaMemcpyHostToDevice));
    delete hc;
    CK(h, h->d_sc.alloc(1));
    CK(h, cudaMemset(h->d_sc, 0, sizeof(SessionCounters)));
    CK(h, h->h_sc.alloc(1));

    const uint64_t n_tiles = c.device_arena_bytes / SCAN_TILE + 128; // one TileRec per 4 KiB region (+ tile round-up)
    CK(h, h->d_tiles.alloc(n_tiles));
    CK(h, h->d_part.alloc(n_tiles * (SCAN_TILE / CRC_GRANULE))); // one u32 per row of every scanned region
    {
        EncodeTiledFn enc = nullptr;
        cudaDriverEntryPointQueryResult qres;
        CK(h, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void **)&enc, cudaEnableDefault, &qres));
        if (!enc || qres != cudaDriverEntryPointSuccess)
            return fail(h, MKSNAP_E_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
        const char *e = getenv("MKSNAP_SCAN_CFG"); // tuning knob: index into SCAN_SHAPES (0 = default)
        if (e && e[0] >= '0' && e[0] <= '9' && atoi(e) < N_SCAN_SHAPES)
            h->scan_cfg = atoi(e);
        const uint64_t n_rows = (c.device_arena_bytes + SLOT_SLACK) / 128;
        const uint32_t box_rows = (uint32_t)SCAN_SHAPES[h->scan_cfg].tile_warps * 32u + 1u; // the row above the tile travels with it
        for (uint32_t s = 0; s < h->n_slots; s++) {
            int rc;
            if ((rc = make_row_map(h, enc, &h->tm_main[s], h->d_slot[s], n_rows, box_rows)))
                return rc;
            if ((rc = make_row_map(h, enc, &h->tm_crc[s], h->d_slot[s], n_rows, ScanCfg<MK_CRC_SCAN_SHAPE>::BOX_ROWS)))
                return rc;
        }
#define MK_SET_SMEM(I, G, T, S) \
    CK(h, cudaFuncSetAttribute(k_roll_scan<G, T, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ScanCfg<G, T, S>::SMEM));
        MK_SCAN_SHAPES(MK_SET_SMEM)
#undef MK_SET_SMEM
        CK(h, cudaFuncSetAttribute(k_roll_scan<MK_CRC_SCAN_SHAPE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)ScanCfg<MK_CRC_SCAN_SHAPE>::SMEM));
        const char *e2 = getenv("MKSNAP_SHA_FMA"); // tuning knob: 0 = plain adds in the chunk SHA-256 kernel
        if (e2 && e2[0] == '0')
            h->sha_fma = false;
        const char *e3 = getenv("MKSNAP_SHA_ORDER"); // tuning knob: 0 = hash chunks in file order instead of longest first
        if (e3 && e3[0] == '0')
            h->sha_order = false;
    }
    // expected candidates = bytes >> loose_bits; 8x headroom (32x at the default 12 bits would be wasteful for
    // dense parameter sets), plus one private block per resident scan warp (x2)
    uint64_t pc = std::max<uint64_t>(1u << 20, (c.device_arena_bytes >> h->cfg.cdc.loose_bits) * 8) +
                  2ull * h->sm_count * 32 * SCAN_POOL_BLOCK;
    if (pc > 0xFFFFFFF0ull)
        pc = 0xFFFFFFF0ull;
    h->pool_cap = (uint32_t)pc;
    CK(h, h->d_pool.alloc(h->pool_cap));
    CK(h, h->d_pool_count.alloc(1));
    CK(h, h->d_crc_session.alloc(std::max<uint64_t>(4 * mx, 1ull << 20)));
    CK(h, h->d_carry.alloc(((uint64_t)h->prm.max_size + 511) / 512 * 512));
    CK(h, h->d_counts.alloc(mx));
    CK(h, h->d_bases.alloc(mx));

    // default: every byte in min-size chunks, plus per file the end-of-file chunk and the two spare cut-list slots of the big-file path
    h->max_chunks = c.max_chunks ? c.max_chunks : c.device_arena_bytes / h->prm.min_size + 3 * mx + 64;
    const uint64_t mc = h->max_chunks;
    CK(h, h->d_chunk_start.alloc(mc));
    CK(h, h->d_chunk_len.alloc(mc));
    CK(h, h->d_order.alloc(mc));
    CK(h, h->d_chunk_end.alloc(mc));
    CK(h, h->d_digests.alloc(mc * 32));
    h->max_streams = mx;
    CK(h, h->d_stream_digests.alloc(h->max_streams * 32));
    CK(h, h->d_stream_state.alloc(h->max_streams));
    CK(h, cudaMemset(h->d_stream_state, 0, h->max_streams * sizeof(StreamState)));
    h->stream_stamp.assign(h->max_streams, 0);
    h->stream_open.assign(h->max_streams, 0);
    h->stream_defer.assign(h->max_streams, 0);
    h->log_count.assign(h->max_streams, 0);
    CK(h, cudaEventCreateWithFlags(h->ev_flush.put(), cudaEventDisableTiming));

    {
        int rc = alloc_table_buffers(h, mc);
        if (rc)
            return rc;
    }

    for (int i = 0; i < N_EV; i++)
        CK(h, cudaEventCreate(h->ev[i].put()));
    for (int i = 0; i < 4; i++)
        CK(h, cudaEventCreate(h->ev_fin[i].put()));
    CK(h, cudaEventCreate(h->ev_copy0.put()));
    CK(h, cudaEventCreate(h->ev_copy1.put()));
    CK(h, cudaEventCreateWithFlags(h->ev_copy_done.put(), cudaEventDisableTiming));
    CK(h, cudaFuncSetAttribute(k_crc32_extents, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CRC_SMEM));
    CK(h, cudaFuncSetAttribute(k_select_cuts_big, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SELB_SMEM));
    CK(h, cudaStreamSynchronize(h->s_comp));
    memset(&h->stats, 0, sizeof h->stats);
    return 0;
}

// sel_rule: a window offset (at most the window, SELB_REGIONS regions) plus max_size stays a 32-bit value
static_assert((uint64_t)SELB_REGIONS * SCAN_TILE + MKSNAP_CDC_MAX_SIZE_LIMIT <= 0xFFFFFFFFull, "max_size limit");

int mksnap_create(const mksnap_config *cfg, mksnap_t **out)
{
    if (!cfg || !out)
        return fail(nullptr, MKSNAP_E_INVAL, "null argument");
    *out = nullptr;
    mksnap *h = new mksnap;
    h->cfg = *cfg;
    mksnap_cdc_params p = cfg->cdc;
    if (p.min_size == 0 && p.max_size == 0)
        mksnap_default_cdc(&p);
    h->cfg.cdc = p;
    if (p.min_size < 64 || p.normal_size < p.min_size || p.max_size < p.normal_size ||
        p.max_size > MKSNAP_CDC_MAX_SIZE_LIMIT || p.strict_bits < p.loose_bits || p.strict_bits > 31 || p.loose_bits < 1) {
        g_create_error = "invalid cdc parameters";
        delete h;
        return MKSNAP_E_INVAL;
    }
    h->prm.min_size = p.min_size;
    h->prm.normal_size = p.normal_size;
    h->prm.max_size = p.max_size;
    h->prm.strict_lim = 1u << (32 - p.strict_bits);
    h->prm.loose_lim = 1u << (32 - p.loose_bits);
    if (cfg->device_arena_bytes == 0 || cfg->device_arena_bytes % 512 || cfg->max_extents == 0 ||
        (cfg->n_host_arenas && (cfg->host_arena_bytes == 0 || cfg->host_arena_bytes > cfg->device_arena_bytes))) {
        g_create_error = "invalid arena configuration (sizes must be non-zero, device arena multiple of 512, host arena <= device arena)";
        delete h;
        return MKSNAP_E_INVAL;
    }
    int rc = create_impl(h);
    if (rc) {
        g_create_error = h->err;
        mksnap_destroy(h);
        return rc;
    }
    *out = h;
    return 0;
}

void mksnap_destroy(mksnap_t *h)
{
    if (!h)
        return;
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    gz_free(h);
    if (h->comm && h->nccl.CommDestroy)
        h->nccl.CommDestroy(h->comm);
    delete h; // the members free the buffers, events and streams
}

int mksnap_begin(mksnap_t *h)
{
    if (!h)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    CK(h, cudaStreamSynchronize(h->s_comp));
    CK(h, cudaMemsetAsync(h->d_sc, 0, sizeof(SessionCounters), h->s_comp));
    CK(h, cudaMemsetAsync(h->d_stream_state, 0, h->max_streams * sizeof(StreamState), h->s_comp));
    if (h->fold_streams) // only the slots the last session folded into are non-zero
        CK(h, cudaMemsetAsync(h->d_stream_pure, 0, h->fold_streams * 4, h->s_comp));
    h->fold_streams = 0;
    for (auto &a : h->arenas) // an arena acquired but never submitted (a packer that failed half way) is reclaimed here
        a.acquired = false;
    h->n_streams = 0;
    h->stream_base = 0;
    h->crc_bytes = 0;
    h->crc_session_n = 0;
    h->crc_host_acc = 0;
    h->crc_host_bytes = 0;
    h->open_file = false;
    if (h->n_open) {
        std::fill(h->stream_open.begin(), h->stream_open.end(), 0);
        h->n_open = 0;
    }
    for (const auto &p : h->log_pending) // pieces of an abandoned session are dropped
        h->log_count[p.stream] = 0;
    h->log_pending.clear();
    h->log_used = 0;
    h->n_unique = 0;
    h->finished = false;
    h->in_session = true;
    return 0;
}

int mksnap_arena_acquire(mksnap_t *h, void **host_ptr, uint64_t *capacity, int32_t *arena_id)
{
    if (!h || !host_ptr || !capacity || !arena_id)
        return MKSNAP_E_INVAL;
    if (h->arenas.empty())
        return fail(h, MKSNAP_E_STATE, "handle was created with n_host_arenas = 0");
    CK(h, cudaSetDevice(h->cfg.device));
    const uint32_t n = (uint32_t)h->arenas.size();
    for (uint32_t k = 0; k < n; k++) {
        uint32_t i = (h->next_arena + k) % n;
        HostArena &a = h->arenas[i];
        if (a.acquired)
            continue;
        if (a.in_flight) {
            CK(h, cudaEventSynchronize(a.ev_h2d));
            a.in_flight = false;
        }
        a.acquired = true;
        h->next_arena = (i + 1) % n;
        *host_ptr = a.ptr;
        *capacity = h->cfg.host_arena_bytes;
        *arena_id = (int32_t)i;
        return 0;
    }
    return fail(h, MKSNAP_E_STATE, "all %u host arenas are acquired and not yet submitted", n);
}

int mksnap_arena_release(mksnap_t *h, int32_t arena_id)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->arenas[arena_id].acquired)
        return fail(h, MKSNAP_E_STATE, "arena %d was not acquired", arena_id);
    h->arenas[arena_id].acquired = false;
    return 0;
}

int mksnap_get_limits(const mksnap_t *h, mksnap_limits *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    out->max_extents = h->cfg.max_extents;
    out->max_streams = h->max_streams;
    out->max_chunks = h->max_chunks;
    out->host_arena_bytes = h->cfg.host_arena_bytes;
    out->device_arena_bytes = h->cfg.device_arena_bytes;
    out->n_host_arenas = (uint32_t)h->arenas.size();
    out->n_device_slots = h->n_slots;
    out->carry_bytes = h->d_carry.size();
    return 0;
}

// [off, off + len) inside one of the ascending spans (empty pieces need no bytes)
static bool in_spans(const mksnap_span *sp, uint64_t n, uint64_t off, uint64_t len)
{
    if (len == 0)
        return true;
    const mksnap_span *it = std::upper_bound(sp, sp + n, off, [](uint64_t v, const mksnap_span &s) { return v < s.off; });
    return it != sp && off + len <= (it - 1)->off + (it - 1)->len;
}

int mksnap_reserve_stream_log(mksnap_t *h, uint64_t bytes)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!h->log_pending.empty())
        return fail(h, MKSNAP_E_STATE, "reserve_stream_log while %llu deferred piece(s) wait in the log",
                    (unsigned long long)h->log_pending.size());
    CK(h, cudaSetDevice(h->cfg.device));
    bytes = (bytes + 63) & ~63ull; // K4 reads a piece's last block in whole 16-byte words
    if (bytes == h->d_log.size())
        return 0;
    CK(h, cudaStreamSynchronize(h->s_comp));
    h->d_log.reset();
    if (bytes && h->d_log.alloc(bytes) != cudaSuccess) {
        cudaGetLastError();
        return fail(h, MKSNAP_E_NOMEM, "stream log of %llu bytes", (unsigned long long)bytes);
    }
    return 0;
}

// Hash every piece waiting in the stream log, enqueued on the compute stream.  Pieces are grouped by stream in log
// order; a piece that continues its stream's previous group (contiguous in the log, or empty) joins it.  Round r is the
// r-th group of every stream: one K4 launch per round keeps K4's rule of one piece per stream per launch, and a slot
// that carried two streams hashes them in order (the first group's final piece closes the midstate the second starts
// from).
static int flush_log(mksnap *h, cudaStream_t sk)
{
    if (h->log_pending.empty()) {
        h->log_used = 0;
        return 0;
    }
    struct Group {
        uint64_t off, len;
        uint32_t stream, more, round;
    };
    std::vector<Group> groups;
    std::vector<uint32_t> per_round;
    std::unordered_map<uint32_t, int64_t> last; // stream -> its latest group
    for (const auto &p : h->log_pending) {
        const auto ins = last.emplace(p.stream, -1);
        int64_t &g = ins.first->second;
        if (g >= 0 && groups[g].more && (p.len == 0 || groups[g].off + groups[g].len == p.off)) {
            groups[g].len += p.len;
            groups[g].more = p.more;
            continue;
        }
        const uint32_t round = g >= 0 ? groups[g].round + 1 : 0;
        if (round == per_round.size())
            per_round.push_back(0);
        per_round[round]++;
        g = (int64_t)groups.size();
        groups.push_back(Group{p.off, p.len, p.stream, p.more, round});
    }
    const uint64_t n = groups.size();
    if (n * 3 > std::min(h->h_flush.size(), h->d_flush.size())) { // either is empty after a failed growth
        CK(h, cudaStreamSynchronize(sk));
        const uint64_t cap = std::max<uint64_t>(n, 1024);
        CK(h, h->h_flush.alloc(cap * 3));
        CK(h, h->d_flush.alloc(cap * 3));
    } else {
        CK(h, cudaEventSynchronize(h->ev_flush));
    }
    // rows ordered by round: [start n][len n][stream n][flags n]
    std::vector<uint64_t> at(per_round.size(), 0);
    for (size_t r = 1; r < per_round.size(); r++)
        at[r] = at[r - 1] + per_round[r - 1];
    uint64_t *start = h->h_flush, *len = start + n;
    uint32_t *stream = reinterpret_cast<uint32_t *>(len + n), *flags = stream + n;
    for (const Group &g : groups) {
        const uint64_t i = at[g.round]++;
        start[i] = g.off;
        len[i] = g.len;
        stream[i] = g.stream;
        flags[i] = g.more ? MKSNAP_R_MORE : 0u;
    }
    CK(h, cudaMemcpyAsync(h->d_flush, h->h_flush, n * 24, cudaMemcpyHostToDevice, sk));
    CK(h, cudaEventRecord(h->ev_flush, sk));
    h->stats.h2d_bytes += n * 24;
    const uint64_t *d_start = h->d_flush, *d_len = d_start + n;
    const uint32_t *d_stream = reinterpret_cast<const uint32_t *>(d_len + n), *d_flags = d_stream + n;
    CK(h, cudaEventRecord(h->ev[6], sk));
    for (uint64_t r = 0, o = 0; r < per_round.size(); o += per_round[r], r++) {
        const uint32_t pairs = (uint32_t)((per_round[r] + 31) / 32);
        CK(h, cudaMemsetAsync(&h->d_sc->work, 0, 4, sk));
        k_sha256_streams<<<std::min<uint32_t>(pairs, (uint32_t)h->sm_count * 4), SS_THREADS, 0, sk>>>(
            h->d_log, d_start + o, d_len + o, per_round[r], d_stream + o, d_flags + o, h->d_stream_state,
            h->d_stream_digests, &h->d_sc->work, 32u, 1u);
        LAUNCH_OK(h);
    }
    CK(h, cudaMemsetAsync(&h->d_sc->work, 0, 4, sk));
    CK(h, cudaEventRecord(h->ev[7], sk));
    h->have_flush_time = true;
    for (const auto &p : h->log_pending)
        h->log_count[p.stream] = 0;
    h->log_pending.clear();
    h->log_used = 0;
    return 0;
}

// src != nullptr: the arena comes from that pinned host arena, and of [0, used) only `spans` travel (the rest is zeroed)
static int submit_common(mksnap *h, uint32_t slot, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
                         const mksnap_range *rng, uint64_t n_rng, HostArena *src, const mksnap_span *spans = nullptr,
                         uint64_t n_spans = 0)
{
    if (!h->in_session || h->finished)
        return fail(h, MKSNAP_E_STATE, "submit outside begin/finish");
    if (used > h->cfg.device_arena_bytes)
        return fail(h, MKSNAP_E_CAPACITY, "used %llu > device arena %llu", (unsigned long long)used,
                    (unsigned long long)h->cfg.device_arena_bytes);
    if (n_ext > h->cfg.max_extents || n_rng > h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "too many extents/ranges (%llu/%llu > %llu)", (unsigned long long)n_ext,
                    (unsigned long long)n_rng, (unsigned long long)h->cfg.max_extents);

    MetaSet &m = h->meta[h->submit_idx % h->meta.size()];
    if (m.in_flight) {
        CK(h, cudaEventSynchronize(m.ev_done));
        m.in_flight = false;
    }
    uint64_t n_crc = 0, n_files = 0, pieces = 0, cdc_bytes = 0, crc_bytes = 0, big_slots = 0, cont_off = 0;
    bool have_cont = false, have_more = false;
    for (uint64_t i = 0; i < n_ext; i++) {
        const mksnap_extent &x = ext[i];
        if ((x.arena_off & 15) || x.arena_off > used || x.len > used - x.arena_off)
            return fail(h, MKSNAP_E_INVAL, "extent %llu out of bounds or not 16-byte aligned", (unsigned long long)i);
        if (x.flags & MKSNAP_X_CRC) {
            m.h_crc[n_crc].off = x.arena_off;
            m.h_crc[n_crc].len = x.len;
            m.h_crc[n_crc].suffix = x.crc_suffix;
            m.h_piece_base[n_crc] = (uint32_t)pieces;
            pieces += (x.len + CRC_PIECE - 1) / CRC_PIECE;
            if (pieces > 0xFFFFFFF0ull)
                return fail(h, MKSNAP_E_CAPACITY, "too many CRC pieces");
            crc_bytes += x.len;
            n_crc++;
        }
        if (x.flags & MKSNAP_X_CDC) {
            const bool cont = (x.flags & MKSNAP_X_CONT) != 0, more = (x.flags & MKSNAP_X_MORE) != 0;
            if (cont) {
                if (n_files != 0 || !h->open_file)
                    return fail(h, MKSNAP_E_STATE, "extent %llu: MKSNAP_X_CONT must be the first CDC extent of the submit that follows a MKSNAP_X_MORE extent",
                                (unsigned long long)i);
                if (x.arena_off < h->d_carry.size())
                    return fail(h, MKSNAP_E_INVAL, "extent %llu: a continuation starts at arena offset >= %llu (room for the open chunk)",
                                (unsigned long long)i, (unsigned long long)h->d_carry.size());
                have_cont = true;
                cont_off = x.arena_off;
            }
            if (have_more)
                return fail(h, MKSNAP_E_INVAL, "extent %llu: a MKSNAP_X_MORE extent must be the last CDC extent of its submit", (unsigned long long)i);
            if (more) {
                if (x.len == 0 || x.reserved == 0)
                    return fail(h, MKSNAP_E_INVAL, "extent %llu: MKSNAP_X_MORE needs a non-empty piece and the bytes that follow in `reserved`",
                                (unsigned long long)i);
                have_more = true;
            }
            m.h_files[n_files].off = x.arena_off;
            m.h_files[n_files].len = x.len;
            m.h_files[n_files].scratch = big_slots;
            m.h_files[n_files].more_after = more ? x.reserved : 0u;
            m.h_files[n_files].cont = cont ? 1u : 0u;
            if (x.len + (cont ? h->d_carry.size() : 0) >= SELECT_BIG_FILE) // a continuation is widened by its open chunk on the device
                big_slots += (x.len + (cont ? h->d_carry.size() : 0)) / h->prm.min_size + 2;
            cdc_bytes += x.len;
            n_files++;
        } else if (x.flags & (MKSNAP_X_MORE | MKSNAP_X_CONT)) {
            return fail(h, MKSNAP_E_INVAL, "extent %llu: MKSNAP_X_MORE / MKSNAP_X_CONT apply to MKSNAP_X_CDC extents", (unsigned long long)i);
        }
    }
    m.h_piece_base[n_crc] = (uint32_t)pieces;
    if (h->open_file && !have_cont)
        return fail(h, MKSNAP_E_STATE, "the previous submit left a file open (MKSNAP_X_MORE): this one must start with its MKSNAP_X_CONT extent");
    if (big_slots > h->table_cap) // the cut lists of the big files live in the (idle) radix key buffer
        return fail(h, MKSNAP_E_CAPACITY, "big-file cut lists need %llu slots, max_chunks allows %llu",
                    (unsigned long long)big_slots, (unsigned long long)h->table_cap);
    if (++h->stamp_epoch == 0) { // epoch wrapped: forget every stamp
        std::fill(h->stream_stamp.begin(), h->stream_stamp.end(), 0);
        h->stamp_epoch = 1;
    }
    for (uint64_t i = 0; i < n_rng; i++) {
        if ((rng[i].arena_off & 15) || rng[i].arena_off > used || rng[i].len > used - rng[i].arena_off)
            return fail(h, MKSNAP_E_INVAL, "range %llu out of bounds or not 16-byte aligned", (unsigned long long)i);
        if (rng[i].stream >= h->max_streams)
            return fail(h, MKSNAP_E_CAPACITY, "range %llu: stream slot %u >= %llu", (unsigned long long)i, rng[i].stream,
                        (unsigned long long)h->max_streams);
        if ((rng[i].flags & MKSNAP_R_MORE) && (rng[i].len == 0 || rng[i].len % 64))
            return fail(h, MKSNAP_E_INVAL, "range %llu: a piece with MKSNAP_R_MORE must be a non-empty multiple of 64 bytes",
                        (unsigned long long)i);
        if (h->stream_stamp[rng[i].stream] == h->stamp_epoch)
            return fail(h, MKSNAP_E_INVAL, "range %llu: stream slot %u already has a piece in this submit (one piece per stream per submit)",
                        (unsigned long long)i, rng[i].stream);
        const bool defer = (rng[i].flags & MKSNAP_R_DEFER) != 0;
        if (h->stream_open[rng[i].stream] && h->stream_defer[rng[i].stream] != defer)
            return fail(h, MKSNAP_E_INVAL, "range %llu: stream slot %u mixes MKSNAP_R_DEFER and inline pieces in one stream",
                        (unsigned long long)i, rng[i].stream);
        h->stream_stamp[rng[i].stream] = h->stamp_epoch;
    }
    // deferred pieces go to the stream log; the rest (and deferred pieces the log cannot hold) is hashed by this submit
    std::vector<uint64_t> logged;
    uint64_t n_inline = 0;
    for (uint64_t i = 0; i < n_rng; i++) {
        if ((rng[i].flags & MKSNAP_R_DEFER) && h->d_log.size() && rng[i].len <= h->d_log.size()) {
            logged.push_back(i);
            continue;
        }
        m.h_rstart[n_inline] = rng[i].arena_off;
        m.h_rlen[n_inline] = rng[i].len;
        m.h_rstream[n_inline] = rng[i].stream;
        m.h_rflags[n_inline] = rng[i].flags & MKSNAP_R_MORE;
        n_inline++;
    }

    uint8_t *d_arena = h->d_slot[slot];
    // ---- copy stream: arena + tables ----
    cudaStream_t sc = h->s_copy, sk = h->s_comp;
    if (h->slot_used[slot])
        CK(h, cudaStreamWaitEvent(sc, h->ev_slot_free[slot], 0));
    if (src) {
        CK(h, cudaEventRecord(h->ev_copy0, sc));
        uint64_t at = 0, sent = 0; // bytes before `at` are placed; a gap between spans is zeroed
        for (uint64_t k = 0; k < n_spans; k++) {
            if (spans[k].off > at)
                CK(h, cudaMemsetAsync(d_arena + at, 0, spans[k].off - at, sc));
            if (spans[k].len)
                CK(h, cudaMemcpyAsync(d_arena + spans[k].off, src->ptr + spans[k].off, spans[k].len, cudaMemcpyHostToDevice, sc));
            at = spans[k].off + spans[k].len;
            sent += spans[k].len;
        }
        if (used > at)
            CK(h, cudaMemsetAsync(d_arena + at, 0, used - at, sc));
        // zero the tail up to the next 512 so row-granular readers see zeros
        const uint64_t padded = std::min<uint64_t>((used + 511) & ~511ull, h->cfg.device_arena_bytes);
        if (padded > used)
            CK(h, cudaMemsetAsync(d_arena + used, 0, padded - used, sc));
        CK(h, cudaEventRecord(h->ev_copy1, sc));
        CK(h, cudaEventRecord(src->ev_h2d, sc));
        src->in_flight = true;
        src->acquired = false;
        h->stats.h2d_bytes += sent;
        h->have_h2d_time = true;
    }
    if (n_crc) {
        CK(h, cudaMemcpyAsync(m.d_crc, m.h_crc, n_crc * sizeof(CrcExtent), cudaMemcpyHostToDevice, sc));
        CK(h, cudaMemcpyAsync(m.d_piece_base, m.h_piece_base, (n_crc + 1) * 4, cudaMemcpyHostToDevice, sc));
    }
    if (n_files)
        CK(h, cudaMemcpyAsync(m.d_files, m.h_files, n_files * sizeof(CdcFile), cudaMemcpyHostToDevice, sc));
    if (n_inline) {
        CK(h, cudaMemcpyAsync(m.d_rstart, m.h_rstart, n_inline * 8, cudaMemcpyHostToDevice, sc));
        CK(h, cudaMemcpyAsync(m.d_rlen, m.h_rlen, n_inline * 8, cudaMemcpyHostToDevice, sc));
        CK(h, cudaMemcpyAsync(m.d_rstream, m.h_rstream, n_inline * 4, cudaMemcpyHostToDevice, sc));
        CK(h, cudaMemcpyAsync(m.d_rflags, m.h_rflags, n_inline * 4, cudaMemcpyHostToDevice, sc));
    }
    h->stats.h2d_bytes += n_crc * sizeof(CrcExtent) + (n_crc ? (n_crc + 1) * 4 : 0) + n_files * sizeof(CdcFile) + n_inline * 16;
    CK(h, cudaEventRecord(h->ev_copy_done, sc));

    // ---- compute stream ----
    CK(h, cudaStreamWaitEvent(sk, h->ev_copy_done, 0));
    if (have_cont) { // prepend the open chunk of the file that continues here (before anything scans the arena)
        k_carry_in<<<1, 256, 0, sk>>>(h->d_carry, d_arena, cont_off, m.d_files, 0u, h->d_sc);
        LAUNCH_OK(h);
    }
    // the scan comes first: with CRC extents in the submit it also leaves the CRC of every arena row in d_part, and
    // K0 combines those instead of reading the arena a second time
    CK(h, cudaEventRecord(h->ev[0], sk));
    if (n_files) {
        const uint32_t n_regions = (uint32_t)((used + SCAN_TILE - 1) / SCAN_TILE);
        CK(h, cudaMemsetAsync(h->d_pool_count, 0, 4, sk));
        int rc = n_crc && pieces ? launch_scan<MK_CRC_SCAN_SHAPE>(h, slot, n_regions, sk)
                                 : launch_scan_cfg(h, slot, n_regions, sk);
        if (rc)
            return rc;
    }
    CK(h, cudaEventRecord(h->ev[1], sk));
    if (n_crc && pieces) {
        const uint32_t grid = (uint32_t)std::min<uint64_t>(h->sm_count, (pieces + 31) / 32);
        CK(h, cudaMemsetAsync(m.d_ext_pure, 0, n_crc * 4, sk));
        k_crc32_extents<<<grid, CRC_THREADS, CRC_SMEM, sk>>>(d_arena, m.d_crc, m.d_piece_base, (uint32_t)n_crc,
                                                            (uint32_t)pieces, h->d_consts, m.d_ext_pure, &h->d_sc->crc_acc,
                                                            n_files ? h->d_part.get() : nullptr);
        LAUNCH_OK(h);
    }
    if (n_crc) { // pure(extent) of this submit's extents joins the session table (zero-length extents keep their slot)
        if (!pieces)
            CK(h, cudaMemsetAsync(m.d_ext_pure, 0, n_crc * 4, sk));
        if (h->crc_session_n < h->d_crc_session.size())
            CK(h, cudaMemcpyAsync(h->d_crc_session + h->crc_session_n, m.d_ext_pure,
                                  std::min<uint64_t>(n_crc, h->d_crc_session.size() - h->crc_session_n) * 4, cudaMemcpyDeviceToDevice, sk));
        h->crc_session_n += n_crc;
    }
    CK(h, cudaEventRecord(h->ev[2], sk));
    if (n_files) {
        const uint32_t nb = (uint32_t)((n_files + 127) / 128);
        k_select_cuts<0><<<nb, 128, 0, sk>>>(m.d_files, (uint32_t)n_files, h->prm, h->d_tiles, h->d_pool, h->d_counts,
                                             nullptr, h->d_sc, h->max_chunks, 0, nullptr, nullptr, nullptr);
        LAUNCH_OK(h);
        const bool big_files = big_slots != 0;
        if (big_files) {
            k_select_cuts_big<<<(uint32_t)n_files, SELB_THREADS, SELB_SMEM, sk>>>(m.d_files, (uint32_t)n_files, h->prm, h->d_tiles,
                                                                       h->d_pool, h->d_counts, h->d_keys[0], h->d_sc);
            LAUNCH_OK(h);
        }
        int rc = scan_u32(h, h->d_counts, h->d_bases, n_files, sk);
        if (rc)
            return rc;
        k_batch_begin<<<1, 64, 0, sk>>>(h->d_sc, h->d_counts, h->d_bases, (uint32_t)n_files, h->max_chunks, cdc_bytes, have_cont ? 1u : 0u);
        LAUNCH_OK(h);
        k_select_cuts<1><<<nb, 128, 0, sk>>>(m.d_files, (uint32_t)n_files, h->prm, h->d_tiles, h->d_pool, h->d_counts,
                                             h->d_bases, h->d_sc, h->max_chunks, h->stream_base, h->d_chunk_start,
                                             h->d_chunk_len, h->d_chunk_end);
        LAUNCH_OK(h);
        if (big_files) {
            k_expand_big_cuts<<<(uint32_t)n_files, 256, 0, sk>>>(m.d_files, (uint32_t)n_files, h->d_counts, h->d_bases,
                                                              h->d_keys[0], h->d_sc, h->max_chunks, h->stream_base,
                                                              h->d_chunk_start, h->d_chunk_len, h->d_chunk_end);
            LAUNCH_OK(h);
        }
    }
    CK(h, cudaEventRecord(h->ev[3], sk));
    if (n_files) {
        const uint32_t *order = nullptr;
        if (h->sha_order) { // longest chunks first (see k_len_order)
            k_len_hist<<<h->sm_count * 2, LEN_THREADS, 0, sk>>>(h->d_chunk_len, h->d_sc);
            LAUNCH_OK(h);
            k_len_order<<<h->sm_count * 2, LEN_THREADS, 0, sk>>>(h->d_chunk_len, h->d_sc, h->d_order);
            LAUNCH_OK(h);
            order = h->d_order;
        }
        if (h->sha_fma)
            k_sha256_ranges<true><<<sha_grid(h), SHA_THREADS, 0, sk>>>(d_arena, h->d_chunk_start, h->d_chunk_len, h->d_sc,
                                                                      h->d_digests, 1u, order);
        else
            k_sha256_ranges<false><<<sha_grid(h), SHA_THREADS, 0, sk>>>(d_arena, h->d_chunk_start, h->d_chunk_len, h->d_sc,
                                                                       h->d_digests, 1u, order);
        LAUNCH_OK(h);
        k_batch_end<<<1, 32, 0, sk>>>(h->d_sc);
        LAUNCH_OK(h);
        if (have_more) { // park the open chunk before this slot is recycled
            k_carry_out<<<1, 256, 0, sk>>>(d_arena, h->d_carry, h->d_carry.size(), h->d_sc);
            LAUNCH_OK(h);
        }
    }
    CK(h, cudaEventRecord(h->ev[4], sk));
    for (const uint64_t i : logged) { // into the log before the slot is recycled; a full log is hashed first
        const mksnap_range &r = rng[i];
        uint64_t off = (h->log_used + 15) & ~15ull;
        if (off + r.len > h->d_log.size()) {
            int rc = flush_log(h, sk);
            if (rc)
                return rc;
            off = 0;
        }
        if (r.len)
            CK(h, cudaMemcpyAsync(h->d_log + off, d_arena + r.arena_off, r.len, cudaMemcpyDeviceToDevice, sk));
        h->log_pending.push_back(mksnap::LogPiece{off, r.len, r.stream, r.flags & MKSNAP_R_MORE});
        h->log_count[r.stream]++;
        h->log_used = off + r.len;
    }
    bool behind_log = false; // an inline piece on a slot whose earlier pieces wait in the log
    for (uint64_t k = 0; k < n_inline; k++)
        behind_log |= h->log_count[m.h_rstream[k]] != 0;
    if (behind_log) {
        int rc = flush_log(h, sk);
        if (rc)
            return rc;
    }
    if (n_inline) {
        // K4: warp pairs, 32 streams each, spread one pair per SM first (a pair then owns its two sub-partitions)
        CK(h, cudaMemsetAsync(&h->d_sc->work, 0, 4, sk));
        const uint32_t pairs = (uint32_t)((n_inline + 31) / 32);
        k_sha256_streams<<<std::min<uint32_t>(pairs, (uint32_t)h->sm_count * 4), SS_THREADS, 0, sk>>>(
            d_arena, m.d_rstart, m.d_rlen, (uint32_t)n_inline, m.d_rstream, m.d_rflags, h->d_stream_state, h->d_stream_digests,
            &h->d_sc->work, 32u, 1u);
        LAUNCH_OK(h);
        CK(h, cudaMemsetAsync(&h->d_sc->work, 0, 4, sk));
    }
    CK(h, cudaEventRecord(h->ev[5], sk));
    CK(h, cudaEventRecord(h->ev_slot_free[slot], sk));
    CK(h, cudaEventRecord(m.ev_done, sk));
    m.in_flight = true;
    h->slot_used[slot] = true;
    h->have_submit_times = true;
    for (uint64_t i = 0; i < n_rng; i++) {
        const bool more = (rng[i].flags & MKSNAP_R_MORE) != 0;
        uint8_t &open = h->stream_open[rng[i].stream];
        if (more && !open)
            h->n_open++;
        else if (!more && open)
            h->n_open--;
        open = more;
        h->stream_defer[rng[i].stream] = (rng[i].flags & MKSNAP_R_DEFER) != 0;
        if (!more)
            h->n_streams = std::max<uint64_t>(h->n_streams, (uint64_t)rng[i].stream + 1);
    }
    h->open_file = have_more;
    h->stream_base += used;
    h->crc_bytes += crc_bytes;
    h->submit_idx++;
    return 0;
}

int mksnap_arena_submit_spans(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_span *spans, uint64_t n_spans,
                              const mksnap_extent *extents, uint64_t n_extents, const mksnap_range *ranges, uint64_t n_ranges)
{
    if (!h)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->arenas[arena_id].acquired)
        return fail(h, MKSNAP_E_STATE, "arena %d was not acquired", arena_id);
    if (used > h->cfg.host_arena_bytes)
        return fail(h, MKSNAP_E_CAPACITY, "used %llu > host arena %llu", (unsigned long long)used,
                    (unsigned long long)h->cfg.host_arena_bytes);
    if ((!spans && n_spans) || (!extents && n_extents) || (!ranges && n_ranges))
        return fail(h, MKSNAP_E_INVAL, "null table");
    for (uint64_t k = 0, end = 0; k < n_spans; k++) {
        const mksnap_span &s = spans[k];
        if ((s.off | s.len) & 15 || s.off < end || s.off > used || s.len > used - s.off)
            return fail(h, MKSNAP_E_INVAL, "span %llu: not 16-byte aligned, out of order or outside [0, used)", (unsigned long long)k);
        end = s.off + s.len;
    }
    for (uint64_t i = 0; i < n_extents; i++)
        if (!in_spans(spans, n_spans, extents[i].arena_off, extents[i].len))
            return fail(h, MKSNAP_E_INVAL, "extent %llu is not inside one of the submitted spans", (unsigned long long)i);
    for (uint64_t i = 0; i < n_ranges; i++)
        if (!in_spans(spans, n_spans, ranges[i].arena_off, ranges[i].len))
            return fail(h, MKSNAP_E_INVAL, "range %llu is not inside one of the submitted spans", (unsigned long long)i);
    const uint32_t slot = (uint32_t)(h->submit_idx % h->n_slots);
    return submit_common(h, slot, used, extents, n_extents, ranges, n_ranges, &h->arenas[arena_id], spans, n_spans);
}

int mksnap_arena_submit(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_extent *extents,
                        uint64_t n_extents, const mksnap_range *ranges, uint64_t n_ranges)
{
    if (!h)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->arenas[arena_id].acquired)
        return fail(h, MKSNAP_E_STATE, "arena %d was not acquired", arena_id);
    if (used > h->cfg.host_arena_bytes)
        return fail(h, MKSNAP_E_CAPACITY, "used %llu > host arena %llu", (unsigned long long)used,
                    (unsigned long long)h->cfg.host_arena_bytes);
    const mksnap_span whole{0, used}; // `used` need not be a multiple of 16 here
    const uint32_t slot = (uint32_t)(h->submit_idx % h->n_slots);
    return submit_common(h, slot, used, extents, n_extents, ranges, n_ranges, &h->arenas[arena_id], &whole, 1);
}

int mksnap_chunks_add(mksnap_t *h, const uint8_t *digests, uint64_t n)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!digests && n)
        return fail(h, MKSNAP_E_INVAL, "chunks_add: null digest table");
    if (!h->in_session || h->finished)
        return fail(h, MKSNAP_E_STATE, "chunks_add outside begin/finish");
    if (n > MKSNAP_CHUNKS_ADD_MAX)
        return fail(h, MKSNAP_E_CAPACITY, "chunks_add: %llu rows in one call, at most %u", (unsigned long long)n,
                    MKSNAP_CHUNKS_ADD_MAX);
    if (n == 0)
        return 0;
    CK(h, cudaSetDevice(h->cfg.device));
    cudaStream_t s = h->s_comp; // behind the submits enqueued before this call
    if (!h->ev_add) { // created last: a first call that failed part-way allocates again
        CK(h, h->h_add.alloc((uint64_t)MKSNAP_CHUNKS_ADD_MAX * 32));
        CK(h, h->d_add.alloc((uint64_t)MKSNAP_CHUNKS_ADD_MAX * 32));
        CK(h, cudaEventCreateWithFlags(h->ev_add.put(), cudaEventDisableTiming));
    } else {
        CK(h, cudaEventSynchronize(h->ev_add)); // the previous call's copy has left the staging buffer
    }
    memcpy(h->h_add, digests, n * 32);
    CK(h, cudaMemcpyAsync(h->d_add, h->h_add, n * 32, cudaMemcpyHostToDevice, s));
    CK(h, cudaEventRecord(h->ev_add, s));
    h->stats.h2d_bytes += n * 32;
    const uint32_t grid = (uint32_t)std::min<uint64_t>((2 * n + APPEND_THREADS - 1) / APPEND_THREADS, (uint64_t)h->sm_count * 4);
    k_chunks_append<<<grid, APPEND_THREADS, 0, s>>>(reinterpret_cast<const uint4 *>(h->d_add.get()), (uint32_t)n, h->d_sc,
                                                    h->max_chunks, reinterpret_cast<uint4 *>(h->d_digests.get()), h->d_chunk_end);
    LAUNCH_OK(h);
    k_chunks_commit<<<1, 32, 0, s>>>(h->d_sc, (uint32_t)n, h->max_chunks);
    LAUNCH_OK(h);
    return 0;
}

int mksnap_get_cdc(const mksnap_t *h, mksnap_cdc_params *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    *out = h->cfg.cdc; // create() filled in the defaults
    return 0;
}

int mksnap_device_arena(mksnap_t *h, uint32_t slot, void **device_ptr, uint64_t *capacity)
{
    if (!h || slot >= h->n_slots || !device_ptr || !capacity)
        return MKSNAP_E_INVAL;
    *device_ptr = h->d_slot[slot];
    *capacity = h->cfg.device_arena_bytes;
    return 0;
}

int mksnap_device_upload(mksnap_t *h, uint32_t slot, uint64_t dst_off, const void *src, uint64_t n)
{
    if (!h || slot >= h->n_slots || dst_off > h->cfg.device_arena_bytes || n > h->cfg.device_arena_bytes - dst_off)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    CK(h, cudaStreamSynchronize(h->s_comp));
    CK(h, cudaMemcpy(h->d_slot[slot] + dst_off, src, n, cudaMemcpyHostToDevice));
    h->stats.h2d_bytes += n;
    return 0;
}

int mksnap_device_download(mksnap_t *h, uint32_t slot, uint64_t src_off, void *dst, uint64_t n)
{
    if (!h || slot >= h->n_slots || src_off > h->cfg.device_arena_bytes || n > h->cfg.device_arena_bytes - src_off)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    CK(h, cudaStreamSynchronize(h->s_comp));
    CK(h, cudaMemcpy(dst, h->d_slot[slot] + src_off, n, cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += n;
    return 0;
}

int mksnap_device_submit(mksnap_t *h, uint32_t slot, uint64_t used, const mksnap_extent *extents, uint64_t n_extents,
                         const mksnap_range *ranges, uint64_t n_ranges)
{
    if (!h || slot >= h->n_slots)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    return submit_common(h, slot, used, extents, n_extents, ranges, n_ranges, nullptr);
}

int mksnap_synth_fill(mksnap_t *h, uint32_t slot, uint64_t byte_off, uint64_t n, uint64_t seed)
{
    if (!h || slot >= h->n_slots || (byte_off & 15) || (n & 15) || byte_off > h->cfg.device_arena_bytes ||
        n > h->cfg.device_arena_bytes - byte_off)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    if (n == 0)
        return 0;
    k_synth_fill<<<h->sm_count * 8, 256, 0, h->s_comp>>>(reinterpret_cast<uint64_t *>(h->d_slot[slot] + byte_off),
                                                         byte_off / 8, n / 8, seed);
    LAUNCH_OK(h);
    return 0;
}

int mksnap_memset(mksnap_t *h, uint32_t slot, uint64_t byte_off, uint64_t n, int value)
{
    if (!h || slot >= h->n_slots || byte_off > h->cfg.device_arena_bytes || n > h->cfg.device_arena_bytes - byte_off)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    CK(h, cudaMemsetAsync(h->d_slot[slot] + byte_off, value, n, h->s_comp));
    return 0;
}

int mksnap_sync(mksnap_t *h)
{
    if (!h)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    CK(h, cudaStreamSynchronize(h->s_copy));
    CK(h, cudaStreamSynchronize(h->s_comp));
    return 0;
}

int mksnap_finish(mksnap_t *h, mksnap_result *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "finish without begin");
    CK(h, cudaSetDevice(h->cfg.device));
    cudaStream_t s = h->s_comp;
    CK(h, cudaMemcpyAsync(h->h_sc, h->d_sc, sizeof(SessionCounters), cudaMemcpyDeviceToHost, s));
    CK(h, cudaStreamSynchronize(s));
    h->stats.d2h_bytes += sizeof(SessionCounters);
    if (h->h_sc->err & 1u)
        return fail(h, MKSNAP_E_CAPACITY, "candidate pool overflow (capacity %u entries): pathologically dense candidates", h->pool_cap);
    if (h->h_sc->err & 4u)
        return fail(h, MKSNAP_E_CUDA, "k_gear_scan: dynamic shared memory does not start where the layout plan assumes");
    if (h->h_sc->err & 8u)
        return fail(h, MKSNAP_E_STATE, "internal: open chunk of a continued file exceeds the carry buffer");
    if (h->open_file)
        return fail(h, MKSNAP_E_STATE, "finish: the last submit left a file open (MKSNAP_X_MORE without its continuation)");
    if (h->n_open)
        return fail(h, MKSNAP_E_STATE, "finish: %llu stream(s) left open (last piece carried MKSNAP_R_MORE)",
                    (unsigned long long)h->n_open);
    if (h->h_sc->err & 2u)
        return fail(h, MKSNAP_E_CAPACITY, "chunk table overflow (max_chunks = %llu)", (unsigned long long)h->max_chunks);
    int rc = flush_log(h, s);
    if (rc)
        return rc;
    const uint64_t n = h->h_sc->n_chunks;
    CK(h, cudaEventRecord(h->ev_fin[0], s));
    rc = sort_unique_root(h, h->d_digests, n, s);
    if (rc)
        return rc;
    CK(h, cudaEventRecord(h->ev_fin[1], s));
    if (h->n_ranks > 1) {
        // one rank of several: the content address is the root of the GLOBAL table, computed by the exchange step;
        // a root over this rank's shard would be latency-bound Merkle levels nobody reads
        memset(h->root, 0, 32);
    } else {
        rc = merkle_root(h, s);
        if (rc)
            return rc;
    }
    CK(h, cudaEventRecord(h->ev_fin[2], s));
    CK(h, cudaStreamSynchronize(s));
    h->have_fin_times = true;
    memset(out, 0, sizeof *out);
    out->crc_pure = h->h_sc->crc_acc ^ h->crc_host_acc;
    out->crc_bytes = h->crc_bytes + h->crc_host_bytes;
    out->cdc_bytes = h->h_sc->cdc_bytes;
    out->n_files = h->h_sc->n_files;
    out->n_chunks = n;
    out->n_unique = h->n_unique;
    memcpy(out->root, h->root, 32);
    out->n_streams = h->n_streams;
    h->last_result = *out;
    h->finished = true;
    return 0;
}

uint32_t mksnap_ctx_crc32(const mksnap_result *res)
{
    // standard CRC = pure ^ (0xFFFFFFFF * x^(8L)) ^ 0xFFFFFFFF
    const uint64_t M = 0xFFFFFFFFull;
    const uint64_t bits = ((res->crc_bytes % M) * 8ull) % M;
    return res->crc_pure ^ crc_mulmod(0xFFFFFFFFu, xpow_bits(bits)) ^ 0xFFFFFFFFu;
}

int mksnap_crc_add(mksnap_t *h, uint32_t pure, uint64_t len, uint64_t crc_suffix)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!h->in_session || h->finished)
        return fail(h, MKSNAP_E_STATE, "crc_add outside begin/finish");
    const uint64_t M = 0xFFFFFFFFull;
    h->crc_host_acc ^= crc_mulmod(pure, xpow_bits(((crc_suffix % M) * 8ull) % M));
    h->crc_host_bytes += len;
    return 0;
}

uint32_t mksnap_crc_concat(uint32_t pure_a, uint32_t pure_b, uint64_t len_b)
{
    const uint64_t M = 0xFFFFFFFFull;
    return crc_mulmod(pure_a, xpow_bits(((len_b % M) * 8ull) % M)) ^ pure_b;
}

int mksnap_get_extent_crcs(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out)
{
    if (!h || !h->finished || !n_out)
        return h ? fail(h, MKSNAP_E_STATE, "get_extent_crcs before finish") : MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    *n_out = h->crc_session_n;
    if (h->crc_session_n > h->d_crc_session.size())
        return fail(h, MKSNAP_E_CAPACITY, "the session submitted %llu CRC extents, the per-extent table keeps %llu",
                    (unsigned long long)h->crc_session_n, (unsigned long long)h->d_crc_session.size());
    if (!pure || h->crc_session_n > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need %llu entries", (unsigned long long)h->crc_session_n);
    if (h->crc_session_n)
        CK(h, cudaMemcpy(pure, h->d_crc_session, h->crc_session_n * 4, cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += h->crc_session_n * 4;
    return 0;
}

static_assert(sizeof(CrcUse) == sizeof(mksnap_crc_use), "k_crc_fold reads mksnap_crc_use rows");

int mksnap_crc_fold(mksnap_t *h, const mksnap_crc_use *uses, uint64_t n)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!uses && n)
        return fail(h, MKSNAP_E_INVAL, "crc_fold: null use table");
    if (!h->in_session || h->finished)
        return fail(h, MKSNAP_E_STATE, "crc_fold outside begin/finish");
    if (n > h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "crc_fold: %llu uses in one call, max_extents is %llu", (unsigned long long)n,
                    (unsigned long long)h->cfg.max_extents);
    if (h->crc_session_n > h->d_crc_session.size())
        return fail(h, MKSNAP_E_CAPACITY, "crc_fold: the session submitted %llu CRC extents, the per-extent table keeps %llu",
                    (unsigned long long)h->crc_session_n, (unsigned long long)h->d_crc_session.size());
    uint64_t hi = 0;
    for (uint64_t i = 0; i < n; i++) {
        const mksnap_crc_use &u = uses[i];
        if (u.flags & ~MKSNAP_U_VALUE)
            return fail(h, MKSNAP_E_INVAL, "crc_fold: use %llu has unknown flags %#x", (unsigned long long)i, u.flags);
        if (u.stream >= h->max_streams)
            return fail(h, MKSNAP_E_INVAL, "crc_fold: use %llu names stream %u, max_streams is %llu", (unsigned long long)i,
                        u.stream, (unsigned long long)h->max_streams);
        if (!(u.flags & MKSNAP_U_VALUE) && u.src >= h->crc_session_n)
            return fail(h, MKSNAP_E_INVAL, "crc_fold: use %llu names extent %llu, the session has submitted %llu CRC extents",
                        (unsigned long long)i, (unsigned long long)u.src, (unsigned long long)h->crc_session_n);
        hi = std::max<uint64_t>(hi, (uint64_t)u.stream + 1);
    }
    if (n == 0)
        return 0;
    CK(h, cudaSetDevice(h->cfg.device));
    cudaStream_t s = h->s_comp; // after the K0 runs and the d_crc_session copies the uses read
    if (!h->d_stream_pure) { // allocated last: a first call that failed part-way allocates again
        CK(h, h->d_uses.alloc(h->cfg.max_extents));
        CK(h, h->d_stream_pure.alloc(h->max_streams));
        CK(h, cudaMemsetAsync(h->d_stream_pure, 0, h->max_streams * 4, s));
    }
    CK(h, cudaMemcpyAsync(h->d_uses, uses, n * sizeof(CrcUse), cudaMemcpyHostToDevice, s));
    CK(h, cudaStreamSynchronize(s)); // the caller's table is free once this returns, pinned or not
    h->stats.h2d_bytes += n * sizeof(CrcUse);
    k_crc_fold<<<(uint32_t)((n + FOLD_THREADS - 1) / FOLD_THREADS), FOLD_THREADS, 0, s>>>(h->d_uses, (uint32_t)n, h->d_crc_session,
                                                                                       h->d_consts, h->d_stream_pure);
    LAUNCH_OK(h);
    h->fold_streams = std::max(h->fold_streams, hi);
    return 0;
}

int mksnap_get_crc_streams(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out)
{
    if (!h || !n_out)
        return MKSNAP_E_INVAL;
    if (!h->finished)
        return fail(h, MKSNAP_E_STATE, "get_crc_streams before finish");
    CK(h, cudaSetDevice(h->cfg.device));
    *n_out = h->fold_streams;
    if (h->fold_streams > capacity || (!pure && h->fold_streams))
        return fail(h, MKSNAP_E_CAPACITY, "need %llu entries", (unsigned long long)h->fold_streams);
    if (h->fold_streams)
        CK(h, cudaMemcpy(pure, h->d_stream_pure, h->fold_streams * 4, cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += h->fold_streams * 4;
    return 0;
}

uint32_t mksnap_crc_prepend(const void *prefix, uint64_t n, uint32_t pure_rest, uint64_t len_rest)
{
    const uint8_t *p = static_cast<const uint8_t *>(prefix);
    uint32_t c = 0; // pure(prefix): the CRC register from 0, no final xor
    for (uint64_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++)
            c = (c >> 1) ^ (MK_CRC_POLY & (0u - (c & 1u)));
    }
    const uint64_t M = 0xFFFFFFFFull;
    const uint32_t pure = crc_mulmod(c, xpow_bits(((len_rest % M) * 8ull) % M)) ^ pure_rest;
    return pure ^ crc_mulmod(0xFFFFFFFFu, xpow_bits((((n + len_rest) % M) * 8ull) % M)) ^ 0xFFFFFFFFu;
}

int mksnap_get_chunks(mksnap_t *h, uint64_t *ends, uint8_t *digests, uint64_t capacity)
{
    if (!h || !h->finished)
        return h ? fail(h, MKSNAP_E_STATE, "get_chunks before finish") : MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    const uint64_t n = h->last_result.n_chunks;
    if (n > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need %llu rows", (unsigned long long)n);
    if (ends && n)
        CK(h, cudaMemcpy(ends, h->d_chunk_end, n * 8, cudaMemcpyDeviceToHost));
    if (digests && n)
        CK(h, cudaMemcpy(digests, h->d_digests, n * 32, cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += (ends ? n * 8 : 0) + (digests ? n * 32 : 0);
    return 0;
}

uint64_t mksnap_table_rows(mksnap_t *h) { return h && h->finished ? h->n_unique : 0; }

int mksnap_get_table(mksnap_t *h, uint8_t *table, uint64_t capacity_rows)
{
    if (!h || !h->finished || !table)
        return h ? fail(h, MKSNAP_E_STATE, "get_table before finish") : MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    if (h->n_unique > capacity_rows)
        return fail(h, MKSNAP_E_CAPACITY, "need %llu rows", (unsigned long long)h->n_unique);
    if (h->n_unique)
        CK(h, cudaMemcpy(table, h->d_table, h->n_unique * 32, cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += h->n_unique * 32;
    return 0;
}

int mksnap_get_stream_digests(mksnap_t *h, uint8_t *digests, uint64_t capacity)
{
    if (!h || !digests)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    if (h->n_streams > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need %llu rows", (unsigned long long)h->n_streams);
    CK(h, cudaStreamSynchronize(h->s_comp));
    if (h->n_streams)
        CK(h, cudaMemcpy(digests, h->d_stream_digests, h->n_streams * 32, cudaMemcpyDeviceToHost));
    h->stats.d2h_bytes += h->n_streams * 32;
    return 0;
}

int mksnap_stats(mksnap_t *h, mksnap_stats_t *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    CK(h, cudaStreamSynchronize(h->s_copy));
    CK(h, cudaStreamSynchronize(h->s_comp));
    if (h->have_submit_times) {
        float t[5];
        for (int i = 0; i < 5; i++)
            CK(h, cudaEventElapsedTime(&t[i], h->ev[i], h->ev[i + 1]));
        h->stats.ms_scan = t[0];
        h->stats.ms_crc = t[1];
        h->stats.ms_select = t[2];
        h->stats.ms_sha = t[3];
        h->stats.ms_stream = t[4];
        CK(h, cudaEventElapsedTime(&h->stats.ms_total, h->ev[0], h->ev[5]));
    }
    if (h->have_h2d_time)
        CK(h, cudaEventElapsedTime(&h->stats.ms_h2d, h->ev_copy0, h->ev_copy1));
    if (h->have_fin_times) {
        CK(h, cudaEventElapsedTime(&h->stats.ms_sort, h->ev_fin[0], h->ev_fin[1]));
        CK(h, cudaEventElapsedTime(&h->stats.ms_root, h->ev_fin[1], h->ev_fin[2]));
    }
    if (h->have_flush_time)
        CK(h, cudaEventElapsedTime(&h->stats.ms_flush, h->ev[6], h->ev[7]));
    *out = h->stats;
    return 0;
}
#include "mksnap_comm.inc"

} // extern "C"

#include "mksnap_inflate.cuh"
