// mksnap_kernels.cuh — hand-written sm_90a kernels of the snapshot+hash path.
//
//   K0  k_crc32_extents   CRC-32/IEEE of the context stream      (HBM-read bound, or a combine of K1's row CRCs)
//   K0f k_crc_fold        extent values folded into many streams (latency, small)
//   K1  k_roll_scan       Roll-32 candidate scan [+ row CRCs]    (HBM-read bound)
//   K1b k_select_cuts     min/normal/max cut selection per file  (latency, tiny)
//   K2  k_sha256_ranges   SHA-256 of the chunks                  (int-ALU bound)
//   K2a k_chunks_append   remembered chunk digests into the table (copy, tiny)
//       (the serial layer-tar streams and the Merkle levels of the table root
//        are K4, mksnap_sha_stream.cuh)
//   K3  radix sort / unique of 256-bit digests                   (HBM, tiny)
//
// Reference arithmetic being replaced (all Go stdlib behind these call sites):
//   hash/crc32   <- lib/builder/step/add_copy_step.go:104-119,230-237
//   crypto/sha256<- lib/builder/step/common.go:44-55
// Everything here is 32-bit integer / byte work: no tensor cores, no floats.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "mksnap_sha_stream.cuh" // K4: serial-stream SHA-256 (warp pairs)

namespace mk {

// ------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------
#define MK_CRC_POLY 0xEDB88320u
#define MK_GOLDEN64 0x9E3779B97F4A7C15ull

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z)
{
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// (a*b) mod P in the reflected representation (bit 31 = x^0).
__host__ __device__ __forceinline__ uint32_t crc_mulmod(uint32_t a, uint32_t b)
{
    uint32_t acc = 0;
#pragma unroll
    for (int k = 31; k >= 0; --k) {
        acc ^= (0u - ((a >> k) & 1u)) & b;
        b = (b >> 1) ^ ((0u - (b & 1u)) & MK_CRC_POLY);
    }
    return acc;
}

// Table lookups: tables are replicated per lane ([value][32 lanes] words) so a warp-wide lookup
// never bank-conflicts.  Address = lane_base + byte*128, built as PRMT (byte extract, ALU pipe) +
// IMAD (FMA pipe) and fed to ld.shared directly: 3 issue slots per lookup instead of the 5 the
// generic-pointer path costs.
__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
template <int K> __device__ __forceinline__ uint32_t byte_of(uint32_t w)
{
    return __byte_perm(w, 0, 0x4440 + K); // zero-extended byte K
}
// a*2^k + b and a + b on the FMA pipe (IMAD): the ALU pipe (LOP3/SHF/PRMT) is the
// bottleneck of every kernel here, so additions that the compiler would emit as IADD3 are steered to IMAD.
__device__ __forceinline__ uint32_t fma_add(uint32_t a, uint32_t b)
{
    uint32_t d;
    asm("mad.lo.u32 %0, %1, 1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
// ptxas folds "a*1+b" back into IADD3; with the multiplier in a register it knows nothing about (the
// host passes 1 as a kernel argument) the addition stays an IMAD on the FMA pipe.
__device__ __forceinline__ uint32_t fma_add_rt(uint32_t a, uint32_t b, uint32_t one)
{
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t fma_2a_plus_b(uint32_t a, uint32_t b)
{
    uint32_t d;
    asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t tab_addr(uint32_t lane_base, uint32_t byte)
{
    return byte * 128u + lane_base;
}

__device__ __forceinline__ uint4 ldg_stream(const uint4 *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// ------------------------------------------------------------------------
// synthetic content: word i (absolute u64 index in the slot) = mix64(seed+(i+1)*G)
// ------------------------------------------------------------------------
__global__ void k_synth_fill(uint64_t *dst, uint64_t word0, uint64_t nwords, uint64_t seed)
{
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x * 2;
    for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < nwords; i += stride) {
        uint64_t a = mix64(seed + (word0 + i + 1) * MK_GOLDEN64);
        if (i + 1 < nwords) {
            uint64_t b = mix64(seed + (word0 + i + 2) * MK_GOLDEN64);
            ulonglong2 v;
            v.x = a;
            v.y = b;
            *reinterpret_cast<ulonglong2 *>(dst + i) = v; // dst 16-byte aligned, i even
        } else {
            dst[i] = a;
        }
    }
}

// ------------------------------------------------------------------------
// K0: CRC-32 of the context stream.
//
// The stream is a list of extents.  With pure(M) = M(x)*x^32 mod P (init 0, no
// xorout) the CRC is GF(2)-linear:
//     pure(stream) = XOR over pieces  pure(piece) * x^(8*bytes_after_piece)
// so every piece is independent and the result is one 32-bit XOR reduction.
// A warp owns a piece (<= PIECE bytes of one extent) and walks it in 512-byte
// rows; lane l keeps four Horner chains, one per 32-bit component of its
// coalesced uint4, chain step  acc = acc*x^4096 mod P  ^ word  done with four
// byte-indexed table lookups.  The tables are replicated per lane in shared
// memory ([4][256][32] words = 128 KiB) so every lookup is bank-conflict free.
//
// When the submit also ran the scan, the scan has left the CRC of every 128-byte
// arena row in `part` (k_roll_scan<.., REP > 0>), and K0 reads those instead of the
// bytes: a granule value h with pure(row) = h*x^32 behaves exactly like a word
// whose last byte is the row's last byte, so the same chains, steps and fold work
// on granules, with constants for a 128-byte element instead of a 4-byte one
// (a warp row = 128 granules = 16 KiB of data).  A first or last granule only
// partly inside its piece is computed from the arena bytes.
// ------------------------------------------------------------------------
struct CrcExtent {
    uint64_t off;    // byte offset in the slot, multiple of 16
    uint64_t len;
    uint64_t suffix; // stream bytes after this extent
};

constexpr uint32_t CRC_PIECE = 256u * 1024u; // bytes per warp-piece (multiple of 512)
constexpr int CRC_THREADS = 1024;
constexpr size_t CRC_SMEM = 4u * 256u * 32u * sizeof(uint32_t);

constexpr uint32_t CRC_GRANULE = 128; // bytes per partial CRC the scan writes (one arena row)

struct CrcConsts {
    uint32_t mulk[4][256];   // byte tables for a -> a*x^4096 mod P
    uint32_t lane_c[128];    // x^(32 + 8*(508-16l-4c)) for (l,c)
    uint32_t xe[4][256];     // x^(v << 8t): x^E = product over the bytes t of E of xe[t][byte t]
    uint32_t mulk_g[4][256]; // granule chains: a -> a*x^(8*128*128) mod P
    uint32_t lane_g[128];    //   x^(32 + 8*128*(127-4l-c)) for (l,c)
    uint32_t word_g[32];     // x^(32*(31-j)): word j of a granule -> its granule value
    uint32_t mulk_w[4][256]; // the scan's per-row chains: a -> a*x^32 mod P
};

__device__ __forceinline__ uint32_t crc_step(uint32_t T, uint32_t a, uint32_t w)
{
    // T = shared address of table 0 + lane*4; table t, value v at T + t*32768 + v*128
    const uint32_t r0 = lds_u32(tab_addr(T, byte_of<0>(a)));
    const uint32_t r1 = lds_u32(tab_addr(T + 32768u, byte_of<1>(a)));
    const uint32_t r2 = lds_u32(tab_addr(T + 65536u, byte_of<2>(a)));
    const uint32_t r3 = lds_u32(tab_addr(T + 98304u, byte_of<3>(a)));
    return r0 ^ r1 ^ r2 ^ r3 ^ w;
}

__global__ void __launch_bounds__(CRC_THREADS, 1)
k_crc32_extents(const uint8_t *__restrict__ arena, const CrcExtent *__restrict__ ext,
                const uint32_t *__restrict__ piece_base, uint32_t n_ext, uint32_t n_pieces,
                const CrcConsts *__restrict__ cst, uint32_t *__restrict__ ext_pure /* [n_ext], zeroed: pure(extent) */,
                uint32_t *__restrict__ acc_out /* pure(stream) accumulator */,
                const uint32_t *__restrict__ part /* granule values of the scan, or null: read the bytes */)
{
    extern __shared__ uint32_t s_tab[];
    const uint32_t *const mulk = part ? &cst->mulk_g[0][0] : &cst->mulk[0][0];
    const uint32_t *const lane_c = part ? cst->lane_g : cst->lane_c;
    for (uint32_t i = threadIdx.x; i < 4u * 256u * 32u; i += blockDim.x)
        s_tab[i] = mulk[i >> 5];
    __syncthreads();

    const uint32_t lane = threadIdx.x & 31;
    const uint32_t T = smem_u32(s_tab) + lane * 4u;
    const uint32_t warps_per_cta = blockDim.x >> 5;
    const uint32_t total_warps = gridDim.x * warps_per_cta;
    uint32_t warp_acc = 0;
    for (uint32_t piece = blockIdx.x * warps_per_cta + (threadIdx.x >> 5); piece < n_pieces;
         piece += total_warps) {
        // extent lookup: largest e with piece_base[e] <= piece
        uint32_t lo = 0, hi = n_ext;
        while (hi - lo > 1) {
            uint32_t mid = (lo + hi) >> 1;
            if (__ldg(piece_base + mid) <= piece)
                lo = mid;
            else
                hi = mid;
        }
        const CrcExtent e = ext[lo];
        const uint64_t start = (uint64_t)(piece - __ldg(piece_base + lo)) * CRC_PIECE;
        const uint64_t left = e.len - start;
        const uint32_t valid = left < CRC_PIECE ? (uint32_t)left : CRC_PIECE;
        uint32_t rows, pad; // chain rows of the piece; zero bytes after the piece to the end of the last row
        uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        if (part) {
            // granules g = 0.. of the run that starts at S (512-aligned: lane l loads granules 4l..4l+3 of a row as one
            // uint4).  Granules before gA and after gE lie outside the piece and count as zero.  When gA or gE is only
            // partly inside it, lanes 0-7 compute gA and lanes 8-15 gE from the bytes, the zero-extended word j of a
            // granule contributing word*x^(32*(31-j)).  Leading zero bytes do not change a pure CRC, trailing ones are
            // `pad`.
            const uint64_t A = e.off + start, Z = A + valid, S = A & ~511ull;
            const uint32_t gA = (uint32_t)((A - S) / CRC_GRANULE), gE = (uint32_t)((Z - 1 - S) / CRC_GRANULE);
            const bool cutA = A % CRC_GRANULE != 0, cutE = Z % CRC_GRANULE != 0;
            uint32_t hg = 0;
            if ((cutA || cutE) && lane < 16) {
                const uint64_t q = S + (uint64_t)(lane < 8 ? gA : gE) * CRC_GRANULE + (lane & 7u) * 16u;
                uint4 w = make_uint4(0, 0, 0, 0);
                if (q >= A && q < Z) {
                    w = ldg_stream(reinterpret_cast<const uint4 *>(arena + q));
                    const uint64_t nb = Z - q;
                    if (nb < 16) {
                        uint32_t m[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            int32_t bytes = (int32_t)nb - 4 * k;
                            m[k] = bytes >= 4 ? 0xFFFFFFFFu : (bytes <= 0 ? 0u : (0xFFFFFFFFu >> (32 - 8 * bytes)));
                        }
                        w.x &= m[0]; w.y &= m[1]; w.z &= m[2]; w.w &= m[3];
                    }
                }
                const uint32_t *wg = cst->word_g + (lane & 7u) * 4u;
                hg = crc_mulmod(w.x, wg[0]) ^ crc_mulmod(w.y, wg[1]) ^ crc_mulmod(w.z, wg[2]) ^ crc_mulmod(w.w, wg[3]);
            }
#pragma unroll
            for (int s = 1; s < 8; s <<= 1)
                hg ^= __shfl_xor_sync(0xFFFFFFFFu, hg, s);
            const uint32_t hA = __shfl_sync(0xFFFFFFFFu, hg, 0), hE = __shfl_sync(0xFFFFFFFFu, hg, 8);
            rows = (gE + 128u) / 128u;
            pad = (uint32_t)(S + (uint64_t)rows * 128u * CRC_GRANULE - Z);
            const uint32_t *pg = part + S / CRC_GRANULE;
            for (uint32_t r = 0; r < rows; ++r) {
                const uint32_t i0 = r * 128u + lane * 4u;
                uint4 p = make_uint4(0, 0, 0, 0);
                if (i0 <= gE)
                    p = ldg_stream(reinterpret_cast<const uint4 *>(pg + i0));
                uint32_t v[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint32_t i = i0 + k;
                    v[k] = (i == gA && cutA) ? hA : (i == gE && cutE) ? hE : (i < gA || i > gE) ? 0u : v[k];
                }
                a0 = crc_step(T, a0, v[0]); a1 = crc_step(T, a1, v[1]); a2 = crc_step(T, a2, v[2]); a3 = crc_step(T, a3, v[3]);
            }
        } else {
            rows = (valid + 511u) >> 9;
            pad = rows * 512u - valid;
            const uint8_t *base = arena + e.off + start + lane * 16u;
            uint32_t r = 0;
            // full rows, 4 loads in flight per lane
            const uint32_t full_rows = valid >> 9;
            for (; r + 4 <= full_rows; r += 4) {
                uint4 w0 = ldg_stream(reinterpret_cast<const uint4 *>(base + (size_t)r * 512));
                uint4 w1 = ldg_stream(reinterpret_cast<const uint4 *>(base + (size_t)(r + 1) * 512));
                uint4 w2 = ldg_stream(reinterpret_cast<const uint4 *>(base + (size_t)(r + 2) * 512));
                uint4 w3 = ldg_stream(reinterpret_cast<const uint4 *>(base + (size_t)(r + 3) * 512));
                a0 = crc_step(T, a0, w0.x); a1 = crc_step(T, a1, w0.y); a2 = crc_step(T, a2, w0.z); a3 = crc_step(T, a3, w0.w);
                a0 = crc_step(T, a0, w1.x); a1 = crc_step(T, a1, w1.y); a2 = crc_step(T, a2, w1.z); a3 = crc_step(T, a3, w1.w);
                a0 = crc_step(T, a0, w2.x); a1 = crc_step(T, a1, w2.y); a2 = crc_step(T, a2, w2.z); a3 = crc_step(T, a3, w2.w);
                a0 = crc_step(T, a0, w3.x); a1 = crc_step(T, a1, w3.y); a2 = crc_step(T, a2, w3.z); a3 = crc_step(T, a3, w3.w);
            }
            for (; r < rows; ++r) {
                // remaining rows; the last one may be partial: bytes past `valid` count as zero
                uint4 w = make_uint4(0, 0, 0, 0);
                const int32_t nb = (int32_t)valid - (int32_t)(r * 512u + lane * 16u);
                if (nb > 0) {
                    w = ldg_stream(reinterpret_cast<const uint4 *>(base + (size_t)r * 512));
                    if (nb < 16) {
                        uint32_t m[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            int32_t bytes = nb - 4 * k;
                            m[k] = bytes >= 4 ? 0xFFFFFFFFu : (bytes <= 0 ? 0u : (0xFFFFFFFFu >> (32 - 8 * bytes)));
                        }
                        w.x &= m[0]; w.y &= m[1]; w.z &= m[2]; w.w &= m[3];
                    }
                }
                a0 = crc_step(T, a0, w.x); a1 = crc_step(T, a1, w.y); a2 = crc_step(T, a2, w.z); a3 = crc_step(T, a3, w.w);
            }
        }
        // fold the 128 chains of the warp: chain (l,c) ends 8*(508-16l-4c) bits (granules: 8*128*(127-4l-c)) before
        // the row end
        uint32_t c = crc_mulmod(a0, lane_c[lane * 4 + 0]) ^ crc_mulmod(a1, lane_c[lane * 4 + 1]) ^
                     crc_mulmod(a2, lane_c[lane * 4 + 2]) ^ crc_mulmod(a3, lane_c[lane * 4 + 3]);
#pragma unroll
        for (int s = 16; s; s >>= 1)
            c ^= __shfl_xor_sync(0xFFFFFFFFu, c, s);
        // c = pure(piece || zero padding to the row end).  Shift it to its place in
        // the stream: x^(8*(bytes after the piece) - 8*pad), exponent mod 2^32-1
        // (x is primitive mod P, so x^(2^32-1) = 1).
        // first to the END OF THE EXTENT: pure(extent) is kept per extent so that the host can remember it per file and
        // fold unchanged files into a later build's cacheID without sending their bytes (mksnap_crc_add) ...
        const uint32_t M = 0xFFFFFFFFu;
        const uint64_t after = left - valid;
        uint32_t E = (uint32_t)(((after % M) * 8ull) % M);
        E = (uint32_t)(((uint64_t)E + M - 8ull * pad) % M);
        // ... and on to its place in the stream: x^(8 * bytes after the extent) further.  Lanes 0-3 build x^E and lanes
        // 4-7 x^(E + 8*suffix), each lane one byte-table factor, two rounds of products, then one multiplication by c
        const uint32_t E2 = (uint32_t)(((uint64_t)E + ((e.suffix % M) * 8ull) % M) % M);
        const uint32_t ex = lane < 4 ? E : E2;
        uint32_t f = lane < 8 ? cst->xe[lane & 3][(ex >> (8 * (lane & 3))) & 255u] : 0x80000000u;
        f = crc_mulmod(f, __shfl_xor_sync(0xFFFFFFFFu, f, 1));
        f = crc_mulmod(f, __shfl_xor_sync(0xFFFFFFFFu, f, 2));
        const uint32_t g = crc_mulmod(c, f);
        const uint32_t v = __shfl_sync(0xFFFFFFFFu, g, 0);
        if (lane == 0 && v)
            atomicXor(ext_pure + lo, v);
        warp_acc ^= __shfl_sync(0xFFFFFFFFu, g, 4);
    }
    if (lane == 0 && warp_acc)
        atomicXor(acc_out, warp_acc);
}

// ------------------------------------------------------------------------
// K0f: fold extent values into many CRC streams (plan-level cacheIDs, mksnap_crc_fold).
// One thread per use: its value -- pure(extent) of this session, or an immediate value -- times x^(8*suffix), XORed
// into the use's stream.  x^E comes from the xe byte tables as in K0: one lookup per byte of E, three products.
// Lanes of a warp that hit the same stream XOR-reduce first (the host emits uses grouped by stream), so a warp issues
// one atomic per distinct stream.  Latency-bound and small: 24 bytes read per use.
// ------------------------------------------------------------------------
struct CrcUse { // layout of mksnap_crc_use
    uint64_t suffix;
    uint64_t src;
    uint32_t stream;
    uint32_t flags; // 1: src holds the value itself
};

constexpr int FOLD_THREADS = 256;

__global__ void __launch_bounds__(FOLD_THREADS)
k_crc_fold(const CrcUse *__restrict__ uses, uint32_t n, const uint32_t *__restrict__ ext_pure,
           const CrcConsts *__restrict__ cst, uint32_t *__restrict__ stream_pure)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t stream = 0xFFFFFFFFu, v = 0; // past the end: a stream no use can name, value 0
    if (i < n) {
        const CrcUse u = uses[i];
        const uint32_t M = 0xFFFFFFFFu; // x^(2^32-1) = 1
        const uint32_t E = (uint32_t)(((u.suffix % M) * 8ull) % M);
        const uint32_t val = (u.flags & 1u) ? (uint32_t)u.src : __ldg(ext_pure + u.src);
        const uint32_t f = crc_mulmod(crc_mulmod(__ldg(&cst->xe[0][E & 255u]), __ldg(&cst->xe[1][(E >> 8) & 255u])),
                                      crc_mulmod(__ldg(&cst->xe[2][(E >> 16) & 255u]), __ldg(&cst->xe[3][E >> 24])));
        v = crc_mulmod(val, f);
        stream = u.stream;
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, stream);
    const uint32_t x = __reduce_xor_sync(peers, v);
    if (i < n && (threadIdx.x & 31u) == (uint32_t)(__ffs(peers) - 1) && x)
        atomicXor(stream_pure + stream, x);
}

// ------------------------------------------------------------------------
// K1: Roll-32 candidate scan (DESIGN.md section 3).
//   u_i = little-endian 32-bit word that ENDS at byte i;  h_i = h_{i-1}*M + u_i (mod 2^32), M = 2*odd, so
//   h_i = sum_{k<32} u_{i-k} * M^k: a 32-position (35-byte) window and NO table.
//   candidate iff the top `bits` bits of h_i are all ones (h_i >= 2^32 - 2^(32-bits)).
// Per byte that is one funnel shift (ALU pipe; none for the aligned position of each word), one IMAD (FMA pipe) and
// half a VIMNMX3 for the test -- 2.25 issue slots per byte and not one shared-memory lookup, so the kernel is bounded
// by HBM and nothing else.  (The round-1/2 kernel hashed with a 256-entry Gear table: PRMT + LDS + IMAD per byte kept
// the LSU at 72 % and issue at 79 % of their peaks, and it stalled at 73 % of the HBM peak.)
//
// Data path: the arena is viewed as a [rows][128 B] tensor.  A producer warp streams tiles of TILE_WARPS*32 rows PLUS
// the row in front of them (one cp.async.bulk.tensor.2d, SWIZZLE_128B, box = ROWS+1 rows starting at row0-1; the row
// before the arena is out of bounds and arrives as zeros) through a STAGES-deep full/empty mbarrier ring.
// Each consumer thread owns ONE 128-byte row.  It warms the hash up over the last 32 positions of the row above it
// (three LDS.128 from that row: after 32 positions the state no longer depends on where it started), then
// rolls it over its own 128 bytes, eight conflict-free LDS.128 (chunk c of row r sits at c ^ (r & 7)).  No carry
// between lanes, no block-level synchronisation: a thread needs nothing but its two rows.
// Candidates are rare (2^-12 per byte): they are collected in per-lane register bitmasks (lane l's mask = its own
// row), compacted in position order with one warp scan, and bump-allocated into the pool: one TileRec per 4 KiB warp
// region, pool entry = pos_in_region | strict<<31.
// ------------------------------------------------------------------------
constexpr uint32_t SCAN_TILE = 4096; // bytes per TileRec region (= one warp x 32 rows x 128 B)
constexpr uint32_t SCAN_POOL_BLOCK = 256; // pool entries a warp reserves per global atomic
constexpr uint32_t ROLL_MULT = 0x9E3779BAu; // M = 2 * 0x4F1BBCDD (oracle/mkoracle.c ROLL_MULT)

struct TileRec {
    uint32_t base;  // first pool entry of this region
    uint32_t count; // candidates in this region
};

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    do {
        // the suspend-time hint lets the hardware park the warp instead of re-issuing the probe: a spinning warp
        // steals issue slots from the warps that have data
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(bar), "r"(parity), "r"(200000u)
                     : "memory");
    } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void *tmap, int32_t x, int32_t y, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(tmap), "r"(x), "r"(y), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ uint4 lds_u128(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}

// h*M + u on the FMA pipe
__device__ __forceinline__ uint32_t roll_step(uint32_t h, uint32_t u)
{
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(h), "n"(ROLL_MULT), "r"(u));
    return d;
}
// the four positions that end in the bytes of `w` (`p` = the word before it), every intermediate state kept
#define MK_ROLL_WORD(p, w, k0)                                      \
    {                                                               \
        h = roll_step(h, __funnelshift_r((p), (w), 8));             \
        hv[(k0)] = h;                                               \
        h = roll_step(h, __funnelshift_r((p), (w), 16));            \
        hv[(k0) + 1] = h;                                           \
        h = roll_step(h, __funnelshift_r((p), (w), 24));            \
        hv[(k0) + 2] = h;                                           \
        h = roll_step(h, (w));                                      \
        hv[(k0) + 3] = h;                                           \
    }
// the same without keeping the states (warm-up over the row above)
#define MK_ROLL_WARM(p, w)                                          \
    {                                                               \
        h = roll_step(h, __funnelshift_r((p), (w), 8));             \
        h = roll_step(h, __funnelshift_r((p), (w), 16));            \
        h = roll_step(h, __funnelshift_r((p), (w), 24));            \
        h = roll_step(h, (w));                                      \
    }

// A tile is TILE_WARPS warps x 32 rows x 128 B plus the row above it (one TMA op); GROUPS groups of TILE_WARPS consumer
// warps take the CTA's tiles round-robin, so the pipeline depth (STAGES) is independent of how many warps hide latency.
// With G groups consuming, STAGES - G stages are in flight from HBM; the chip needs ~45 KiB per SM in flight to cover
// the HBM bandwidth x ~1 us of loaded latency.  With no table in shared memory all 227 KiB hold stages.
// Shared-memory plan (dynamic region, 1 KiB aligned): STAGES stages of PITCH bytes (box rounded up to whole swizzle
// atoms), then the mbarriers.
// The CRC variant (REP > 0) also keeps the slicing-by-4 tables of the per-row CRC chain after the stages, REP copies of
// each entry: lane l reads copy l % REP.
template <int SCAN_GROUPS, int TW = 6, int ST = 8, int REP = 0> struct ScanCfg {
    static constexpr uint32_t STAGES = ST;
    static constexpr uint32_t TILE_WARPS = TW;
    static constexpr uint32_t GROUPS = SCAN_GROUPS;
    static constexpr uint32_t ROWS = TILE_WARPS * 32;
    static constexpr uint32_t BOX_ROWS = ROWS + 1;                 // the row above the tile travels with it
    static constexpr uint32_t TILE_BYTES = BOX_ROWS * 128;         // bytes one TMA op delivers
    static constexpr uint32_t PITCH = (TILE_BYTES + 1023) / 1024 * 1024;
    static constexpr uint32_t CONSUMER_WARPS = SCAN_GROUPS * TILE_WARPS;
    static constexpr uint32_t THREADS = (CONSUMER_WARPS + 1) * 32;
    static constexpr uint32_t TAB_OFF = STAGES * PITCH;
    static constexpr uint32_t TAB_BYTES = 4u * 256u * REP * 4u;
    static constexpr uint32_t BARS_OFF = TAB_OFF + TAB_BYTES;
    static constexpr uint32_t SMEM = BARS_OFF + 2 * STAGES * 8 + 1024; // dynamic bytes to request, alignment slack included
    static_assert(BOX_ROWS <= 256, "one TMA box");
    // Each stage must always be consumed by the same group.  Otherwise a group can reach a stage while its full barrier
    // is still two phases behind, and the parity wait, which cannot tell phase k from phase k-2, passes on stale data.
    static_assert(STAGES % GROUPS == 0, "groups must divide stages");
    static_assert(SMEM <= 227 * 1024, "exceeds the 227 KiB per-CTA limit");
};

// a*x^32 ^ w with REP-fold replicated byte tables (table t, value v, copy k at word (t*256 + v)*REP + k)
template <int REP> __device__ __forceinline__ uint32_t crc_step_rep(uint32_t T, uint32_t a, uint32_t w)
{
    const uint32_t r0 = lds_u32(byte_of<0>(a) * (4u * REP) + T);
    const uint32_t r1 = lds_u32(byte_of<1>(a) * (4u * REP) + (T + 1024u * REP));
    const uint32_t r2 = lds_u32(byte_of<2>(a) * (4u * REP) + (T + 2048u * REP));
    const uint32_t r3 = lds_u32(byte_of<3>(a) * (4u * REP) + (T + 3072u * REP));
    return r0 ^ r1 ^ r2 ^ r3 ^ w;
}

// REP > 0: the CRC variant.  Besides the candidates, every consumer thread runs a CRC chain h = h*x^32 ^ word over the
// 32 words of its row as they pass through the roll, and writes h (pure(row) = h*x^32) to part[global row]: K0 then
// takes whole rows of an extent from `part` instead of reading the arena a second time.
template <int SCAN_GROUPS, int TW, int ST, int REP = 0>
__global__ void __launch_bounds__((SCAN_GROUPS * TW + 1) * 32, 1)
k_roll_scan(const __grid_constant__ CUtensorMap tm_main, uint32_t n_tiles, uint32_t strict_lim, uint32_t loose_lim,
            TileRec *__restrict__ tiles, uint32_t *__restrict__ pool, uint32_t pool_cap,
            uint32_t *__restrict__ pool_count, uint32_t *__restrict__ err_flag,
            const uint32_t *__restrict__ crc_tab /* [4][256] a -> a*x^32 (REP > 0) */, uint32_t *__restrict__ part)
{
    using Cfg = ScanCfg<SCAN_GROUPS, TW, ST, REP>;
    constexpr uint32_t STAGES = Cfg::STAGES;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t s0 = (smem_u32(smem_raw) + 1023u) & ~1023u; // swizzle atoms are 1 KiB: align the stages ourselves
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t bar_full = s0 + Cfg::BARS_OFF, bar_empty = bar_full + STAGES * 8;
    const uint32_t strict_thr = 0u - strict_lim, loose_thr = 0u - loose_lim; // top `bits` bits all ones

    if constexpr (REP > 0) {
        uint32_t *tab = reinterpret_cast<uint32_t *>(smem_raw + (s0 - smem_u32(smem_raw)) + Cfg::TAB_OFF);
        for (uint32_t i = threadIdx.x; i < 1024u * REP; i += blockDim.x)
            tab[i] = __ldg(crc_tab + i / REP);
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < (int)STAGES; ++s) {
            mbar_init(bar_full + s * 8, 1);
            mbar_init(bar_empty + s * 8, Cfg::TILE_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == Cfg::CONSUMER_WARPS) {
        // ------------------------- TMA producer -------------------------
        if (lane == 0) {
            uint32_t it = 0;
            for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
                const uint32_t s = it % STAGES;
                if (it >= STAGES)
                    mbar_wait(bar_empty + s * 8, ((it / STAGES) & 1u) ^ 1u);
                mbar_arrive_expect_tx(bar_full + s * 8, Cfg::TILE_BYTES);
                tma_load_2d(s0 + s * Cfg::PITCH, &tm_main, 0, (int32_t)(tile * Cfg::ROWS) - 1, bar_full + s * 8);
            }
        }
        return;
    }

    // ----------------------------- consumers -----------------------------
    const uint32_t group = warp / Cfg::TILE_WARPS, wt = warp % Cfg::TILE_WARPS; // wt = warp within the tile
    const uint32_t row = wt * 32u + lane;   // row of the tile; it sits at box row `row + 1`, the row above it at `row`
    const uint32_t ra_off = (row + 1u) * 128u, swz = ((row + 1u) & 7u) << 4;
    const uint32_t rp_off = row * 128u, swp = (row & 7u) << 4;
    const uint32_t T = s0 + Cfg::TAB_OFF + (REP > 0 ? lane % REP : 0u) * 4u; // this lane's table copy
    uint32_t blk_next = 0, blk_end = 0; // this warp's private slice of the pool (warp-uniform)
    // CTA-local tile sequence it = 0,1,2,... (global tile = blockIdx.x + it*gridDim.x); group g takes it = g (mod GROUPS)
    for (uint32_t it = group;; it += SCAN_GROUPS) {
        const uint64_t tile64 = (uint64_t)blockIdx.x + (uint64_t)it * gridDim.x;
        if (tile64 >= n_tiles)
            break;
        const uint32_t tile = (uint32_t)tile64;
        const uint32_t s = it % STAGES;
        const uint32_t sb = s0 + s * Cfg::PITCH;
        mbar_wait(bar_full + s * 8, (it / STAGES) & 1u);

        // warm-up: the 32 positions that end in bytes 96..127 of the row above (their words reach back to byte 93)
        uint32_t h = 0, pw;
        {
            const uint32_t rp = sb + rp_off;
            // bytes 92..95: the whole 16-byte chunk is read (a 4-byte read of its last word is a 4-way bank conflict:
            // the 32 rows of a warp put that word in only 8 banks)
            const uint32_t w5 = lds_u128(rp + ((5u << 4) ^ swp)).w;
            const uint4 a = lds_u128(rp + ((6u << 4) ^ swp)), b = lds_u128(rp + ((7u << 4) ^ swp));
            MK_ROLL_WARM(w5, a.x) MK_ROLL_WARM(a.x, a.y) MK_ROLL_WARM(a.y, a.z) MK_ROLL_WARM(a.z, a.w)
            MK_ROLL_WARM(a.w, b.x) MK_ROLL_WARM(b.x, b.y) MK_ROLL_WARM(b.y, b.z) MK_ROLL_WARM(b.z, b.w)
            pw = b.w;
        }

        const uint32_t ra = sb + ra_off;
        uint32_t mL0 = 0, mL1 = 0, mL2 = 0, mL3 = 0; // loose candidates, bit p of the row
        uint32_t mS0 = 0, mS1 = 0, mS2 = 0, mS3 = 0; // strict candidates
        uint32_t hc = 0;                             // CRC chain of the row (REP > 0)
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const uint4 w = lds_u128(ra + ((uint32_t)(c << 4) ^ swz));
            if constexpr (REP > 0) {
                hc = c == 0 ? w.x : crc_step_rep<REP>(T, hc, w.x);
                hc = crc_step_rep<REP>(T, hc, w.y);
                hc = crc_step_rep<REP>(T, hc, w.z);
                hc = crc_step_rep<REP>(T, hc, w.w);
            }
            uint32_t hv[16];
            MK_ROLL_WORD(pw, w.x, 0) MK_ROLL_WORD(w.x, w.y, 4) MK_ROLL_WORD(w.y, w.z, 8) MK_ROLL_WORD(w.z, w.w, 12)
            pw = w.w;
            uint32_t m = hv[0];
#pragma unroll
            for (int i = 1; i < 16; ++i)
                m = max(m, hv[i]);
            // ~0.4 % of lane-chunks hold a candidate, so ~12 % of the time some lane of the warp does: the vote makes
            // the branch warp-uniform (no BSSY/BSYNC pair around it on the 88 % path)
            if (__any_sync(0xFFFFFFFFu, m >= loose_thr) && m >= loose_thr) {
                uint32_t bl = 0, bs = 0;
#pragma unroll
                for (int i = 0; i < 16; ++i)
                    if (hv[i] >= loose_thr)
                        bl |= 1u << i;
                if (m >= strict_thr) { // 1/16 of those
#pragma unroll
                    for (int i = 0; i < 16; ++i)
                        if (hv[i] >= strict_thr)
                            bs |= 1u << i;
                }
                const uint32_t sh = (c & 1) * 16;
                if ((c >> 1) == 0) { mL0 |= bl << sh; mS0 |= bs << sh; }
                if ((c >> 1) == 1) { mL1 |= bl << sh; mS1 |= bs << sh; }
                if ((c >> 1) == 2) { mL2 |= bl << sh; mS2 |= bs << sh; }
                if ((c >> 1) == 3) { mL3 |= bl << sh; mS3 |= bs << sh; }
            }
        }
        // the stage is consumed: hand it back to the producer before the tail work
        __syncwarp();
        if (lane == 0)
            mbar_arrive(bar_empty + s * 8);
        if constexpr (REP > 0)
            part[(size_t)tile * Cfg::ROWS + row] = hc;

        // ordered compaction: lane l's candidates precede lane l+1's
        const uint32_t cnt = __popc(mL0) + __popc(mL1) + __popc(mL2) + __popc(mL3);
        // exclusive prefix over lanes.  Nearly always every lane holds 0 or 1 candidate: two ballots do it.
        const uint32_t b1 = __ballot_sync(0xFFFFFFFFu, cnt != 0);
        const uint32_t b2 = __ballot_sync(0xFFFFFFFFu, cnt > 1);
        uint32_t incl, total;
        if (b2 == 0) {
            incl = __popc(b1 & (0xFFFFFFFFu >> (31 - lane)));
            total = __popc(b1);
        } else {
            incl = cnt;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, sft);
                if (lane >= sft)
                    incl += v;
            }
            total = __shfl_sync(0xFFFFFFFFu, incl, 31);
        }
        if (total > blk_end - blk_next) { // refill: rare (every ~SCAN_POOL_BLOCK candidates)
            uint32_t nb = 0;
            if (lane == 0) {
                const uint32_t want = total > SCAN_POOL_BLOCK ? total : SCAN_POOL_BLOCK;
                nb = atomicAdd(pool_count, want);
                if (nb + want > pool_cap || nb + want < nb) {
                    atomicExch(err_flag, 1u);
                    nb = 0xFFFFFFFFu;
                }
            }
            nb = __shfl_sync(0xFFFFFFFFu, nb, 0);
            blk_next = nb;
            blk_end = nb == 0xFFFFFFFFu ? nb : nb + (total > SCAN_POOL_BLOCK ? total : SCAN_POOL_BLOCK);
        }
        const uint32_t base = blk_next;
        if (base != 0xFFFFFFFFu)
            blk_next += total;
        if (lane == 0) {
            TileRec tr;
            tr.base = base;
            tr.count = base == 0xFFFFFFFFu ? 0u : total;
            tiles[(size_t)tile * Cfg::TILE_WARPS + wt] = tr;
        }
        if (total) {
            if (base != 0xFFFFFFFFu && cnt) {
                uint32_t o = base + incl - cnt;
                const uint32_t p0 = lane * 128u;
#define MK_EMIT(ML, MS, WORD)                                              \
    {                                                                      \
        uint32_t bits = (ML);                                              \
        while (bits) {                                                     \
            const uint32_t b = __ffs(bits) - 1;                            \
            bits &= bits - 1;                                              \
            pool[o++] = (p0 + (WORD) * 32u + b) | ((((MS) >> b) & 1u) << 31); \
        }                                                                  \
    }
                MK_EMIT(mL0, mS0, 0) MK_EMIT(mL1, mS1, 1) MK_EMIT(mL2, mS2, 2) MK_EMIT(mL3, mS3, 3)
#undef MK_EMIT
            }
        }
    }
}

// ------------------------------------------------------------------------
// K1b: cut selection.  One thread per file walks the ordered candidates of the
// tiles its file covers.  pass 0 counts chunks, pass 1 writes (start,len).
// ------------------------------------------------------------------------
struct CdcFile {
    uint64_t off;
    uint64_t len;
    uint64_t scratch; // big files: first slot of this file's cut list in the scratch buffer (len/min + 2 slots)
    uint32_t more_after; // bytes of this file that follow in LATER submits (saturated); 0 = the file ends in this piece
    uint32_t cont;       // 1 = continues the open file of the previous submit (k_carry_in prepended the open chunk)
};

struct CdcParamsDev {
    uint32_t min_size, normal_size, max_size, strict_lim, loose_lim;
};

struct SessionCounters {
    unsigned long long n_chunks;   // chunks appended so far in this session
    unsigned long long n_files;
    unsigned long long cdc_bytes;
    unsigned long long n_streams;
    uint32_t batch_chunks;         // chunks of the batch being processed
    uint32_t err;                  // 1 = candidate pool overflow, 2 = chunk table overflow
    uint32_t crc_acc;              // XOR accumulator of K0
    uint32_t work;                 // work-stealing counter of K2
    unsigned long long carry_off;  // open chunk of a file that continues in the next submit: slot offset of its first byte
    unsigned long long carry_len;  //   and its length (< max_size); consumed by k_carry_in of the next submit
    uint32_t len_bins[64];         // K2 work order: chunks of the batch per length class (2 KiB classes)
    uint32_t len_cursor[64];       //   slots handed out per class while the order is written
};
constexpr uint32_t LEN_CLASSES = 64;
constexpr uint32_t LEN_CLASS_SHIFT = 11;

// One application of the cut rule (DESIGN.md section 3) from `prev`, reading tile records and candidates from
// global memory.
// `more_after` > 0: the file continues in a later submit, `end` is only the end of this PIECE.  The rule is then
// applied to the whole file (rem counts the bytes still to come); when it cannot be decided from the bytes at hand --
// no qualifying candidate before `end` and the forced cut / file end lies beyond it -- CUT_OPEN is returned and the
// open chunk [prev, end) is carried into the next submit (k_carry_in).
constexpr uint64_t CUT_OPEN = ~0ull;
__device__ __forceinline__ uint64_t select_one_cut(uint64_t prev, uint64_t end, uint32_t more_after, const CdcParamsDev &prm,
                                                   const TileRec *__restrict__ tiles, const uint32_t *__restrict__ pool)
{
    const uint64_t rem = end - prev + more_after;
    if (rem <= prm.min_size)
        return more_after ? CUT_OPEN : end;
    const uint64_t limit_end = prev + (rem < prm.max_size ? rem : prm.max_size); // may lie beyond `end`
    const uint64_t scan_end = limit_end < end ? limit_end : end;
    const uint64_t lo = prev + prm.min_size - 1;
    const uint64_t normal_pos = prev + prm.normal_size - 1; // pos >= this: loose accepted
    for (uint64_t t = lo / SCAN_TILE; t * SCAN_TILE < scan_end; ++t) {
        const TileRec tr = tiles[t];
        const uint64_t tb = t * SCAN_TILE;
        for (uint32_t j = 0; j < tr.count; ++j) {
            const uint32_t ent = __ldg(pool + tr.base + j);
            const uint64_t pos = tb + (ent & 0x7FFFFFFFu);
            if (pos < lo)
                continue;
            if (pos >= scan_end)
                return limit_end <= end ? limit_end : CUT_OPEN;
            if (pos >= normal_pos || (ent >> 31))
                return pos + 1;
        }
    }
    return limit_end <= end ? limit_end : CUT_OPEN;
}

constexpr uint64_t SELECT_BIG_FILE = 4ull << 20; // files at least this long get a CTA and shared-memory staging

template <int PASS>
__global__ void __launch_bounds__(128)
k_select_cuts(const CdcFile *__restrict__ files, uint32_t n_files, CdcParamsDev prm,
              const TileRec *__restrict__ tiles, const uint32_t *__restrict__ pool,
              uint32_t *__restrict__ counts, const uint32_t *__restrict__ bases,
              SessionCounters *__restrict__ sc, uint64_t max_chunks, uint64_t stream_base,
              uint64_t *__restrict__ chunk_start, uint64_t *__restrict__ chunk_len,
              uint64_t *__restrict__ chunk_end_out)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_files)
        return;
    if (PASS == 1 && sc->err)
        return;
    const CdcFile fl = files[f];
    if (fl.len >= SELECT_BIG_FILE)
        return; // k_select_cuts_big owns this file
    uint64_t prev = fl.off;
    const uint64_t end = fl.off + fl.len;
    uint64_t out = 0;
    if (PASS == 1)
        out = sc->n_chunks + bases[f];
    uint32_t n = 0;
    if (fl.more_after == 0) { // the common case, kept free of the continuation logic (literal 0: the compiler drops it)
        while (prev < end) {
            const uint64_t cut = select_one_cut(prev, end, 0u, prm, tiles, pool);
            if (PASS == 1) {
                if (out + n < max_chunks) {
                    chunk_start[out + n] = prev;
                    chunk_len[out + n] = cut - prev;
                    chunk_end_out[out + n] = stream_base + cut;
                }
            }
            ++n;
            prev = cut;
        }
    } else {
        while (prev < end) {
            const uint64_t cut = select_one_cut(prev, end, fl.more_after, prm, tiles, pool);
            if (cut == CUT_OPEN) { // the file continues in the next submit: [prev, end) travels with it
                if (PASS == 1) {
                    sc->carry_off = prev;
                    sc->carry_len = end - prev;
                }
                break;
            }
            if (PASS == 1) {
                if (out + n < max_chunks) {
                    chunk_start[out + n] = prev;
                    chunk_len[out + n] = cut - prev;
                    chunk_end_out[out + n] = stream_base + cut;
                }
            }
            ++n;
            prev = cut;
        }
    }
    if (PASS == 0)
        counts[f] = n;
}

// Long files: a single thread chasing TileRecs and pool entries through L2 pays a dependent L2 round trip per
// candidate, so a file of many chunks would take one thread a long time.  Here a CTA owns the file and works window by window (4 MiB of file):
//   1. stage: tile records -> block scan -> the window's candidates, position ordered, in shared memory;
//   2. next[]: for EVERY candidate q, in parallel, apply the cut rule with prev = pos(q)+1 and record where
//      the chain goes (another candidate, a forced/end position, or "beyond this window");
//   3. chase: one thread follows next[] from the current cut -- one shared-memory load per chunk.
// The rule itself is sel_rule(): identical to select_one_cut() but over the staged list.
// Window size: every window costs two dependent round trips to global memory (tile records, then their candidates)
// plus block barriers, and a CTA works alone on its file, so the cost per window is latency, not bandwidth: 512 threads
// x 16 MiB windows amortise the same latencies over four times the bytes of 128 threads x 4 MiB windows.
constexpr uint32_t SELB_THREADS = 512;
constexpr uint32_t SELB_REGIONS = 4096; // window = 16 MiB of file
constexpr uint32_t SELB_CANDS = 16384;  // candidate capacity of a window (expected 4096 at the default mask)
constexpr size_t SELB_SMEM = (SELB_REGIONS + 1 + 2 * SELB_CANDS) * sizeof(uint32_t); // s_off, s_cand, s_next (dynamic)
constexpr uint32_t NX_CAND = 0u << 30;  // value = candidate index: cut = pos(value) + 1
constexpr uint32_t NX_POS = 1u << 30;   // value = window-relative cut position that is not after a candidate
constexpr uint32_t NX_OUT = 2u << 30;   // the search range leaves the staged window: restage
constexpr uint32_t NX_VAL = (1u << 30) - 1;

struct SelWin {
    const uint32_t *cand; // offset | strict << 31, ascending
    uint32_t ncand;
    uint32_t wend;        // staged candidates cover window offsets [0, wend)
    uint32_t fend;        // file end as a window offset, or 0xFFFFFFFF if beyond the window
};

// first index >= from whose position is >= lo (cand is sorted)
__device__ __forceinline__ uint32_t sel_lower_bound(const SelWin &w, uint32_t from, uint32_t lo)
{
    uint32_t a = from, b = w.ncand;
    while (a < b) {
        const uint32_t m = (a + b) >> 1;
        if ((w.cand[m] & 0x7FFFFFFFu) < lo)
            a = m + 1;
        else
            b = m;
    }
    return a;
}

// cut rule from window offset `prev`; `from` = an index at or before the first candidate that can matter
__device__ __forceinline__ uint32_t sel_rule(const SelWin &w, const CdcParamsDev &prm, uint32_t prev, uint32_t from)
{
    const bool ends = w.fend != 0xFFFFFFFFu;
    const uint32_t rem = ends ? w.fend - prev : 0xFFFFFFFFu;
    if (rem <= prm.min_size)
        return NX_POS | w.fend;
    const uint32_t limit = prev + (rem < prm.max_size ? rem : prm.max_size);
    if (limit > w.wend && !ends)
        return NX_OUT;
    const uint32_t lo = prev + prm.min_size - 1;
    const uint32_t normal_pos = prev + prm.normal_size - 1;
    // candidates are ~4 KiB apart and min is 4 KiB: a short linear probe usually beats the binary search
    uint32_t q = from;
    for (int k = 0; k < 4 && q < w.ncand && (w.cand[q] & 0x7FFFFFFFu) < lo; ++k)
        ++q;
    if (q < w.ncand && (w.cand[q] & 0x7FFFFFFFu) < lo)
        q = sel_lower_bound(w, q, lo);
    for (; q < w.ncand; ++q) {
        const uint32_t ent = w.cand[q];
        const uint32_t pos = ent & 0x7FFFFFFFu;
        if (pos >= limit)
            break;
        if (pos >= normal_pos || (ent >> 31))
            return NX_CAND | q;
    }
    return NX_POS | limit;
}

// Single pass: the cut END offsets (relative to the file start, fit 40 bits -> stored as u64) go to `cuts`
// at files[f].scratch; k_expand_big_cuts turns them into chunk records once the bases are known.
__global__ void __launch_bounds__(SELB_THREADS)
k_select_cuts_big(const CdcFile *__restrict__ files, uint32_t n_files, CdcParamsDev prm,
                  const TileRec *__restrict__ tiles, const uint32_t *__restrict__ pool,
                  uint32_t *__restrict__ counts, uint64_t *__restrict__ cuts, SessionCounters *__restrict__ sc)
{
    constexpr int PASS = 0;
    const uint32_t f = blockIdx.x;
    if (f >= n_files)
        return;
    const CdcFile fl = files[f];
    if (fl.len < SELECT_BIG_FILE)
        return;
    uint64_t *const my_cuts = cuts + fl.scratch;
    extern __shared__ uint32_t selb_smem[];
    uint32_t *const s_off = selb_smem;                      // [SELB_REGIONS + 1] exclusive prefix of candidate counts per region
    uint32_t *const s_cand = s_off + SELB_REGIONS + 1;      // [SELB_CANDS] offset within the window | strict << 31
    uint32_t *const s_next = s_cand + SELB_CANDS;           // [SELB_CANDS] where the chain goes from each candidate
    __shared__ uint32_t s_w[SELB_THREADS / 32];
    __shared__ unsigned long long s_prev, s_open;
    __shared__ uint32_t s_n;

    const uint64_t end = fl.off + fl.len;
    if (threadIdx.x == 0) {
        s_prev = fl.off;
        s_open = CUT_OPEN;
        s_n = 0;
    }
    __syncthreads();
    for (;;) {
        const uint64_t prev0 = s_prev;
        if (prev0 >= end)
            break;
        // ---- 1. stage the window that starts at the region holding `prev` ----
        const uint64_t t0 = prev0 / SCAN_TILE;
        const uint64_t t_last = (end - 1) / SCAN_TILE;
        const uint32_t want = (uint32_t)((t_last - t0 + 1 < SELB_REGIONS) ? (t_last - t0 + 1) : SELB_REGIONS);
        constexpr uint32_t PER = SELB_REGIONS / SELB_THREADS;
        uint32_t cnt[PER], bs[PER], mine = 0;
#pragma unroll
        for (uint32_t k = 0; k < PER; ++k) {
            const uint32_t r = threadIdx.x * PER + k;
            cnt[k] = 0;
            bs[k] = 0;
            if (r < want) {
                const TileRec tr = tiles[t0 + r];
                cnt[k] = tr.count;
                bs[k] = tr.base;
            }
            mine += cnt[k];
        }
        const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t incl = mine;
#pragma unroll
        for (int sft = 1; sft < 32; sft <<= 1) {
            const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, sft);
            if (lane >= sft)
                incl += v;
        }
        if (lane == 31)
            s_w[warp] = incl;
        __syncthreads();
        uint32_t woff = 0;
        for (uint32_t k = 0; k < warp; ++k)
            woff += s_w[k];
        uint32_t o = woff + incl - mine;
#pragma unroll
        for (uint32_t k = 0; k < PER; ++k) {
            const uint32_t r = threadIdx.x * PER + k;
            s_off[r] = o;
            if (o + cnt[k] <= SELB_CANDS) {
                for (uint32_t j = 0; j < cnt[k]; ++j) {
                    const uint32_t ent = __ldg(pool + bs[k] + j);
                    s_cand[o + j] = (r * SCAN_TILE + (ent & 0x7FFFFFFFu)) | (ent & 0x80000000u);
                }
            }
            o += cnt[k];
        }
        if (threadIdx.x == SELB_THREADS - 1)
            s_off[SELB_REGIONS] = o;
        __syncthreads();
        uint32_t nreg = want; // regions whose candidates all fit in s_cand (same value in every thread)
        while (nreg > 0 && s_off[nreg] > SELB_CANDS)
            --nreg;
        const uint64_t wbase = t0 * SCAN_TILE;
        SelWin w;
        w.cand = s_cand;
        w.ncand = s_off[nreg];
        w.wend = nreg * SCAN_TILE;
        // a piece whose file continues (more_after) has no file end in sight: the chain stops with NX_OUT near the
        // piece end and the exact rule (select_one_cut with more_after) finishes from global memory.  Its window ends
        // at the piece end, not at the end of the piece's last region: bytes behind the piece are not the file's, and
        // neither a forced cut nor a candidate there may end a chunk.
        if (fl.more_after && wbase + w.wend > end)
            w.wend = (uint32_t)(end - wbase);
        w.fend = (wbase + w.wend >= end && !fl.more_after) ? (uint32_t)(end - wbase) : 0xFFFFFFFFu;
        // ---- 2. next[] for every candidate, in parallel ----
        for (uint32_t q = threadIdx.x; q < w.ncand; q += SELB_THREADS) {
            const uint32_t prev = (s_cand[q] & 0x7FFFFFFFu) + 1;
            s_next[q] = (w.fend != 0xFFFFFFFFu && prev >= w.fend) ? (NX_POS | w.fend) : sel_rule(w, prm, prev, q + 1);
        }
        __syncthreads();
        // ---- 3. chase the chain ----
        if (threadIdx.x == 0) {
            uint32_t prev = (uint32_t)(prev0 - wbase);
            uint32_t n = s_n;
            bool progressed = false;
            // is `prev` the position right after a staged candidate?
            uint32_t cur = 0xFFFFFFFFu;
            if (prev > 0) {
                const uint32_t q = sel_lower_bound(w, 0, prev - 1);
                if (q < w.ncand && (s_cand[q] & 0x7FFFFFFFu) == prev - 1)
                    cur = q;
            }
            for (;;) {
                if (w.fend != 0xFFFFFFFFu && prev >= w.fend)
                    break;
                const uint32_t nx = cur != 0xFFFFFFFFu ? s_next[cur] : sel_rule(w, prm, prev, 0);
                const uint32_t kind = nx & ~NX_VAL, val = nx & NX_VAL;
                if (kind == NX_OUT)
                    break;
                uint32_t cut;
                if (kind == NX_CAND) {
                    cut = (s_cand[val] & 0x7FFFFFFFu) + 1;
                    cur = val;
                } else {
                    cut = val;
                    cur = 0xFFFFFFFFu;
                }
                my_cuts[n] = wbase + cut - fl.off;
                ++n;
                prev = cut;
                progressed = true;
            }
            uint64_t prev64 = wbase + prev;
            if (!progressed && prev64 < end) {
                // pathologically dense candidates (the staged window is too short for one search range), or the last
                // stretch of a piece whose file continues in the next submit: one cut straight from global memory
                const uint64_t cut = select_one_cut(prev64, end, fl.more_after, prm, tiles, pool);
                if (cut == CUT_OPEN) {
                    s_open = prev64;
                    prev64 = end; // leave the loop; [s_open, end) is the open chunk
                } else {
                    my_cuts[n] = cut - fl.off;
                    ++n;
                    prev64 = cut;
                }
            }
            s_prev = prev64;
            s_n = n;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        counts[f] = s_n;
        if (s_open != CUT_OPEN) {
            sc->carry_off = s_open;
            sc->carry_len = end - s_open;
        }
    }
    (void)PASS;
}

// chunk records of the big files from their cut lists (one CTA per file, coalesced)
__global__ void __launch_bounds__(256)
k_expand_big_cuts(const CdcFile *__restrict__ files, uint32_t n_files, const uint32_t *__restrict__ counts,
                  const uint32_t *__restrict__ bases, const uint64_t *__restrict__ cuts,
                  const SessionCounters *__restrict__ sc, uint64_t max_chunks, uint64_t stream_base,
                  uint64_t *__restrict__ chunk_start, uint64_t *__restrict__ chunk_len,
                  uint64_t *__restrict__ chunk_end_out)
{
    const uint32_t f = blockIdx.x;
    if (f >= n_files || sc->err)
        return;
    const CdcFile fl = files[f];
    if (fl.len < SELECT_BIG_FILE)
        return;
    const uint64_t out = sc->n_chunks + bases[f];
    const uint64_t *c = cuts + fl.scratch;
    for (uint32_t j = threadIdx.x; j < counts[f]; j += blockDim.x) {
        const uint64_t s0 = j ? c[j - 1] : 0, e0 = c[j];
        if (out + j < max_chunks) {
            chunk_start[out + j] = fl.off + s0;
            chunk_len[out + j] = e0 - s0;
            chunk_end_out[out + j] = stream_base + fl.off + e0;
        }
    }
}

// after the scan of counts: publish the batch chunk count / overflow
__global__ void k_batch_begin(SessionCounters *sc, const uint32_t *counts, const uint32_t *bases, uint32_t n_files,
                              uint64_t max_chunks, uint64_t cdc_bytes, uint32_t n_continued /* pieces of files counted earlier */)
{
    if (blockIdx.x == 0 && threadIdx.x < LEN_CLASSES) {
        sc->len_bins[threadIdx.x] = 0;
        sc->len_cursor[threadIdx.x] = 0;
    }
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        uint32_t total = n_files ? bases[n_files - 1] + counts[n_files - 1] : 0;
        sc->batch_chunks = total;
        sc->work = 0;
        if (sc->n_chunks + total > max_chunks)
            sc->err |= 2u;
        sc->n_files += n_files - n_continued;
        sc->cdc_bytes += cdc_bytes;
    }
}

// A file larger than one arena (tario.WriteEntry streams any size, lib/tario/write.go:45).  The piece of such a file
// ends with an OPEN chunk the cut rule cannot close without the bytes that follow (sc->carry_off/len, < max_size).
// k_carry_out parks it in a side buffer at the end of its submit (the slot may be overwritten by the next H2D);
// k_carry_in of the next submit copies it in FRONT of the continuation, which the packer placed at `cont_off` of the
// new arena with at least max_size free bytes before it, and widens the file record to start at the open chunk.
// k_carry_in runs on the compute stream after the new arena's H2D copy has landed.  One CTA each.
__global__ void __launch_bounds__(256)
k_carry_out(const uint8_t *__restrict__ src_slot, uint8_t *__restrict__ carry, uint64_t carry_cap, SessionCounters *__restrict__ sc)
{
    const uint64_t n = sc->carry_len, from = sc->carry_off;
    if (n > carry_cap) {
        if (threadIdx.x == 0)
            sc->err |= 8u;
        return;
    }
    for (uint64_t i = threadIdx.x; i < n; i += blockDim.x)
        carry[i] = src_slot[from + i];
}

__global__ void __launch_bounds__(256)
k_carry_in(const uint8_t *__restrict__ carry, uint8_t *__restrict__ dst_slot, uint64_t cont_off, CdcFile *__restrict__ files,
           uint32_t cont_index, SessionCounters *__restrict__ sc)
{
    const uint64_t n = sc->carry_len;
    if (n > cont_off) { // cannot happen: carry_len < max_size <= cont_off (checked at submit)
        if (threadIdx.x == 0)
            sc->err |= 8u;
        return;
    }
    uint8_t *d = dst_slot + cont_off - n;
    for (uint64_t i = threadIdx.x; i < n; i += blockDim.x)
        d[i] = carry[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        files[cont_index].off = cont_off - n;
        files[cont_index].len += n;
        sc->carry_len = 0;
        sc->carry_off = 0;
    }
}

__global__ void k_batch_end(SessionCounters *sc)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        if (!sc->err)
            sc->n_chunks += sc->batch_chunks;
        sc->batch_chunks = 0;
        sc->work = 0;
    }
}

// K2a: chunk digests remembered from an earlier session (mksnap_chunks_add) join the chunk table behind the chunks of
// the submits enqueued before them.  Chunks never span files, so a file's digests depend on its bytes alone and the
// sorted-unique table -- hence the root -- of the union is that of a full pass.  k_chunks_append writes rows
// [n_chunks, n_chunks + n) (digest, end = UINT64_MAX so that callers of mksnap_get_chunks can tell them from computed
// chunks); k_chunks_commit then publishes them.  Both apply the same test first: a session that already failed, or rows
// that would run past max_chunks, write nothing, and k_chunks_commit sets the table-overflow bit (finish reports
// MKSNAP_E_CAPACITY).  Two launches instead of one keep the counter read of every CTA ahead of the update.
constexpr int APPEND_THREADS = 256;

__device__ __forceinline__ bool chunks_append_refused(const SessionCounters *sc, uint32_t n, uint64_t max_chunks)
{
    return sc->err != 0 || sc->n_chunks + n > max_chunks;
}

__global__ void __launch_bounds__(APPEND_THREADS)
k_chunks_append(const uint4 *__restrict__ rows, uint32_t n, const SessionCounters *__restrict__ sc, uint64_t max_chunks,
                uint4 *__restrict__ digests, uint64_t *__restrict__ chunk_end)
{
    if (chunks_append_refused(sc, n, max_chunks))
        return;
    const uint64_t base = sc->n_chunks;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * n; i += gridDim.x * blockDim.x) { // 2 x 16 B per row
        digests[2 * base + i] = rows[i];
        if (!(i & 1u))
            chunk_end[base + i / 2] = ~0ull;
    }
}

__global__ void k_chunks_commit(SessionCounters *sc, uint32_t n, uint64_t max_chunks)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        if (!chunks_append_refused(sc, n, max_chunks))
            sc->n_chunks += n;
        else if (!sc->err)
            sc->err |= 2u;
    }
}

// ------------------------------------------------------------------------
// K2 work order.  A lane hashes one chunk serially (slowly: one lane of a full SM), so when the work list runs
// dry every warp keeps issuing for as long as its LONGEST unfinished chunk lasts: with content-defined lengths
// (4 KiB .. 128 KiB) that drain is a visible share of the kernel (measured against equal-length chunks).  Handing chunks out
// longest class first leaves only the shortest ones for the end.  Counting sort by 2 KiB length class:
// k_len_hist counts, k_len_order writes batch-relative chunk indices, largest class first (order inside a class
// is arbitrary: digests are stored by chunk index, so the result does not depend on it).
// ------------------------------------------------------------------------
constexpr int LEN_THREADS = 256;
constexpr int LEN_ITEMS = 8;

__device__ __forceinline__ uint32_t len_class(uint64_t len)
{
    const uint64_t c = len >> LEN_CLASS_SHIFT;
    return c < LEN_CLASSES - 1 ? (uint32_t)c : LEN_CLASSES - 1;
}

__global__ void __launch_bounds__(LEN_THREADS) k_len_hist(const uint64_t *__restrict__ len, SessionCounters *sc)
{
    if (sc->err)
        return;
    __shared__ uint32_t s_cnt[LEN_CLASSES];
    if (threadIdx.x < LEN_CLASSES)
        s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t n = sc->batch_chunks, first = sc->n_chunks;
    for (uint64_t i = (uint64_t)blockIdx.x * LEN_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * LEN_THREADS)
        atomicAdd(&s_cnt[len_class(len[first + i])], 1u);
    __syncthreads();
    if (threadIdx.x < LEN_CLASSES && s_cnt[threadIdx.x])
        atomicAdd(&sc->len_bins[threadIdx.x], s_cnt[threadIdx.x]);
}

__global__ void __launch_bounds__(LEN_THREADS) k_len_order(const uint64_t *__restrict__ len, SessionCounters *sc,
                                                           uint32_t *__restrict__ order)
{
    if (sc->err)
        return;
    __shared__ uint32_t s_cnt[LEN_CLASSES], s_base[LEN_CLASSES], s_got[LEN_CLASSES];
    const uint32_t t = threadIdx.x;
    if (t < LEN_CLASSES) { // first slot of class t = number of chunks in longer classes
        uint32_t b = 0;
        for (uint32_t c = t + 1; c < LEN_CLASSES; ++c)
            b += sc->len_bins[c];
        s_base[t] = b;
    }
    const uint64_t n = sc->batch_chunks, first = sc->n_chunks;
    constexpr uint64_t TILE = (uint64_t)LEN_THREADS * LEN_ITEMS;
    for (uint64_t t0 = (uint64_t)blockIdx.x * TILE; t0 < n; t0 += (uint64_t)gridDim.x * TILE) {
        if (t < LEN_CLASSES)
            s_cnt[t] = 0;
        __syncthreads();
        uint32_t cls[LEN_ITEMS], rank[LEN_ITEMS];
#pragma unroll
        for (int j = 0; j < LEN_ITEMS; ++j) {
            const uint64_t i = t0 + (uint64_t)j * LEN_THREADS + t;
            cls[j] = LEN_CLASSES;
            if (i < n) {
                cls[j] = len_class(len[first + i]);
                rank[j] = atomicAdd(&s_cnt[cls[j]], 1u);
            }
        }
        __syncthreads();
        if (t < LEN_CLASSES && s_cnt[t])
            s_got[t] = atomicAdd(&sc->len_cursor[t], s_cnt[t]);
        __syncthreads();
#pragma unroll
        for (int j = 0; j < LEN_ITEMS; ++j)
            if (cls[j] < LEN_CLASSES)
                order[s_base[cls[j]] + s_got[cls[j]] + rank[j]] = (uint32_t)(t0 + (uint64_t)j * LEN_THREADS + t);
        __syncthreads();
    }
}

// ------------------------------------------------------------------------
// K2: SHA-256 of the chunks of the chunk table.  One lane per chunk, one
// 64-byte block per loop iteration; a lane that finishes its chunk pulls the
// next one from a global counter, so a warp stays converged on "compress one
// block" no matter how ragged the chunk lengths are.  Chunks start at
// arbitrary byte alignment (cut points are content defined): each lane
// stages the five aligned 16-byte words that cover its block in shared
// memory and reads the 17 words from the one that holds the block's first
// byte back, so the word rotation costs no ALU instruction; one PRMT per word
// does the byte shift and the big-endian swap together.
// ------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

// FMA_ADDS = true: additions as IMAD (throughput: many chunks, ALU pipe saturated);
// false: plain adds (IADD3, shorter dependent chain).
template <bool FMA_ADDS> __device__ __forceinline__ uint32_t sha_add(uint32_t a, uint32_t b, uint32_t one)
{
    return FMA_ADDS ? fma_add_rt(a, b, one) : a + b;
}

// x + K (round constant): IMAD(one, K, x) keeps this add off the ALU pipe as well; after unrolling K is an
// immediate operand of the IMAD.
template <bool FMA_ADDS> __device__ __forceinline__ uint32_t sha_addk(uint32_t x, uint32_t k, uint32_t one)
{
    if (!FMA_ADDS)
        return x + k;
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(one), "r"(k), "r"(x));
    return d;
}

#ifndef SHA_SHR_MULHI
#define SHA_SHR_MULHI 0
#endif
// Register budget: the kernel is ALU-pipe bound; 5 CTAs per SM (20 warps) keep the pipe fed and the extra
// registers remove moves.
#ifndef SHA_MINBLOCKS
#define SHA_MINBLOCKS 5
#endif
#define SHA_LAUNCH_BOUNDS __launch_bounds__(SHA_THREADS, SHA_MINBLOCKS)
// x >> n as the high half of x * 2^(32-n): one IMAD.HI on the FMA pipe instead of one SHF on the ALU pipe.  The
// multiplier is a runtime value (derived from the `one` kernel argument) so ptxas cannot turn it back into a shift.
__device__ __forceinline__ uint32_t shr_mulhi(uint32_t x, uint32_t pow2)
{
    uint32_t d;
    asm("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(pow2));
    return d;
}

template <bool FMA_ADDS>
__device__ __forceinline__ void sha256_compress(uint32_t st[8], uint32_t w[16], const uint32_t one)
{
    const uint32_t p29 = one << 29, p22 = one << 22;
    (void)p29; (void)p22;
    constexpr uint32_t K[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
        0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
        0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
        0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
        0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
        0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
        0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
        0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        uint32_t wi;
        if (i < 16) {
            wi = w[i];
        } else {
            const uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            const uint32_t sh3 = (FMA_ADDS && SHA_SHR_MULHI >= 1) ? shr_mulhi(w15, p29) : (w15 >> 3);
            const uint32_t sh10 = (FMA_ADDS && SHA_SHR_MULHI >= 2) ? shr_mulhi(w2, p22) : (w2 >> 10);
            const uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ sh3;
            const uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ sh10;
            wi = sha_add<FMA_ADDS>(sha_add<FMA_ADDS>(w[i & 15], s0, one), sha_add<FMA_ADDS>(w[(i + 9) & 15], s1, one), one);
            w[i & 15] = wi;
        }
        const uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
        const uint32_t ch = (e & f) ^ (~e & g);
        const uint32_t t1 = sha_add<FMA_ADDS>(sha_add<FMA_ADDS>(h, S1, one), sha_add<FMA_ADDS>(ch, wi + K[i], one), one);
        const uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
        const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        h = g; g = f; f = e; e = sha_add<FMA_ADDS>(d, t1, one);
        d = c; c = b; b = a; a = sha_add<FMA_ADDS>(sha_add<FMA_ADDS>(t1, S0, one), mj, one);
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d;
    st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

constexpr int SHA_THREADS = 128;
constexpr int SHA_WIN = 5; // 16-byte words of a block's aligned window: 80 bytes cover 64 at any alignment

// Stage a block's window (SHA_WIN aligned 16-byte words from q; word k only if bit k of `mask` is set) at shared
// address `wr`.
__device__ __forceinline__ void sha_stage(uint32_t wr, const uint4 *q, uint32_t mask)
{
#pragma unroll
    for (int k = 0; k < SHA_WIN; ++k)
        if (mask & (1u << k)) {
            const uint4 v = __ldg(q + k);
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};"
                         :: "r"(wr + 16 * k), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
        }
}

// The 16 big-endian message words of a staged block: 17 words from shared address `rd` (the word holding the block's
// first byte), one PRMT each for the byte shift and the swap.
__device__ __forceinline__ void sha_unstage(uint32_t w[16], uint32_t rd, uint32_t sel)
{
    uint32_t z[17];
#pragma unroll
    for (int i = 0; i < 17; ++i)
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(z[i]) : "r"(rd + 4 * i));
#pragma unroll
    for (int i = 0; i < 16; ++i) // prmt, not __byte_perm: `sel` is a valid selector, no mask per block
        asm("prmt.b32 %0, %1, %2, %3;" : "=r"(w[i]) : "r"(z[i]), "r"(z[i + 1]), "r"(sel));
}

// Chunk i of the batch is row sc->n_chunks + i of start/len/out; `order` (or nullptr: batch order) is the order in
// which the lanes take them.  A chunk is at most max_size (32-bit) bytes long.
template <bool FMA_ADDS>
__global__ void SHA_LAUNCH_BOUNDS
k_sha256_ranges(const uint8_t *__restrict__ data, const uint64_t *__restrict__ start, const uint64_t *__restrict__ len,
                SessionCounters *__restrict__ sc, uint8_t *__restrict__ out, const uint32_t one,
                const uint32_t *__restrict__ order)
{
    // a lane's window at a stride of 20 words: the STS.128 of a quarter warp hit 8 distinct 16-byte bank groups
    __shared__ uint4 s_win[SHA_THREADS * SHA_WIN];
    if (sc->err)
        return;
    const uint32_t n = sc->batch_chunks;
    const uint64_t first = sc->n_chunks;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(s_win + threadIdx.x * SHA_WIN);

    uint32_t st[8];
    const uint4 *q = nullptr; // window of the next block: its first 16-byte word holds the block's first byte
    uint32_t a = 0;           // the chunk's start mod 16, the same for every block of it
    uint32_t wr = base;       // shared address of this lane's window
    uint32_t rd = 0;          // shared address of the window's word that holds the block's first byte
    uint32_t sel = 0;         // PRMT selector: byte shift by a & 3 and big-endian swap
    uint32_t left = 0;        // phase 1: bytes of the chunk not yet compressed; otherwise 0
    uint32_t total = 0;       // chunk length
    uint64_t my = 0;          // row of the chunk in start/len/out
    uint32_t phase = 0;       // 0 idle, 1 data blocks, 2 needs extra length block
    bool exhausted = false;

    for (;;) {
        // Only a lane within 80 bytes of its chunk's end, or without a chunk, needs more than a full block.
        bool full = __all_sync(0xFFFFFFFFu, left >= 80);
        if (!full) {
            // ---- refill idle lanes (warp-aggregated fetch) ----
            const uint32_t need = __ballot_sync(0xFFFFFFFFu, phase == 0 && !exhausted);
            if (need) {
                uint32_t basei = 0;
                const uint32_t leader = __ffs(need) - 1;
                if (lane == leader)
                    basei = atomicAdd(&sc->work, __popc(need));
                basei = __shfl_sync(0xFFFFFFFFu, basei, leader);
                if (phase == 0 && !exhausted) {
                    const uint32_t idx = basei + __popc(need & ((1u << lane) - 1u));
                    if (idx < n) {
                        my = first + (order ? order[idx] : idx);
                        const uint8_t *p = data + start[my];
                        total = left = (uint32_t)len[my];
                        a = (uint32_t)((uintptr_t)p & 15u);
                        q = reinterpret_cast<const uint4 *>(p - a);
                        rd = base + (a & 12u);
                        wr = rd & ~15u; // = base; derived from rd so that it stays in a register
                        sel = 0x0123u + 0x1111u * (a & 3u);
                        phase = 1;
                        st[0] = 0x6a09e667; st[1] = 0xbb67ae85; st[2] = 0x3c6ef372; st[3] = 0xa54ff53a;
                        st[4] = 0x510e527f; st[5] = 0x9b05688c; st[6] = 0x1f83d9ab; st[7] = 0x5be0cd19;
                    } else {
                        exhausted = true;
                    }
                }
            }
            if (!__any_sync(0xFFFFFFFFu, phase != 0))
                break;
            full = left >= 80;
        }

        uint32_t w[16];
        bool last = false;
        if (full) {
            // full block: the window starts at or before the block and ends before its byte 80, inside the chunk
            sha_stage(wr, q, 0x1Fu);
            sha_unstage(w, rd, sel);
            q += 4;
            left -= 64;
        } else if (phase == 0) {
            continue;
        } else if (phase == 2) {
#pragma unroll
            for (int i = 0; i < 14; ++i)
                w[i] = 0;
            w[14] = total >> 29;
            w[15] = total << 3;
            last = true;
        } else {
            // the chunk's last one or two blocks: only the 16-byte words that hold bytes of the chunk are read.  The
            // others keep an earlier block's bytes, which all lie past the chunk's end and are masked off below.
            const uint32_t lim = a + (left < 64 ? left : 64u);
            uint32_t mask = 0;
#pragma unroll
            for (int k = 0; k < SHA_WIN; ++k)
                mask |= (uint32_t)(16 * k < lim) << k;
            sha_stage(wr, q, mask);
            sha_unstage(w, rd, sel);
            if (left >= 64) {
                q += 4;
                left -= 64;
            } else {
                // final data block: keep `left` bytes, append 0x80, zero the rest
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int32_t k = (int32_t)left - 4 * i; // valid bytes in this word
                    uint32_t keep = k >= 4 ? 0xFFFFFFFFu : (k <= 0 ? 0u : ~(0xFFFFFFFFu >> (8 * k)));
                    uint32_t v = w[i] & keep;
                    if (k >= 0 && k < 4)
                        v |= 0x80000000u >> (8 * k);
                    w[i] = v;
                }
                if (left < 56) {
                    w[14] = total >> 29;
                    w[15] = total << 3;
                    last = true;
                } else {
                    phase = 2;
                }
                left = 0;
            }
        }
        sha256_compress<FMA_ADDS>(st, w, one);
        if (last) {
            uint4 o0, o1;
            o0.x = __byte_perm(st[0], 0, 0x0123); o0.y = __byte_perm(st[1], 0, 0x0123);
            o0.z = __byte_perm(st[2], 0, 0x0123); o0.w = __byte_perm(st[3], 0, 0x0123);
            o1.x = __byte_perm(st[4], 0, 0x0123); o1.y = __byte_perm(st[5], 0, 0x0123);
            o1.z = __byte_perm(st[6], 0, 0x0123); o1.w = __byte_perm(st[7], 0, 0x0123);
            uint4 *dst = reinterpret_cast<uint4 *>(out + my * 32);
            dst[0] = o0;
            dst[1] = o1;
            phase = 0;
        }
    }
}

// ------------------------------------------------------------------------
// generic exclusive scan of u32 (block = 256 threads x 4 items)
// ------------------------------------------------------------------------
constexpr uint32_t SCAN_ITEMS = 1024;

__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t *s_w, uint32_t &total)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, s);
        if (lane >= s)
            incl += t;
    }
    if (lane == 31)
        s_w[warp] = incl;
    __syncthreads();
    uint32_t woff = 0;
    total = 0;
#pragma unroll
    for (uint32_t k = 0; k < 8; ++k) {
        const uint32_t t = s_w[k];
        if (k < warp)
            woff += t;
        total += t;
    }
    __syncthreads();
    return woff + incl - v;
}

__global__ void __launch_bounds__(256) k_scan_reduce(const uint32_t *in, uint64_t n, uint32_t *sums)
{
    __shared__ uint32_t s_w[8];
    const uint64_t b0 = (uint64_t)blockIdx.x * SCAN_ITEMS + threadIdx.x * 4;
    uint32_t v = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (b0 + k < n)
            v += in[b0 + k];
    uint32_t total;
    block_exclusive_scan_256(v, s_w, total);
    if (threadIdx.x == 0)
        sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(256) k_scan_apply(const uint32_t *in, uint64_t n, const uint32_t *block_off, uint32_t *out)
{
    __shared__ uint32_t s_w[8];
    const uint64_t b0 = (uint64_t)blockIdx.x * SCAN_ITEMS + threadIdx.x * 4;
    uint32_t x[4], v = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        x[k] = b0 + k < n ? in[b0 + k] : 0;
        v += x[k];
    }
    uint32_t total;
    uint32_t ex = block_exclusive_scan_256(v, s_w, total) + (block_off ? block_off[blockIdx.x] : 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (b0 + k < n)
            out[b0 + k] = ex;
        ex += x[k];
    }
}

// ------------------------------------------------------------------------
// K3: LSD radix sort of (u64 key, u32 payload), 8 bits per pass, then unique.
// key = first 8 digest bytes big-endian.  Only the top SORT_KEY_BITS are radix-sorted (SHA-256 output is
// uniform: at 10^7..10^8 rows a 32-bit prefix leaves runs of a few rows); k_fix_ties then orders every run of
// equal prefix on the full 256 bits, so the final order is the full bytewise order.
constexpr int SORT_KEY_BITS = 32;
// ------------------------------------------------------------------------
constexpr uint32_t SORT_THREADS = 256;
constexpr uint32_t SORT_ITEMS = 16;
constexpr uint32_t SORT_TILE = SORT_THREADS * SORT_ITEMS;

__global__ void k_make_keys(const uint8_t *__restrict__ digests, uint64_t n, uint64_t *keys, uint32_t *idx)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const uint2 v = *reinterpret_cast<const uint2 *>(digests + i * 32);
    keys[i] = ((uint64_t)__byte_perm(v.x, 0, 0x0123) << 32) | __byte_perm(v.y, 0, 0x0123);
    idx[i] = (uint32_t)i;
}

// histogram: hist[digit * nblocks + block]
__global__ void __launch_bounds__(SORT_THREADS)
k_radix_hist(const uint64_t *__restrict__ keys, uint64_t n, int shift, uint32_t *__restrict__ hist, uint32_t nblocks)
{
    __shared__ uint32_t s_h[256];
    s_h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t b0 = (uint64_t)blockIdx.x * SORT_TILE;
    for (uint32_t k = 0; k < SORT_ITEMS; ++k) {
        const uint64_t i = b0 + k * SORT_THREADS + threadIdx.x;
        if (i < n)
            atomicAdd(&s_h[(keys[i] >> shift) & 0xFF], 1u);
    }
    __syncthreads();
    hist[(uint64_t)threadIdx.x * nblocks + blockIdx.x] = s_h[threadIdx.x];
}

__global__ void __launch_bounds__(SORT_THREADS)
k_radix_scatter(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals, uint64_t n, int shift,
                const uint32_t *__restrict__ offs, uint32_t nblocks, uint64_t *__restrict__ keys_out,
                uint32_t *__restrict__ vals_out)
{
    __shared__ uint32_t s_cnt[SORT_THREADS / 32][256];
    __shared__ uint32_t s_run[256];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    s_run[threadIdx.x] = offs[(uint64_t)threadIdx.x * nblocks + blockIdx.x];
    const uint64_t b0 = (uint64_t)blockIdx.x * SORT_TILE;
    for (uint32_t k = 0; k < SORT_ITEMS; ++k) {
        for (uint32_t j = threadIdx.x; j < (SORT_THREADS / 32) * 256; j += SORT_THREADS)
            (&s_cnt[0][0])[j] = 0;
        __syncthreads();
        const uint64_t i = b0 + k * SORT_THREADS + threadIdx.x;
        const bool ok = i < n;
        uint64_t key = 0;
        uint32_t val = 0, d = 0, rank = 0;
        if (ok) {
            key = keys[i];
            val = vals[i];
            d = (uint32_t)(key >> shift) & 0xFF;
        }
        const uint32_t okmask = __ballot_sync(0xFFFFFFFFu, ok);
        if (ok) {
            const uint32_t peers = __match_any_sync(okmask, d);
            rank = __popc(peers & ((1u << lane) - 1u));
            if (rank == 0)
                s_cnt[warp][d] = __popc(peers);
        }
        __syncthreads();
        if (ok) {
            uint32_t before = 0;
            for (uint32_t wq = 0; wq < warp; ++wq)
                before += s_cnt[wq][d];
            const uint32_t dst = s_run[d] + before + rank;
            keys_out[dst] = key;
            vals_out[dst] = val;
        }
        __syncthreads();
        {
            uint32_t add = 0;
#pragma unroll
            for (uint32_t wq = 0; wq < SORT_THREADS / 32; ++wq)
                add += s_cnt[wq][threadIdx.x];
            s_run[threadIdx.x] += add;
        }
        __syncthreads();
    }
}

__global__ void k_gather_digests(const uint8_t *__restrict__ digests, const uint32_t *__restrict__ idx, uint64_t n,
                                 uint8_t *__restrict__ out)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t i = t >> 1;
    if (i >= n)
        return;
    const uint4 *src = reinterpret_cast<const uint4 *>(digests + (uint64_t)idx[i] * 32);
    reinterpret_cast<uint4 *>(out + i * 32)[t & 1] = src[t & 1];
}

__device__ __forceinline__ int digest_cmp(const uint8_t *a, const uint8_t *b)
{
    // bytewise order == order of big-endian words
    const uint32_t *x = reinterpret_cast<const uint32_t *>(a), *y = reinterpret_cast<const uint32_t *>(b);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t p = __byte_perm(x[k], 0, 0x0123), q = __byte_perm(y[k], 0, 0x0123);
        if (p != q)
            return p < q ? -1 : 1;
    }
    return 0;
}

// Runs of equal radix prefix are put in full 256-bit order.  SHA-256 output is uniform, so between DISTINCT digests a
// run is a handful of rows and one thread's insertion sort is the cheapest thing to do.  Long runs are duplicates: an
// all-zero context is one max-size chunk repeated (a 50 GiB zero context = 400 k identical rows), which one thread
// would walk for tens of milliseconds.  Runs longer than FIX_SHORT rows go to a list instead and k_fix_long_runs
// checks each of them with a whole CTA: all rows equal (the only case seen in practice) => nothing to do; otherwise
// (distinct digests sharing 32 bits AND a long run of duplicates, ~n/2^32 likely) thread 0 insertion-sorts it.
constexpr uint32_t FIX_SHORT = 64;
constexpr uint32_t FIX_LONG_CAP = 8192; // list entries; a further long run is sorted by its own thread

__device__ __forceinline__ void fix_insertion_sort(uint8_t *__restrict__ d, uint64_t i, uint64_t e)
{
    for (uint64_t j = i + 1; j < e; ++j) {
        uint64_t k = j;
        while (k > i && digest_cmp(d + (k - 1) * 32, d + k * 32) > 0) {
            uint4 *a = reinterpret_cast<uint4 *>(d + (k - 1) * 32), *b = reinterpret_cast<uint4 *>(d + k * 32);
            uint4 t0 = a[0], t1 = a[1];
            a[0] = b[0]; a[1] = b[1];
            b[0] = t0; b[1] = t1;
            --k;
        }
    }
}

__global__ void k_fix_ties(const uint64_t *__restrict__ keys, uint64_t n, uint8_t *__restrict__ d, int shift,
                           uint2 *__restrict__ long_runs, uint32_t *__restrict__ n_long)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const uint64_t ki = keys[i] >> shift; // only the bits the radix passes sorted on
    if (i > 0 && (keys[i - 1] >> shift) == ki)
        return; // not a run start
    if (i + 1 >= n || (keys[i + 1] >> shift) != ki)
        return; // a run of one
    // run end: gallop, then binary search (keys are sorted on these bits)
    uint64_t lo = i + 1, step = 1;
    while (lo + step < n && (keys[lo + step] >> shift) == ki) {
        lo += step;
        step <<= 1;
    }
    uint64_t hi = lo + step < n ? lo + step : n; // keys[lo] is in the run, keys[hi] (if any) is not
    while (hi - lo > 1) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if ((keys[mid] >> shift) == ki)
            lo = mid;
        else
            hi = mid;
    }
    const uint64_t e = hi;
    if (e - i > FIX_SHORT && e <= 0xFFFFFFFFull) {
        const uint32_t slot = atomicAdd(n_long, 1u);
        if (slot < FIX_LONG_CAP) {
            long_runs[slot] = make_uint2((uint32_t)i, (uint32_t)e);
            return;
        }
    }
    fix_insertion_sort(d, i, e);
}

__global__ void __launch_bounds__(256) k_fix_long_runs(uint8_t *__restrict__ d, const uint2 *__restrict__ long_runs,
                                                       const uint32_t *__restrict__ n_long)
{
    const uint32_t total = *n_long < FIX_LONG_CAP ? *n_long : FIX_LONG_CAP;
    for (uint32_t r = blockIdx.x; r < total; r += gridDim.x) {
        const uint64_t i = long_runs[r].x, e = long_runs[r].y;
        const uint4 f0 = reinterpret_cast<const uint4 *>(d + i * 32)[0], f1 = reinterpret_cast<const uint4 *>(d + i * 32)[1];
        int differs = 0;
        for (uint64_t j = i + 1 + threadIdx.x; j < e; j += blockDim.x) {
            const uint4 a = reinterpret_cast<const uint4 *>(d + j * 32)[0], b = reinterpret_cast<const uint4 *>(d + j * 32)[1];
            differs |= (a.x ^ f0.x) | (a.y ^ f0.y) | (a.z ^ f0.z) | (a.w ^ f0.w) | (b.x ^ f1.x) | (b.y ^ f1.y) | (b.z ^ f1.z) | (b.w ^ f1.w);
        }
        if (__syncthreads_or(differs) && threadIdx.x == 0)
            fix_insertion_sort(d, i, e);
        __syncthreads();
    }
}

__global__ void k_unique_flags(const uint8_t *__restrict__ d, uint64_t n, uint32_t *__restrict__ flags)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    flags[i] = (i == 0 || digest_cmp(d + (i - 1) * 32, d + i * 32) != 0) ? 1u : 0u;
}

__global__ void k_compact_digests(const uint8_t *__restrict__ d, const uint32_t *__restrict__ flags,
                                  const uint32_t *__restrict__ pos, uint64_t n, uint8_t *__restrict__ out)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t i = t >> 1;
    if (i >= n || !flags[i])
        return;
    reinterpret_cast<uint4 *>(out + (uint64_t)pos[i] * 32)[t & 1] = reinterpret_cast<const uint4 *>(d + i * 32)[t & 1];
}

} // namespace mk
