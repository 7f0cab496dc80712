// mksnap_inflate.cuh -- gunzip on the device (mksnap_gunzip_open / _read / _close / _get_times), included at the end of
// mksnap.cu (the entry points have C linkage through include/mksnap.h).
//
//   K5a k_gz_scan_headers                  member body starts into a bitmap (one bit per blob byte)   (HBM, tiny)
//       k_gz_scan_count / k_gz_scan_write  candidate segment starts in offset order: the byte after every
//                                          00 00 FF FF, and every body start of the bitmap            (HBM, tiny)
//   K5b k_gz_decode     count mode: speculative decode of every candidate, no output;                 (latency bound)
//                       write mode: the true segments of one window, 16-bit symbols
//       k_gz_decode_bits  the same for mksnap_gunzip_open_indexed: bit positions, count decodes record block starts
//   K5c k_gz_resolve    window tails in segment order, one CTA                                        (latency, small)
//   K5d k_gz_narrow     markers -> bytes, 16-bit symbols -> bytes                                     (HBM)
//   K0  k_crc32_extents the CRC-32 of every member piece of the window (the context-CRC kernel as it is)
//
// The DEFLATE and gzip logic is mksnap_inflate_core.h (shared with the CPU mock of the engine).  The link -- following
// the segment ends from each member start, reading trailers and the next member header -- runs on the host over the
// count results.  Every member body start is a scanned candidate (the scan accepts any header the link accepts), so the
// members of a bgzip / eStargz / concatenated blob are count-decoded in parallel like flush segments; only a start whose
// count decode was cut short by the K limit is decoded again on the device without the limit, one such start per
// launch.  The link treats both kinds of candidate alike: a block that ends on either is a block boundary.
//
// Device memory of an open gunzip: the blob (gz_len), 8 bytes per candidate start and 32 per count result (at most
// gz_len / 4 + gz_len / 3 + 1 candidates: 00 00 FF FF cannot overlap itself, 1f 8b 08 cannot overlap itself or it, and
// each header start gives one body start), a bitmap of gz_len / 8 bytes during the scan only, the segment and extent
// tables, two 32 KiB history buffers, and one output window of max(GZ_WINDOW, largest segment) bytes at 3 bytes per
// output byte (16-bit symbols plus bytes), copied once per window to a pinned host buffer of the same size that the
// reads copy from.  It does not grow with the decompressed length except through the largest segment: a member without
// flush points is one segment, unless it is opened indexed: there segments are cut about every 1 MiB of output at
// recorded block starts, and the open adds 8 bytes per point and per cut to the candidate tables, 32 per point to the
// count results, and a record buffer of REC_CAP * 24 bytes (1.5 MiB).  Everything runs on the gunzip's own stream: reads interleaved with an ingest session
// do not queue behind its kernels.
#include "mksnap_inflate_core.h"

namespace gz {

constexpr uint64_t GZ_WINDOW = 256ull << 20;  // output bytes per window (at least one whole segment)
constexpr uint32_t SCAN_CHUNK = 4096;          // blob bytes per scan thread
constexpr int DEC_WARPS = 2;                   // warps per CTA of k_gz_decode (one segment per warp)

// Member headers: thread c parses every header that starts in [c * SCAN_CHUNK, (c + 1) * SCAN_CHUNK), reading past
// its chunk as far as the header goes, and sets bit p of `body` for its body start p (from < p <= gz_len).  Body
// starts are neither ordered nor distinct across header starts, so they meet in a bitmap, and the two kernels below
// read them back in offset order.
__global__ void k_gz_scan_headers(const uint8_t *__restrict__ gz, uint64_t gz_len, uint64_t from,
                                  uint32_t *__restrict__ body, uint32_t n_chunks)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks)
        return;
    const uint64_t a = (uint64_t)c * SCAN_CHUNK, b = min(a + SCAN_CHUNK, gz_len);
    for (uint64_t q = a; q < b; ++q) {
        if (gz[q] != 0x1f)
            continue;
        const int64_t p = mki::member_body(gz, gz_len, q);
        if (p > (int64_t)from)
            atomicOr(body + (p >> 5), 1u << (p & 31));
    }
}

__device__ __forceinline__ bool is_cand(const uint8_t *__restrict__ gz, const uint32_t *__restrict__ body, uint64_t p)
{
    return mki::flush_end(gz, p) || ((body[p >> 5] >> (p & 31)) & 1u);
}

// candidates p, from < p <= to, per chunk: counts (and their sum in *total, to catch a 32-bit scan overflow), then
// the offsets in order
__global__ void k_gz_scan_count(const uint8_t *__restrict__ gz, uint64_t from, uint64_t to,
                                const uint32_t *__restrict__ body, uint32_t *__restrict__ cnt, uint32_t n_chunks,
                                unsigned long long *__restrict__ total)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks)
        return;
    const uint64_t a = from + 1 + (uint64_t)c * SCAN_CHUNK, b = min(a + SCAN_CHUNK, to + 1);
    uint32_t k = 0;
    for (uint64_t p = a; p < b; ++p)
        k += is_cand(gz, body, p);
    cnt[c] = k;
    atomicAdd(total, (unsigned long long)k);
}

__global__ void k_gz_scan_write(const uint8_t *__restrict__ gz, uint64_t from, uint64_t to,
                                const uint32_t *__restrict__ body, const uint32_t *__restrict__ base, uint32_t n_chunks,
                                uint64_t *__restrict__ cand)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks)
        return;
    const uint64_t a = from + 1 + (uint64_t)c * SCAN_CHUNK, b = min(a + SCAN_CHUNK, to + 1);
    uint64_t *o = cand + 1 + base[c]; // cand[0] is the first member's body start
    for (uint64_t p = a; p < b; ++p)
        if (is_cand(gz, body, p))
            *o++ = p;
}

// Count mode (segs == nullptr): decode from starts[i], i < n, with limit K, into res[i].  Write mode: decode window
// segment i into sym + segs[i].out_off - win_off; a result that differs from what the count pass found (it cannot,
// unless the write mode finds a distance before the member start) sets *bad.
__global__ void __launch_bounds__(32 * DEC_WARPS)
k_gz_decode(const uint8_t *__restrict__ gz, uint64_t gz_len, const uint64_t *__restrict__ cand, uint64_t n_cand,
            const uint64_t *__restrict__ starts, uint64_t n, uint32_t K, mki::SegRes *__restrict__ res,
            const mki::Seg *__restrict__ segs, uint64_t win_off, uint16_t *__restrict__ sym, uint32_t *__restrict__ bad)
{
    const uint64_t i = (uint64_t)blockIdx.x * DEC_WARPS + (threadIdx.x >> 5);
    if (i >= n || (threadIdx.x & 31u))
        return;
    mki::Tables t;
    if (!segs) {
        res[i] = mki::decode_segment(gz, gz_len, starts[i], cand, n_cand, K, nullptr, 0, 0, &t);
        return;
    }
    const mki::Seg s = segs[i];
    const mki::SegRes r = mki::decode_segment(gz, gz_len, s.start, cand, n_cand, mki::NO_LIMIT, sym + (s.out_off - win_off),
                                              s.out_len, s.member_pos, &t);
    if (r.status != (s.final ? mki::SEG_FINAL : mki::SEG_CAND) || r.end != s.end || r.out_len != s.out_len)
        atomicOr(bad, 1u);
}

// k_gz_decode of an indexed open: starts, candidates and segment ends are bit offsets, and count decodes record block
// starts into `rec` (mksnap_inflate_core.h, Recorder).  A kernel of its own, so that k_gz_decode is unchanged.
__global__ void __launch_bounds__(32 * DEC_WARPS)
k_gz_decode_bits(const uint8_t *__restrict__ gz, uint64_t gz_len, const uint64_t *__restrict__ cand, uint64_t n_cand,
                 const uint64_t *__restrict__ starts, uint64_t n, uint32_t K, mki::SegRes *__restrict__ res,
                 const mki::Seg *__restrict__ segs, uint64_t win_off, uint16_t *__restrict__ sym,
                 uint32_t *__restrict__ bad, mki::Recorder rec)
{
    const uint64_t i = (uint64_t)blockIdx.x * DEC_WARPS + (threadIdx.x >> 5);
    if (i >= n || (threadIdx.x & 31u))
        return;
    mki::Tables t;
    if (!segs) {
        res[i] = mki::decode_segment_t<true>(gz, gz_len, starts[i], cand, n_cand, K, nullptr, 0, 0, &t, &rec);
        return;
    }
    const mki::Seg s = segs[i];
    const mki::SegRes r = mki::decode_segment_t<true>(gz, gz_len, s.start, cand, n_cand, mki::NO_LIMIT,
                                                      sym + (s.out_off - win_off), s.out_len, s.member_pos, &t, nullptr);
    if (r.status != (s.final ? mki::SEG_FINAL : mki::SEG_CAND) || r.end != s.end || r.out_len != s.out_len)
        atomicOr(bad, 1u);
}

__global__ void __launch_bounds__(1024) k_gz_resolve(uint16_t *__restrict__ sym, const uint8_t *__restrict__ hist,
                                                     const mki::Seg *__restrict__ segs, uint64_t n, uint64_t win_off)
{
    for (uint64_t i = 0; i < n; ++i) {
        mki::resolve_segment_tail(sym, hist, segs[i].out_off - win_off, segs[i].out_len, threadIdx.x, blockDim.x);
        __syncthreads();
    }
}

// seg_off[k] = window offset of segment k (ascending); markers find their segment by binary search
__global__ void k_gz_narrow(const uint16_t *__restrict__ sym, const uint8_t *__restrict__ hist,
                            const uint64_t *__restrict__ seg_off, uint64_t n_seg, uint64_t len, uint8_t *__restrict__ out)
{
    for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < len; p += (uint64_t)gridDim.x * blockDim.x) {
        const uint16_t v = sym[p];
        uint64_t o = 0;
        if (v & mki::MARK) {
            uint64_t lo = 0, hi = n_seg; // last k with seg_off[k] <= p
            while (hi - lo > 1) {
                const uint64_t mid = (lo + hi) / 2;
                if (seg_off[mid] <= p)
                    lo = mid;
                else
                    hi = mid;
            }
            o = seg_off[lo];
        }
        out[p] = mki::resolve_symbol(sym, hist, o, v);
    }
}

// the 32 KiB of output before the next window: the tail of (hist || window)
__global__ void k_gz_hist(const uint8_t *__restrict__ hist, const uint8_t *__restrict__ out, uint64_t len,
                          uint8_t *__restrict__ next)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < mki::WSIZE; i += gridDim.x * blockDim.x) {
        const int64_t q = (int64_t)len - (int64_t)mki::WSIZE + i;
        next[i] = q >= 0 ? out[q] : hist[mki::WSIZE + q];
    }
}

struct Window {
    uint64_t seg0, seg1;     // segments [seg0, seg1)
    uint64_t out_off, len;   // decompressed range
};

} // namespace gz

struct mksnap_gunzip_state {
    Stream s; // the gunzip's own stream: window decodes do not queue behind an open ingest session (declared first, so
              // destroyed after the buffers and events used on it)
    DevBuf<uint8_t> d_gz;
    uint64_t gz_len = 0;
    DevBuf<uint64_t> d_cand;
    uint64_t n_cand = 0;
    DevBuf<mki::SegRes> d_res;
    DevBuf<mki::Seg> d_segs;
    DevBuf<uint64_t> d_seg_off;
    DevBuf<uint16_t> d_sym;
    DevBuf<uint8_t> d_out;
    PinnedBuf<uint8_t> h_out; // pinned copy of the decoded window: reads are host copies, one D2H per window
    DevBuf<uint8_t> d_hist[2];
    int hist_cur = 0;
    DevBuf<CrcExtent> d_ext;
    DevBuf<uint32_t> d_pb, d_pure, d_bad; // piece bases, pure(extent), flags
    std::vector<mki::Seg> segs;
    std::vector<mki::Member> mems;
    std::vector<gz::Window> wins;
    std::vector<uint32_t> mem_pure; // running pure CRC of each member
    uint64_t next_win = 0;          // next window to decode
    uint64_t win_end = 0;           // decompressed offset where the current window ends
    uint64_t pos = 0;               // decompressed bytes handed out
    uint64_t fail_at = UINT64_MAX;  // the read that reaches this offset fails: a member with a bad trailer ends there
    bool broken = false;            // a window failed to decode: every later read fails
    bool indexed = false;           // opened by mksnap_gunzip_open_indexed: bit positions, k_gz_decode_bits
    std::vector<uint64_t> index;    // ... and the points mksnap_gunzip_get_index returns
    mksnap_gunzip_index_info idx{};
    mksnap_gunzip_times times{};
    Event ev[6];
};

namespace {

void gz_free(mksnap *h)
{
    mksnap_gunzip_state *g = h->gz;
    if (!g)
        return;
    if (g->s)
        cudaStreamSynchronize(g->s);
    delete g;
    h->gz = nullptr;
}

float gz_ms(mksnap_gunzip_state *g, int a, int b)
{
    float t = 0;
    cudaEventElapsedTime(&t, g->ev[a], g->ev[b]);
    return t;
}

// the body of mksnap_gunzip_open; on failure the caller frees the state
int gz_open(mksnap *h, mksnap_gunzip_state *g, const uint8_t *gz, uint64_t gz_len, const uint64_t *points,
            uint64_t n_points, mksnap_gunzip_info *info)
{
    // candidate counts and their scan are 32-bit: flush points alone are at most gz_len / 4 + 1; a blob whose member
    // headers push the total past that is refused after the count (MKSNAP_E_CAPACITY)
    if (gz_len / 4 + 2 > 0xFFFFFFFFull)
        return fail(h, MKSNAP_E_CAPACITY, "gunzip: blob of %llu bytes exceeds the 16 GiB limit", (unsigned long long)gz_len);
    CK(h, cudaStreamCreateWithFlags(g->s.put(), cudaStreamNonBlocking));
    const cudaStream_t s = g->s;
    for (Event &e : g->ev)
        CK(h, cudaEventCreate(e.put()));
    mki::LinkState st;
    if (mki::link_start(&st, gz, gz_len) != mki::LINK_NEXT)
        return fail(h, MKSNAP_E_DATA, "gunzip: no gzip member header at offset 0");
    // the candidate scan uses the handle's scan scratch: start after the work already queued on the session stream
    CK(h, cudaEventRecord(g->ev[5], h->s_comp));
    CK(h, cudaStreamWaitEvent(s, g->ev[5], 0));
    g->gz_len = gz_len;
    CK(h, g->d_gz.alloc(gz_len));
    CK(h, cudaMemcpyAsync(g->d_gz, gz, gz_len, cudaMemcpyHostToDevice, s));
    h->stats.h2d_bytes += gz_len;

    // K5a: candidates after the first body start, which is candidate 0
    const uint64_t from = st.pos, to = gz_len;
    const uint64_t n_chunks = (to - from + gz::SCAN_CHUNK - 1) / gz::SCAN_CHUNK;
    if (n_chunks > 0xFFFFFFF0ull)
        return fail(h, MKSNAP_E_CAPACITY, "gunzip: blob too large");
    const uint64_t n_hchunks = (gz_len + gz::SCAN_CHUNK - 1) / gz::SCAN_CHUNK, body_words = gz_len / 32 + 1;
    DevBuf<uint32_t> d_cnt, d_body;
    DevBuf<unsigned long long> d_tot; // the 64-bit candidate total
    CK(h, d_cnt.alloc(n_chunks + 1));
    CK(h, d_body.alloc(body_words));
    CK(h, d_tot.alloc(1));
    CK(h, cudaMemsetAsync(d_cnt, 0, (n_chunks + 1) * 4, s));
    CK(h, cudaMemsetAsync(d_body, 0, body_words * 4, s));
    CK(h, cudaMemsetAsync(d_tot, 0, 8, s));
    CK(h, cudaEventRecord(g->ev[0], s));
    const uint32_t tb = 256, nb = (uint32_t)((n_chunks + tb - 1) / tb);
    if (n_chunks) {
        gz::k_gz_scan_headers<<<(uint32_t)((n_hchunks + tb - 1) / tb), tb, 0, s>>>(g->d_gz, gz_len, from, d_body,
                                                                                  (uint32_t)n_hchunks);
        LAUNCH_OK(h);
        gz::k_gz_scan_count<<<nb, tb, 0, s>>>(g->d_gz, from, to, d_body, d_cnt, (uint32_t)n_chunks, d_tot);
        LAUNCH_OK(h);
    }
    // exclusive scan over n_chunks + 1 entries: the last one is the total
    uint64_t scan_words = 0;
    {
        uint64_t n = n_chunks + 1;
        while (n > SCAN_ITEMS) {
            n = (n + SCAN_ITEMS - 1) / SCAN_ITEMS;
            scan_words += n;
        }
    }
    if (scan_words > h->d_scan_tmp.size())
        return fail(h, MKSNAP_E_CAPACITY, "gunzip: blob too large for the scan scratch of this handle");
    int rc = scan_u32(h, d_cnt, d_cnt, n_chunks + 1, s);
    uint32_t total = 0;
    unsigned long long total64 = 0;
    if (rc == 0 && cudaMemcpyAsync(&total, d_cnt + n_chunks, 4, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
        cudaMemcpyAsync(&total64, d_tot, 8, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
        cudaStreamSynchronize(s) == cudaSuccess) {
        g->n_cand = (uint64_t)total + 1;
        if (total64 != total || total64 + 2 > 0xFFFFFFFFull)
            rc = fail(h, MKSNAP_E_CAPACITY, "gunzip: %llu candidate starts exceed the 32-bit candidate scan", total64);
        else if (g->d_cand.alloc(g->n_cand) != cudaSuccess ||
                 cudaMemcpyAsync(g->d_cand, &st.pos, 8, cudaMemcpyHostToDevice, s) != cudaSuccess)
            rc = fail(h, MKSNAP_E_NOMEM, "gunzip: candidate table of %llu rows", (unsigned long long)g->n_cand);
        else if (n_chunks) {
            gz::k_gz_scan_write<<<nb, tb, 0, s>>>(g->d_gz, from, to, d_body, d_cnt, (uint32_t)n_chunks, g->d_cand);
            h->stats.kernel_launches++;
        }
    } else if (rc == 0) {
        rc = fail(h, MKSNAP_E_CUDA, "gunzip: candidate scan: %s", cudaGetErrorString(cudaGetLastError()));
    }
    cudaStreamSynchronize(s);
    if (rc)
        return rc;
    CK(h, cudaGetLastError());
    d_body.reset(); // the bitmap is not needed past the scan: keep it out of the count pass's peak

    // indexed open: the candidates become bit offsets, merged with the caller's points
    std::vector<uint64_t> byte_cand, bit_cand;
    DevBuf<mki::Rec> rec;
    DevBuf<unsigned long long> rec_n;
    mki::Recorder recorder{nullptr, nullptr, mki::REC_CAP};
    if (g->indexed) {
        byte_cand.resize(g->n_cand);
        CK(h, cudaMemcpyAsync(byte_cand.data(), g->d_cand, g->n_cand * 8, cudaMemcpyDeviceToHost, s));
        CK(h, cudaStreamSynchronize(s));
        bit_cand = mki::merge_points(byte_cand, points, n_points);
        g->n_cand = bit_cand.size();
        if (g->d_cand.alloc(g->n_cand) != cudaSuccess)
            return fail(h, MKSNAP_E_NOMEM, "gunzip: candidate table of %llu rows", (unsigned long long)g->n_cand);
        CK(h, cudaMemcpyAsync(g->d_cand, bit_cand.data(), g->n_cand * 8, cudaMemcpyHostToDevice, s));
        CK(h, rec.alloc(mki::REC_CAP));
        CK(h, rec_n.alloc(1));
        CK(h, cudaMemsetAsync(rec_n, 0, 8, s));
        recorder.buf = rec;
        recorder.n = rec_n;
        st.pos *= 8;
    }
    CK(h, cudaEventRecord(g->ev[1], s));

    // K5b count mode over every candidate
    CK(h, g->d_res.alloc(g->n_cand));
    const uint64_t dgrid = (g->n_cand + gz::DEC_WARPS - 1) / gz::DEC_WARPS;
    if (g->indexed)
        gz::k_gz_decode_bits<<<(uint32_t)dgrid, 32 * gz::DEC_WARPS, 0, s>>>(
            g->d_gz, gz_len, g->d_cand, g->n_cand, g->d_cand, g->n_cand, mki::K_PASS, g->d_res, nullptr, 0, nullptr,
            nullptr, recorder);
    else
        gz::k_gz_decode<<<(uint32_t)dgrid, 32 * gz::DEC_WARPS, 0, s>>>(g->d_gz, gz_len, g->d_cand, g->n_cand, g->d_cand,
                                                                      g->n_cand, mki::K_PASS, g->d_res, nullptr, 0,
                                                                      nullptr, nullptr);
    LAUNCH_OK(h);
    CK(h, cudaEventRecord(g->ev[2], s));
    std::vector<uint64_t> cand(g->n_cand);
    std::vector<mki::SegRes> res(g->n_cand);
    CK(h, cudaMemcpyAsync(cand.data(), g->d_cand, g->n_cand * 8, cudaMemcpyDeviceToHost, s));
    CK(h, cudaMemcpyAsync(res.data(), g->d_res, g->n_cand * sizeof(mki::SegRes), cudaMemcpyDeviceToHost, s));
    CK(h, cudaStreamSynchronize(s));
    h->stats.d2h_bytes += g->n_cand * (8 + sizeof(mki::SegRes));
    g->times.ms_scan += gz_ms(g, 0, 1);
    g->times.ms_count += gz_ms(g, 1, 2);

    // link: follow the true chain; starts without a usable count result are decoded again without the K limit
    DevBuf<uint64_t> d_one; // the start and result of such a decode
    DevBuf<mki::SegRes> d_one_res;
    const auto redecode = [&](uint64_t pos, mki::SegRes *r) -> int {
        if (!d_one_res) {
            CK(h, d_one.alloc(1));
            CK(h, d_one_res.alloc(1));
        }
        CK(h, cudaMemcpyAsync(d_one, &pos, 8, cudaMemcpyHostToDevice, s));
        CK(h, cudaEventRecord(g->ev[1], s));
        if (g->indexed)
            gz::k_gz_decode_bits<<<1, 32, 0, s>>>(g->d_gz, gz_len, g->d_cand, g->n_cand, d_one, 1, mki::NO_LIMIT,
                                                  d_one_res, nullptr, 0, nullptr, nullptr, recorder);
        else
            gz::k_gz_decode<<<1, 32, 0, s>>>(g->d_gz, gz_len, g->d_cand, g->n_cand, d_one, 1, mki::NO_LIMIT,
                                             d_one_res, nullptr, 0, nullptr, nullptr);
        LAUNCH_OK(h);
        CK(h, cudaEventRecord(g->ev[2], s));
        CK(h, cudaMemcpyAsync(r, d_one_res, sizeof *r, cudaMemcpyDeviceToHost, s));
        CK(h, cudaStreamSynchronize(s));
        g->times.ms_count += gz_ms(g, 1, 2);
        g->times.extra_decodes++;
        return 0;
    };
    const int lk = g->indexed ? mki::link_all<true>(&st, cand.data(), res.data(), g->n_cand, gz, gz_len, redecode,
                                                    &g->segs, &g->mems)
                              : mki::link_all<false>(&st, cand.data(), res.data(), g->n_cand, gz, gz_len, redecode,
                                                     &g->segs, &g->mems);
    if (lk == mki::LINK_ERR)
        return fail(h, MKSNAP_E_DATA, "gunzip: malformed data in member %u (compressed offset %llu)", st.member,
                    (unsigned long long)(g->indexed ? st.pos / 8 : st.pos));
    if (lk != mki::LINK_DONE)
        return lk;
    g->d_res.reset(); // the count results are not needed past the link: keep them out of the windows' peak
    if (g->indexed) { // cut long segments at the records of their decode; the cuts join the write candidates
        unsigned long long n_rec = 0;
        CK(h, cudaMemcpyAsync(&n_rec, rec_n, 8, cudaMemcpyDeviceToHost, s));
        CK(h, cudaStreamSynchronize(s));
        std::vector<mki::Rec> recs(std::min<uint64_t>(n_rec, mki::REC_CAP));
        CK(h, cudaMemcpyAsync(recs.data(), rec, recs.size() * sizeof(mki::Rec), cudaMemcpyDeviceToHost, s));
        CK(h, cudaStreamSynchronize(s));
        h->stats.d2h_bytes += recs.size() * sizeof(mki::Rec);
        const mki::IndexCounts c = mki::split_segments(&g->segs, std::move(recs), &cand, byte_cand, points, n_points,
                                                       &g->index);
        g->idx = mksnap_gunzip_index_info{n_points, c.linked, c.recorded, g->index.size()};
        if (c.recorded) {
            g->n_cand = cand.size();
            if (g->d_cand.alloc(g->n_cand) != cudaSuccess)
                return fail(h, MKSNAP_E_NOMEM, "gunzip: candidate table of %llu rows", (unsigned long long)g->n_cand);
            CK(h, cudaMemcpyAsync(g->d_cand, cand.data(), g->n_cand * 8, cudaMemcpyHostToDevice, s));
        }
    }

    // windows of whole segments
    uint64_t max_seg = 0, max_mem_per_win = 1;
    for (uint64_t k = 0; k < g->segs.size();) {
        gz::Window w{k, k, g->segs[k].out_off, 0};
        uint32_t mems_in = 1;
        while (w.seg1 < g->segs.size() && (w.seg1 == k || w.len + g->segs[w.seg1].out_len <= gz::GZ_WINDOW)) {
            if (w.seg1 > k && g->segs[w.seg1].member != g->segs[w.seg1 - 1].member)
                ++mems_in;
            w.len += g->segs[w.seg1].out_len;
            max_seg = std::max(max_seg, g->segs[w.seg1].out_len);
            ++w.seg1;
        }
        max_mem_per_win = std::max<uint64_t>(max_mem_per_win, mems_in);
        g->wins.push_back(w);
        k = w.seg1;
    }
    const uint64_t win_cap = std::max(gz::GZ_WINDOW, max_seg);
    CK(h, g->d_segs.alloc(g->segs.size()));
    CK(h, cudaMemcpyAsync(g->d_segs, g->segs.data(), g->segs.size() * sizeof(mki::Seg), cudaMemcpyHostToDevice, s));
    CK(h, g->d_seg_off.alloc(g->segs.size()));
    CK(h, g->d_sym.alloc(win_cap + 32));
    CK(h, g->d_out.alloc(win_cap + 64)); // K0 reads up to 16 bytes past an extent
    CK(h, g->h_out.alloc(win_cap));
    for (int k = 0; k < 2; ++k)
        CK(h, g->d_hist[k].alloc(mki::WSIZE));
    CK(h, cudaMemsetAsync(g->d_hist[0], 0, mki::WSIZE, s));
    const uint64_t ext_cap = 2 * max_mem_per_win;
    CK(h, g->d_ext.alloc(ext_cap));
    CK(h, g->d_pb.alloc(ext_cap + 1));
    CK(h, g->d_pure.alloc(ext_cap + 1)); // the last word takes K0's stream accumulator
    CK(h, g->d_bad.alloc(1));
    CK(h, cudaStreamSynchronize(s));
    g->mem_pure.assign(g->mems.size(), 0);

    info->gz_bytes = gz_len;
    info->out_bytes = st.out;
    info->n_members = g->mems.size();
    info->n_segments = g->segs.size();
    return 0;
}

// decode window g->next_win into h_out and check the trailers of the members that end in it; any error leaves the
// gunzip broken (gz_window)
int gz_window_impl(mksnap *h, mksnap_gunzip_state *g)
{
    const cudaStream_t s = g->s;
    const gz::Window w = g->wins[g->next_win++];
    const uint64_t n = w.seg1 - w.seg0;
    std::vector<uint64_t> off(n);
    for (uint64_t k = 0; k < n; ++k)
        off[k] = g->segs[w.seg0 + k].out_off - w.out_off;
    CK(h, cudaMemcpyAsync(g->d_seg_off, off.data(), n * 8, cudaMemcpyHostToDevice, s));
    CK(h, cudaMemsetAsync(g->d_bad, 0, 4, s));
    CK(h, cudaEventRecord(g->ev[0], s));
    const uint32_t dgrid = (uint32_t)((n + gz::DEC_WARPS - 1) / gz::DEC_WARPS);
    if (g->indexed)
        gz::k_gz_decode_bits<<<dgrid, 32 * gz::DEC_WARPS, 0, s>>>(g->d_gz, g->gz_len, g->d_cand, g->n_cand, nullptr, n,
                                                                  mki::NO_LIMIT, nullptr, g->d_segs + w.seg0, w.out_off,
                                                                  g->d_sym, g->d_bad, mki::Recorder{nullptr, nullptr, 0});
    else
        gz::k_gz_decode<<<dgrid, 32 * gz::DEC_WARPS, 0, s>>>(g->d_gz, g->gz_len, g->d_cand, g->n_cand, nullptr, n,
                                                             mki::NO_LIMIT, nullptr, g->d_segs + w.seg0, w.out_off,
                                                             g->d_sym, g->d_bad);
    LAUNCH_OK(h);
    CK(h, cudaEventRecord(g->ev[1], s));
    const uint8_t *hist = g->d_hist[g->hist_cur];
    gz::k_gz_resolve<<<1, 1024, 0, s>>>(g->d_sym, hist, g->d_segs + w.seg0, n, w.out_off);
    LAUNCH_OK(h);
    CK(h, cudaEventRecord(g->ev[2], s));
    if (w.len) {
        const uint32_t grid = (uint32_t)std::min<uint64_t>((w.len + 255) / 256, (uint64_t)h->sm_count * 16);
        gz::k_gz_narrow<<<grid, 256, 0, s>>>(g->d_sym, hist, g->d_seg_off, n, w.len, g->d_out);
        LAUNCH_OK(h);
    }
    gz::k_gz_hist<<<32, 256, 0, s>>>(hist, g->d_out, w.len, g->d_hist[1 - g->hist_cur]);
    LAUNCH_OK(h);
    g->hist_cur = 1 - g->hist_cur;
    CK(h, cudaEventRecord(g->ev[3], s));

    // CRC-32 of every member piece [a, b) of the window with K0: extents [a16, b) and [a16, a), a16 = a rounded down
    // to 16 (K0 wants 16-byte aligned extents); pure([a, b)) = pure([a16, b)) ^ pure([a16, a)) * x^(8 (b - a))
    struct Piece {
        uint32_t member;
        uint64_t a, b;
    };
    std::vector<Piece> pcs;
    for (uint64_t k = w.seg0; k < w.seg1; ++k) {
        const mki::Seg &sg = g->segs[k];
        const uint64_t a = sg.out_off - w.out_off, b = a + sg.out_len;
        if (!pcs.empty() && pcs.back().member == sg.member)
            pcs.back().b = b;
        else
            pcs.push_back(Piece{sg.member, a, b});
    }
    std::vector<CrcExtent> ext;
    std::vector<uint32_t> pb;
    uint64_t pieces = 0;
    for (const Piece &p : pcs) {
        const uint64_t a16 = p.a & ~15ull;
        ext.push_back(CrcExtent{a16, p.b - a16, 0});
        ext.push_back(CrcExtent{a16, p.a - a16, 0});
    }
    for (const CrcExtent &e : ext) {
        pb.push_back((uint32_t)pieces);
        pieces += (e.len + CRC_PIECE - 1) / CRC_PIECE;
    }
    pb.push_back((uint32_t)pieces);
    std::vector<uint32_t> pure(ext.size(), 0);
    if (pieces) {
        CK(h, cudaMemcpyAsync(g->d_ext, ext.data(), ext.size() * sizeof(CrcExtent), cudaMemcpyHostToDevice, s));
        CK(h, cudaMemcpyAsync(g->d_pb, pb.data(), pb.size() * 4, cudaMemcpyHostToDevice, s));
        CK(h, cudaMemsetAsync(g->d_pure, 0, (ext.size() + 1) * 4, s));
        const uint32_t grid = (uint32_t)std::min<uint64_t>(h->sm_count, (pieces + 31) / 32);
        k_crc32_extents<<<grid, CRC_THREADS, CRC_SMEM, s>>>(g->d_out, g->d_ext, g->d_pb, (uint32_t)ext.size(),
                                                            (uint32_t)pieces, h->d_consts, g->d_pure,
                                                            g->d_pure + ext.size(), nullptr);
        LAUNCH_OK(h);
        CK(h, cudaMemcpyAsync(pure.data(), g->d_pure, ext.size() * 4, cudaMemcpyDeviceToHost, s));
    }
    CK(h, cudaEventRecord(g->ev[4], s));
    CK(h, cudaMemcpyAsync(g->h_out, g->d_out, w.len, cudaMemcpyDeviceToHost, s));
    h->stats.d2h_bytes += w.len;
    uint32_t bad = 0;
    CK(h, cudaMemcpyAsync(&bad, g->d_bad, 4, cudaMemcpyDeviceToHost, s));
    CK(h, cudaStreamSynchronize(s));
    g->times.ms_write += gz_ms(g, 0, 1);
    g->times.ms_resolve += gz_ms(g, 1, 3);
    g->times.ms_crc += gz_ms(g, 3, 4);
    if (bad) {
        return fail(h, MKSNAP_E_DATA, "gunzip: malformed data (a distance reaches before the start of its member)");
    }
    const uint64_t M = 0xFFFFFFFFull;
    for (size_t k = 0; k < pcs.size(); ++k) {
        const Piece &p = pcs[k];
        const uint64_t L = p.b - p.a;
        const uint32_t pp = pure[2 * k] ^ crc_mulmod(pure[2 * k + 1], xpow_bits(((L % M) * 8ull) % M));
        g->mem_pure[p.member] = crc_mulmod(g->mem_pure[p.member], xpow_bits(((L % M) * 8ull) % M)) ^ pp;
    }
    // members that end in this window: the last segment of the member is in it
    for (uint64_t k = w.seg0; k < w.seg1; ++k) {
        const mki::Seg &sg = g->segs[k];
        if (!sg.final)
            continue;
        const mki::Member &m = g->mems[sg.member];
        const uint32_t crc = g->mem_pure[sg.member] ^
                             crc_mulmod(0xFFFFFFFFu, xpow_bits(((m.out_len % M) * 8ull) % M)) ^ 0xFFFFFFFFu;
        if ((crc != m.crc || (uint32_t)m.out_len != m.isize) && m.out_off + m.out_len < g->fail_at)
            g->fail_at = m.out_off + m.out_len;
    }
    g->win_end = w.out_off + w.len;
    return 0;
}

int gz_window(mksnap *h, mksnap_gunzip_state *g)
{
    const int rc = gz_window_impl(h, g);
    if (rc) {
        g->broken = true;
        cudaGetLastError();
    }
    return rc;
}

} // namespace

namespace {

int gz_open_entry(mksnap_t *h, const void *gz, uint64_t gz_len, const uint64_t *points, uint64_t n_points, bool indexed,
                  mksnap_gunzip_info *info)
{
    if (h->gz)
        return fail(h, MKSNAP_E_STATE, "gunzip: already open (close it first)");
    CK(h, cudaSetDevice(h->cfg.device));
    memset(info, 0, sizeof *info);
    h->gz = new mksnap_gunzip_state();
    h->gz->indexed = indexed;
    const int rc = gz_open(h, h->gz, (const uint8_t *)gz, gz_len, points, n_points, info);
    if (rc) {
        gz_free(h);
        cudaGetLastError();
        memset(info, 0, sizeof *info);
    }
    return rc;
}

} // namespace

int mksnap_gunzip_open(mksnap_t *h, const void *gz, uint64_t gz_len, mksnap_gunzip_info *info)
{
    if (!h || (!gz && gz_len) || !info)
        return MKSNAP_E_INVAL;
    return gz_open_entry(h, gz, gz_len, nullptr, 0, false, info);
}

int mksnap_gunzip_open_indexed(mksnap_t *h, const void *gz, uint64_t gz_len, const uint64_t *points,
                               uint64_t n_points, mksnap_gunzip_info *info)
{
    if (!h || (!gz && gz_len) || !info || (!points && n_points))
        return MKSNAP_E_INVAL;
    for (uint64_t k = 0; k < n_points; ++k)
        if (points[k] / 8 >= gz_len || (k && points[k] <= points[k - 1]))
            return fail(h, MKSNAP_E_INVAL, "gunzip: index point %llu (bit %llu) is out of order or past the blob",
                        (unsigned long long)k, (unsigned long long)points[k]);
    return gz_open_entry(h, gz, gz_len, points, n_points, true, info);
}

int mksnap_gunzip_get_index(mksnap_t *h, uint64_t *points, uint64_t cap, mksnap_gunzip_index_info *out)
{
    if (!h || !out || (!points && cap))
        return MKSNAP_E_INVAL;
    if (!h->gz)
        return fail(h, MKSNAP_E_STATE, "gunzip: not open");
    if (!h->gz->indexed)
        return fail(h, MKSNAP_E_STATE, "gunzip: not opened by mksnap_gunzip_open_indexed");
    *out = h->gz->idx;
    std::copy_n(h->gz->index.begin(), std::min<uint64_t>(cap, h->gz->index.size()), points);
    return 0;
}

int mksnap_gunzip_read(mksnap_t *h, void *dst, uint64_t cap, uint64_t *got)
{
    if (!h || !got || (!dst && cap))
        return MKSNAP_E_INVAL;
    *got = 0;
    mksnap_gunzip_state *g = h->gz;
    if (!g)
        return fail(h, MKSNAP_E_STATE, "gunzip: not open");
    CK(h, cudaSetDevice(h->cfg.device));
    uint8_t *d = (uint8_t *)dst;
    while (*got < cap) {
        if (g->broken)
            return fail(h, MKSNAP_E_DATA, "gunzip: malformed data");
        if (g->pos >= g->fail_at)
            return fail(h, MKSNAP_E_DATA, "gunzip: CRC-32 or length mismatch in a member trailer");
        if (g->pos == g->win_end) {
            if (g->next_win == g->wins.size())
                break;
            const int rc = gz_window(h, g);
            if (rc)
                return rc;
            continue;
        }
        const uint64_t w0 = g->wins[g->next_win - 1].out_off;
        const uint64_t n = std::min({cap - *got, g->win_end - g->pos, g->fail_at - g->pos});
        memcpy(d + *got, g->h_out + (g->pos - w0), n);
        g->pos += n;
        *got += n;
    }
    // the member that ends exactly here has a bad trailer, or the windows still to decode end the stream with one
    if (g->pos >= g->fail_at)
        return fail(h, MKSNAP_E_DATA, "gunzip: CRC-32 or length mismatch in a member trailer");
    return 0;
}

int mksnap_gunzip_close(mksnap_t *h)
{
    if (!h)
        return MKSNAP_E_INVAL;
    CK(h, cudaSetDevice(h->cfg.device));
    gz_free(h);
    return 0;
}

int mksnap_gunzip_get_times(mksnap_t *h, mksnap_gunzip_times *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    if (!h->gz)
        return fail(h, MKSNAP_E_STATE, "gunzip: not open");
    *out = h->gz->times;
    return 0;
}
