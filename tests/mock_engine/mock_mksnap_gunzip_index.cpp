// mock_mksnap_gunzip_index.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock of mock_mksnap_defer.cpp (gunzip and deferred
// streams, so that runs of layers ingest on it) plus the indexed open (mksnap_gunzip_open_indexed,
// mksnap_gunzip_get_index).  The open runs what mksnap_inflate.cuh runs for it, from mksnap_inflate_core.h: the scanned candidates merged with the points (mki::merge_points), count decodes
// at bit granularity that record block starts (decode_segment_t<true>, mki::Recorder), the link over bit positions
// (link_feed<true>) and the cut of long segments at the records (mki::split_segments).  Windows, reads, resolve and
// trailer checks are the base mock's; its write decodes call mki::decode_segment, which this file routes to the
// bit-granular decoder while a read of an indexed gunzip runs.  An indexed gunzip is closed before its handle is
// destroyed (the tests always close).
// tests/test_host_gunzip_index_cpu.py builds this file (also with ASan/UBSan) and loads it with RTLD_GLOBAL before
// libmkhost.
#include "../../makisu_b200/csrc/mksnap_inflate_core.h"

namespace mki {
bool g_bits_mode = false; // set while a read of an indexed gunzip runs

inline SegRes decode_segment_sel(const uint8_t *gz, uint64_t gz_len, uint64_t start, const uint64_t *cand,
                                 uint64_t n_cand, uint32_t K, uint16_t *out, uint64_t out_cap, uint64_t member_pos,
                                 Tables *t)
{
    return g_bits_mode ? decode_segment_t<true>(gz, gz_len, start, cand, n_cand, K, out, out_cap, member_pos, t, nullptr)
                       : decode_segment_t<false>(gz, gz_len, start, cand, n_cand, K, out, out_cap, member_pos, t, nullptr);
}
} // namespace mki

#define decode_segment decode_segment_sel
#define mksnap_gunzip_read mock_base_gunzip_read
#define mksnap_gunzip_close mock_base_gunzip_close
#include "mock_mksnap_defer.cpp"
#undef mksnap_gunzip_close
#undef mksnap_gunzip_read
#undef decode_segment

namespace {

struct MockIndex {
    std::vector<uint64_t> points;
    mksnap_gunzip_index_info info{};
};
std::map<const mksnap *, MockIndex> g_index; // handles with an indexed gunzip open
uint64_t g_records = 0;                      // records the count decodes of the last indexed open offered

int gz_open_indexed(mksnap *h, MockGz &g, const uint64_t *points, uint64_t n_points, mksnap_gunzip_info *info,
                    MockIndex *ix)
{
    mki::LinkState st;
    if (mki::link_start<true>(&st, g.gz.data(), g.gz.size()) != mki::LINK_NEXT)
        return fail(h, MKSNAP_E_DATA, "gunzip: no gzip member header at offset 0");
    const uint64_t body0 = st.pos / 8;
    std::vector<uint8_t> member(g.gz.size() + 1, 0); // k_gz_scan_*
    for (uint64_t q = 0; q < g.gz.size(); ++q) {
        const int64_t p = mki::member_body(g.gz.data(), g.gz.size(), q);
        if (p > (int64_t)body0)
            member[p] = 1;
    }
    std::vector<uint64_t> byte_cand{body0};
    for (uint64_t p = body0 + 1; p <= g.gz.size(); ++p)
        if (member[p] || mki::flush_end(g.gz.data(), p))
            byte_cand.push_back(p);
    g.cand = mki::merge_points(byte_cand, points, n_points);
    std::vector<mki::Rec> recs(mki::REC_CAP);
    unsigned long long n_rec = 0;
    const mki::Recorder rec{recs.data(), &n_rec, mki::REC_CAP};
    std::vector<mki::SegRes> res(g.cand.size());
    mki::Tables t;
    g_consumed = 0;
    g_candidates = g.cand.size();
    for (size_t i = 0; i < g.cand.size(); ++i) { // k_gz_decode_bits, count mode
        res[i] = mki::decode_segment_t<true>(g.gz.data(), g.gz.size(), g.cand[i], g.cand.data(), g.cand.size(),
                                             mki::K_PASS, nullptr, 0, 0, &t, &rec);
        g_consumed += res[i].consumed;
    }
    for (;;) { // link
        const uint64_t i = mki::upper_bound(g.cand.data(), g.cand.size(), st.pos);
        mki::SegRes r;
        if (i > 0 && g.cand[i - 1] == st.pos && res[i - 1].status != mki::SEG_SUSPEND) {
            r = res[i - 1];
        } else {
            r = mki::decode_segment_t<true>(g.gz.data(), g.gz.size(), st.pos, g.cand.data(), g.cand.size(),
                                            mki::NO_LIMIT, nullptr, 0, 0, &t, &rec);
            g.times.extra_decodes++;
        }
        mki::Seg seg;
        mki::Member mem;
        bool ended = false;
        const int lk = mki::link_feed<true>(&st, r, g.gz.data(), g.gz.size(), &seg, &mem, &ended);
        if (lk == mki::LINK_ERR)
            return fail(h, MKSNAP_E_DATA, "gunzip: malformed data in member " + std::to_string(st.member));
        g.segs.push_back(seg);
        if (ended)
            g.mems.push_back(mem);
        if (lk == mki::LINK_DONE)
            break;
    }
    g_records = n_rec;
    recs.resize(std::min<uint64_t>(n_rec, mki::REC_CAP));
    const mki::IndexCounts c = mki::split_segments(&g.segs, std::move(recs), &g.cand, byte_cand, points, n_points,
                                                   &ix->points);
    ix->info = mksnap_gunzip_index_info{n_points, c.linked, c.recorded, ix->points.size()};
    for (uint64_t k = 0; k < g.segs.size();) {
        uint64_t e = k, len = 0;
        while (e < g.segs.size() && (e == k || len + g.segs[e].out_len <= MOCK_WINDOW))
            len += g.segs[e++].out_len;
        g.wins.emplace_back(k, e);
        k = e;
    }
    g.mem_crc.assign(g.mems.size(), 0);
    info->gz_bytes = g.gz.size();
    info->out_bytes = st.out;
    info->n_members = g.mems.size();
    info->n_segments = g.segs.size();
    return 0;
}

} // namespace

extern "C" {

// records offered by the count decodes of the last indexed open (before the capacity)
uint64_t mock_gunzip_records(void) { return g_records; }

// the segments of the open gunzip: start and end (bit offsets after an indexed open), decompressed length
uint64_t mock_gunzip_segments(const mksnap_t *h, uint64_t *start, uint64_t *end, uint64_t *out_len, uint64_t cap)
{
    auto it = g_gz.find(h);
    if (it == g_gz.end())
        return 0;
    const auto &s = it->second.segs;
    for (uint64_t k = 0; k < std::min<uint64_t>(cap, s.size()); ++k) {
        start[k] = s[k].start;
        end[k] = s[k].end;
        out_len[k] = s[k].out_len;
    }
    return s.size();
}

int mksnap_gunzip_open_indexed(mksnap_t *h, const void *gz, uint64_t gz_len, const uint64_t *points,
                               uint64_t n_points, mksnap_gunzip_info *info)
{
    if (!h || (!gz && gz_len) || !info || (!points && n_points))
        return MKSNAP_E_INVAL;
    for (uint64_t k = 0; k < n_points; ++k)
        if (points[k] / 8 >= gz_len || (k && points[k] <= points[k - 1]))
            return fail(h, MKSNAP_E_INVAL, "gunzip: index point " + std::to_string(k) + " is out of order or past the blob");
    if (g_gz.count(h))
        return fail(h, MKSNAP_E_STATE, "gunzip: already open (close it first)");
    memset(info, 0, sizeof *info);
    MockGz &g = g_gz[h];
    g.gz.assign((const uint8_t *)gz, (const uint8_t *)gz + gz_len);
    MockIndex ix;
    const int rc = gz_open_indexed(h, g, points, n_points, info, &ix);
    if (rc) {
        g_gz.erase(h);
        memset(info, 0, sizeof *info);
    } else {
        g_index[h] = std::move(ix);
    }
    return rc;
}

int mksnap_gunzip_get_index(mksnap_t *h, uint64_t *points, uint64_t cap, mksnap_gunzip_index_info *out)
{
    if (!h || !out || (!points && cap))
        return MKSNAP_E_INVAL;
    if (!g_gz.count(h))
        return fail(h, MKSNAP_E_STATE, "gunzip: not open");
    auto it = g_index.find(h);
    if (it == g_index.end())
        return fail(h, MKSNAP_E_STATE, "gunzip: not opened by mksnap_gunzip_open_indexed");
    *out = it->second.info;
    std::copy_n(it->second.points.begin(), std::min<uint64_t>(cap, it->second.points.size()), points);
    return 0;
}

int mksnap_gunzip_read(mksnap_t *h, void *dst, uint64_t cap, uint64_t *got)
{
    mki::g_bits_mode = h && g_index.count(h);
    const int rc = mock_base_gunzip_read(h, dst, cap, got);
    mki::g_bits_mode = false;
    return rc;
}

int mksnap_gunzip_close(mksnap_t *h)
{
    if (h)
        g_index.erase(h);
    return mock_base_gunzip_close(h);
}

} // extern "C"
