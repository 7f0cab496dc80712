// mock_mksnap_gunzip.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock engine of mock_mksnap.cpp plus the gunzip entry
// points (mksnap_gunzip_open / _read / _close / _get_times).  Every step runs the engine's own code from
// makisu_b200/csrc/mksnap_inflate_core.h -- speculative count decodes of every candidate start with the K limit, the
// link, write decodes into 16-bit symbols, resolve, trailer checks -- in the order mksnap_inflate.cuh runs it on the
// device, one loop iteration where the device runs one thread.  Windows are small (MOCK_WINDOW) so that CPU-sized blobs
// span several.  tests/test_host_gunzip_cpu.py builds this file (also with ASan/UBSan) and loads it with RTLD_GLOBAL
// before libmkhost.
#define mksnap_destroy mock_base_destroy
#include "mock_mksnap.cpp"
#undef mksnap_destroy
#include "../../makisu_b200/csrc/mksnap_inflate_core.h"

namespace {

constexpr uint64_t MOCK_WINDOW = 256 * 1024;

struct MockGz {
    std::vector<uint8_t> gz;
    std::vector<uint64_t> cand;
    std::vector<mki::Seg> segs;
    std::vector<mki::Member> mems;
    std::vector<std::pair<uint64_t, uint64_t>> wins; // segments [first, second)
    uint64_t next_win = 0, win_off = 0, win_end = 0, pos = 0, fail_at = UINT64_MAX;
    std::vector<uint8_t> out, hist = std::vector<uint8_t>(mki::WSIZE, 0);
    std::vector<uint32_t> mem_crc; // running CRC-32 per member
    bool broken = false;
    mksnap_gunzip_times times{};
};

std::map<const mksnap *, MockGz> g_gz;
uint64_t g_consumed = 0, g_candidates = 0; // count-pass work of the last open

int gz_window(mksnap *h, MockGz &g)
{
    const auto w = g.wins[g.next_win++];
    const mki::Seg &s0 = g.segs[w.first];
    g.win_off = s0.out_off;
    uint64_t len = 0;
    for (uint64_t k = w.first; k < w.second; ++k)
        len += g.segs[k].out_len;
    std::vector<uint16_t> sym(len + 1);
    mki::Tables t;
    for (uint64_t k = w.first; k < w.second; ++k) { // k_gz_decode, write mode
        const mki::Seg &s = g.segs[k];
        const mki::SegRes r = mki::decode_segment(g.gz.data(), g.gz.size(), s.start, g.cand.data(), g.cand.size(),
                                                  mki::NO_LIMIT, sym.data() + (s.out_off - g.win_off), s.out_len,
                                                  s.member_pos, &t);
        if (r.status != (s.final ? mki::SEG_FINAL : mki::SEG_CAND) || r.end != s.end || r.out_len != s.out_len) {
            g.broken = true;
            return fail(h, MKSNAP_E_DATA, "gunzip: malformed data (a distance reaches before the start of its member)");
        }
    }
    for (uint64_t k = w.first; k < w.second; ++k) // k_gz_resolve
        mki::resolve_segment_tail(sym.data(), g.hist.data(), g.segs[k].out_off - g.win_off, g.segs[k].out_len, 0, 1);
    g.out.assign(len, 0);
    for (uint64_t k = w.first; k < w.second; ++k) { // k_gz_narrow
        const uint64_t o = g.segs[k].out_off - g.win_off;
        for (uint64_t j = 0; j < g.segs[k].out_len; ++j)
            g.out[o + j] = mki::resolve_symbol(sym.data(), g.hist.data(), o, sym[o + j]);
    }
    std::vector<uint8_t> nh(mki::WSIZE); // k_gz_hist
    for (uint32_t i = 0; i < mki::WSIZE; ++i) {
        const int64_t q = (int64_t)len - (int64_t)mki::WSIZE + i;
        nh[i] = q >= 0 ? g.out[q] : g.hist[mki::WSIZE + q];
    }
    g.hist.swap(nh);
    for (uint64_t k = w.first; k < w.second; ++k) { // member CRC-32 and trailer checks
        const mki::Seg &s = g.segs[k];
        g.mem_crc[s.member] = mki::crc32_update(g.mem_crc[s.member], g.out.data() + (s.out_off - g.win_off), s.out_len);
        if (!s.final)
            continue;
        const mki::Member &m = g.mems[s.member];
        if ((g.mem_crc[s.member] != m.crc || (uint32_t)m.out_len != m.isize) && m.out_off + m.out_len < g.fail_at)
            g.fail_at = m.out_off + m.out_len;
    }
    g.win_end = g.win_off + len;
    return 0;
}

int gz_open(mksnap *h, MockGz &g, mksnap_gunzip_info *info)
{
    mki::LinkState st;
    if (mki::link_start(&st, g.gz.data(), g.gz.size()) != mki::LINK_NEXT)
        return fail(h, MKSNAP_E_DATA, "gunzip: no gzip member header at offset 0");
    g.cand.push_back(st.pos); // k_gz_scan_*
    for (uint64_t p = st.pos + 1; p <= g.gz.size(); ++p)
        if (p >= 4 && g.gz[p - 1] == 0xFF && g.gz[p - 2] == 0xFF && g.gz[p - 3] == 0 && g.gz[p - 4] == 0)
            g.cand.push_back(p);
    std::vector<mki::SegRes> res(g.cand.size());
    mki::Tables t;
    g_consumed = 0;
    g_candidates = g.cand.size();
    for (size_t i = 0; i < g.cand.size(); ++i) { // k_gz_decode, count mode
        res[i] = mki::decode_segment(g.gz.data(), g.gz.size(), g.cand[i], g.cand.data(), g.cand.size(), mki::K_PASS,
                                     nullptr, 0, 0, &t);
        g_consumed += res[i].consumed;
    }
    for (;;) { // link
        const uint64_t i = mki::upper_bound(g.cand.data(), g.cand.size(), st.pos);
        mki::SegRes r;
        if (i > 0 && g.cand[i - 1] == st.pos && res[i - 1].status != mki::SEG_SUSPEND) {
            r = res[i - 1];
        } else {
            r = mki::decode_segment(g.gz.data(), g.gz.size(), st.pos, g.cand.data(), g.cand.size(), mki::NO_LIMIT,
                                    nullptr, 0, 0, &t);
            g.times.extra_decodes++;
        }
        mki::Seg seg;
        mki::Member mem;
        bool ended = false;
        const int lk = mki::link_feed(&st, r, g.gz.data(), g.gz.size(), &seg, &mem, &ended);
        if (lk == mki::LINK_ERR)
            return fail(h, MKSNAP_E_DATA, "gunzip: malformed data in member " + std::to_string(st.member));
        g.segs.push_back(seg);
        if (ended)
            g.mems.push_back(mem);
        if (lk == mki::LINK_DONE)
            break;
    }
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

// count-pass work of the last mksnap_gunzip_open: input bytes all speculative decodes went through, candidate starts
uint64_t mock_gunzip_consumed(void) { return g_consumed; }
uint64_t mock_gunzip_candidates(void) { return g_candidates; }

void mksnap_destroy(mksnap_t *h)
{
    g_gz.erase(h);
    mock_base_destroy(h);
}

int mksnap_gunzip_open(mksnap_t *h, const void *gz, uint64_t gz_len, mksnap_gunzip_info *info)
{
    if (!h || (!gz && gz_len) || !info)
        return MKSNAP_E_INVAL;
    if (g_gz.count(h))
        return fail(h, MKSNAP_E_STATE, "gunzip: already open (close it first)");
    memset(info, 0, sizeof *info);
    MockGz &g = g_gz[h];
    g.gz.assign((const uint8_t *)gz, (const uint8_t *)gz + gz_len);
    const int rc = gz_open(h, g, info);
    if (rc) {
        g_gz.erase(h);
        memset(info, 0, sizeof *info);
    }
    return rc;
}

int mksnap_gunzip_read(mksnap_t *h, void *dst, uint64_t cap, uint64_t *got)
{
    if (!h || !got || (!dst && cap))
        return MKSNAP_E_INVAL;
    *got = 0;
    auto it = g_gz.find(h);
    if (it == g_gz.end())
        return fail(h, MKSNAP_E_STATE, "gunzip: not open");
    MockGz &g = it->second;
    uint8_t *d = (uint8_t *)dst;
    while (*got < cap) {
        if (g.broken)
            return fail(h, MKSNAP_E_DATA, "gunzip: malformed data");
        if (g.pos >= g.fail_at)
            return fail(h, MKSNAP_E_DATA, "gunzip: CRC-32 or length mismatch in a member trailer");
        if (g.pos == g.win_end) {
            if (g.next_win == g.wins.size())
                break;
            const int rc = gz_window(h, g);
            if (rc)
                return rc;
            continue;
        }
        const uint64_t n = std::min({cap - *got, g.win_end - g.pos, g.fail_at - g.pos});
        memcpy(d + *got, g.out.data() + (g.pos - g.win_off), n);
        g.pos += n;
        *got += n;
    }
    if (g.pos >= g.fail_at)
        return fail(h, MKSNAP_E_DATA, "gunzip: CRC-32 or length mismatch in a member trailer");
    return 0;
}

int mksnap_gunzip_close(mksnap_t *h)
{
    if (!h)
        return MKSNAP_E_INVAL;
    g_gz.erase(h);
    return 0;
}

int mksnap_gunzip_get_times(mksnap_t *h, mksnap_gunzip_times *out)
{
    auto it = h ? g_gz.find(h) : g_gz.end();
    if (!out || it == g_gz.end())
        return MKSNAP_E_INVAL;
    *out = it->second.times;
    return 0;
}

} // extern "C"
