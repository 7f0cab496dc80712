// mock_mksnap_gunzip_members.cpp -- TEST INFRASTRUCTURE ONLY: the gunzip mock of mock_mksnap_gunzip.cpp with the
// engine's full candidate rule.  mock_mksnap_gunzip.cpp scans only flush points (the byte after every 00 00 FF FF);
// mksnap_inflate.cuh also scans every member body start (k_gz_scan_headers), so that the members of a bgzip /
// eStargz / concatenated blob are count-decoded in parallel.  This file reuses that mock's windows, reads, close and
// times unchanged and replaces mksnap_gunzip_open with one that builds the candidate table as the device does:
// mki::flush_end or mki::member_body (mksnap_inflate_core.h), sorted and unique, every candidate tagged with its
// kind.  The flush-only open stays in the library as mock_flush_only_gunzip_open.
// tests/test_host_gunzip_members_cpu.py builds this file (also with ASan/UBSan) and loads it with RTLD_GLOBAL before
// libmkhost.
#define mksnap_gunzip_open mock_flush_only_gunzip_open
#include "mock_mksnap_gunzip.cpp"
#undef mksnap_gunzip_open

namespace {

std::vector<uint8_t> g_cand_kind; // CAND_FLUSH / CAND_MEMBER bits of each candidate of the last open
std::vector<uint64_t> g_cand_off; // ... and its offset

int gz_open_members(mksnap *h, MockGz &g, mksnap_gunzip_info *info)
{
    mki::LinkState st;
    if (mki::link_start(&st, g.gz.data(), g.gz.size()) != mki::LINK_NEXT)
        return fail(h, MKSNAP_E_DATA, "gunzip: no gzip member header at offset 0");
    std::vector<uint8_t> kind(g.gz.size() + 1, 0); // k_gz_scan_headers (the device keeps only the member bit)
    for (uint64_t q = 0; q < g.gz.size(); ++q) {
        const int64_t p = mki::member_body(g.gz.data(), g.gz.size(), q);
        if (p > (int64_t)st.pos)
            kind[p] |= mki::CAND_MEMBER;
    }
    g.cand.push_back(st.pos); // k_gz_scan_count / _write
    g_cand_kind.assign(1, mki::CAND_MEMBER);
    for (uint64_t p = st.pos + 1; p <= g.gz.size(); ++p) {
        if (mki::flush_end(g.gz.data(), p))
            kind[p] |= mki::CAND_FLUSH;
        if (kind[p]) {
            g.cand.push_back(p);
            g_cand_kind.push_back(kind[p]);
        }
    }
    g_cand_off = g.cand;
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

// candidate i of the last open: its offset in *off, and its CAND_FLUSH / CAND_MEMBER bits (0: no such candidate)
uint32_t mock_gunzip_candidate(uint64_t i, uint64_t *off)
{
    if (i >= g_cand_kind.size())
        return 0;
    *off = g_cand_off[i];
    return g_cand_kind[i];
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
    const int rc = gz_open_members(h, g, info);
    if (rc) {
        g_gz.erase(h);
        memset(info, 0, sizeof *info);
    }
    return rc;
}

} // extern "C"
