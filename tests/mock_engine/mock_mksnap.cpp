// mock_mksnap.cpp -- TEST INFRASTRUCTURE ONLY: a CPU stand-in for libmksnap.  Digests and CRCs come from the oracle
// (oracle/mkoracle.c); gunzip runs the engine's own DEFLATE, link and resolve code (makisu_b200/csrc/
// mksnap_inflate_core.h) in the order mksnap_inflate.cuh runs it on the device, one loop iteration where the device
// runs one thread.  It exists so that the host side of libmkhost (layer commit across several arenas, tar ingest,
// per-file digests, untar and materialise from the arena, the incremental commit, plan cacheIDs, deferred streams, gzip
// layers) can be exercised without a GPU: the CPU tests load it with RTLD_GLOBAL *before* libmkhost in a fresh process
// (tests/mock_engine/__init__.py), so libmkhost's mksnap_* references bind here.  It is never loaded by the product,
// lives under tests/, and enforces the same contract the real library does (offsets inside `used`, 16-byte aligned
// ranges, non-final stream pieces non-empty multiples of 64 bytes, one piece per stream per submit, stream slot <
// max_extents, no stream left open at finish, all pieces of a stream deferred or none, ...).
//
// Where it differs from the engine on purpose:
//   - a sparse submit (mksnap_arena_submit_spans) zeroes the arena outside its spans, which is what the device holds,
//     so a packer that leaves out a byte the engine reads computes a different root than the plain commit;
//   - deferred stream pieces are hashed when they are submitted (a digest cannot depend on when it is hashed); the
//     stream log is kept as bookkeeping only: which pieces it takes, and when one that does not fit forces a flush;
//   - the per-extent CRC table that mksnap_crc_fold reads keeps 4 * max_extents values (the engine keeps
//     max(4 * max_extents, 2^20)), so that a CPU test can outrun it with a few hundred segments;
//   - gunzip windows are MOCK_WINDOW bytes, so that CPU-sized blobs span several.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "../../include/mksnap.h"
#include "../../makisu_b200/csrc/mksnap_inflate_core.h"
extern "C" {
#include "../../oracle/mkoracle.h"
}

namespace {

constexpr uint64_t MOCK_WINDOW = 256 * 1024;

struct MockGz {
    std::vector<uint8_t> gz;
    bool indexed = false;      // opened by mksnap_gunzip_open_indexed: bit positions
    std::vector<uint64_t> cand;
    std::vector<mki::Seg> segs;
    std::vector<mki::Member> mems;
    std::vector<std::pair<uint64_t, uint64_t>> wins; // segments [first, second)
    uint64_t next_win = 0, win_off = 0, win_end = 0, pos = 0, fail_at = UINT64_MAX;
    std::vector<uint8_t> out, hist = std::vector<uint8_t>(mki::WSIZE, 0);
    std::vector<uint32_t> mem_crc; // running CRC-32 per member
    bool broken = false;
    mksnap_gunzip_times times{};
    std::vector<uint64_t> index; // mksnap_gunzip_get_index
    mksnap_gunzip_index_info idx{};
};

// a piece of a CDC file: where its first byte lies in the concatenation of the arenas the session submitted
struct Piece {
    uint64_t gbase, len;
};

// everything mksnap_begin starts afresh
struct Session {
    uint32_t crc_pure = 0, host_acc = 0; // submitted extents; mksnap_crc_add contributions
    uint64_t crc_bytes = 0, host_bytes = 0, cdc_bytes = 0, n_files = 0, n_streams = 0;
    std::vector<uint32_t> ext_pure;          // pure(extent) of every CRC extent of the session
    std::map<uint32_t, uint32_t> crc_folds;  // mksnap_crc_fold: stream slot -> pure value
    std::vector<uint8_t> digests;            // 32 B per chunk row, in order
    std::vector<uint64_t> ends;              // per row: chunk end in the submitted bytes (UINT64_MAX: mksnap_chunks_add)
    uint64_t submitted = 0;                  // bytes of the arenas submitted so far
    bool file_open = false;                  // MKSNAP_X_MORE seen: the next submit must start with the continuation
    uint64_t open_follow = 0;
    std::vector<Piece> file;                 // the pieces of the CDC file being gathered ...
    std::vector<uint8_t> file_bytes;         // ... and their bytes: the whole file is chunked when its last piece arrives
    bool overflow = false;                   // mksnap_chunks_add past max_chunks: finish fails
    std::string log;                         // mock_chunk_log
    std::map<uint32_t, mko_sha256_ctx> open_streams;
    std::map<uint32_t, std::vector<uint8_t>> stream_digest;
    std::map<uint32_t, bool> open_defer;     // slot of an open stream -> its pieces are deferred
    uint64_t log_used = 0, log_pending = 0;  // the stream log: bytes taken, pieces waiting for a flush
};

} // namespace

struct mksnap {
    mksnap_config cfg;
    std::string err;
    std::vector<std::vector<uint8_t>> arenas;
    std::vector<bool> acquired;
    uint32_t next = 0;
    bool in_session = false, finished = false;
    uint64_t submits = 0;                      // mock_submits
    uint64_t log_cap = 0, log_flushes = 0;     // mksnap_reserve_stream_log; mock_log_flushes
    std::unique_ptr<MockGz> gz;
    Session ses;
};

namespace {

std::string g_err;
// the last gunzip open: count-pass work, block-start records, and the byte candidates with their CAND_* kinds
uint64_t g_consumed = 0, g_candidates = 0, g_records = 0;
std::vector<uint64_t> g_cand_off;
std::vector<uint8_t> g_cand_kind;

int fail(mksnap *h, int code, const std::string &m)
{
    (h ? h->err : g_err) = m;
    return code;
}

mko_cdc_params cdc_params(const mksnap *h)
{
    mko_cdc_params p;
    mko_cdc_default_params(&p);
    if (h->cfg.cdc.min_size)
        memcpy(&p, &h->cfg.cdc, sizeof p);
    return p;
}

// chunk the gathered file: a digest and an end per chunk
void chunk_file(const mko_cdc_params &p, Session &s)
{
    const uint8_t *fp = s.file_bytes.data();
    std::vector<uint64_t> cuts(s.file_bytes.size() / p.min_size + 2);
    const size_t n = mko_cdc_cuts(fp, s.file_bytes.size(), &p, cuts.data(), cuts.size());
    uint64_t prev = 0, pstart = 0;
    size_t k = 0;
    for (size_t j = 0; j < n; ++j) {
        uint8_t d[32];
        mko_sha256(fp + prev, cuts[j] - prev, d);
        s.digests.insert(s.digests.end(), d, d + 32);
        while (cuts[j] > pstart + s.file[k].len) // the piece that holds the chunk's last byte
            pstart += s.file[k++].len;
        s.ends.push_back(s.file[k].gbase + (cuts[j] - pstart));
        prev = cuts[j];
    }
    s.file.clear();
    s.file_bytes.clear();
}

// mksnap_arena_submit and, after it has zeroed the bytes outside the spans, mksnap_arena_submit_spans
int submit(mksnap *h, int32_t arena_id, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
           const mksnap_range *rng, uint64_t n_rng, const std::string &log_tail)
{
    Session &s = h->ses;
    for (uint64_t i = 0; i < n_rng; ++i) {
        auto it = s.open_defer.find(rng[i].stream);
        if (it != s.open_defer.end() && it->second != ((rng[i].flags & MKSNAP_R_DEFER) != 0))
            return fail(h, MKSNAP_E_INVAL, "a stream mixes MKSNAP_R_DEFER and inline pieces");
    }
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->acquired[arena_id])
        return fail(h, MKSNAP_E_STATE, "arena was not acquired");
    if (used > h->arenas[arena_id].size())
        return fail(h, MKSNAP_E_CAPACITY, "used exceeds the arena");
    if (n_ext > h->cfg.max_extents || n_rng > h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "too many extents / ranges in one submit");
    const uint8_t *a = h->arenas[arena_id].data();
    const mko_cdc_params p = cdc_params(h);
    const size_t rows0 = s.digests.size() / 32;
    uint64_t n_cdc = 0;
    bool saw_more = false;
    for (uint64_t i = 0; i < n_ext; ++i) {
        const mksnap_extent &e = ext[i];
        if (e.arena_off % 16 || e.arena_off + e.len > used)
            return fail(h, MKSNAP_E_INVAL, "extent outside the submitted bytes or not 16-byte aligned");
        if (e.flags & MKSNAP_X_CRC) {
            const uint32_t pv = mko_crc32_pure(a + e.arena_off, e.len);
            s.ext_pure.push_back(pv);
            s.crc_pure ^= mko_crc32_mulmod(pv, mko_crc32_xpow8n(e.crc_suffix));
            s.crc_bytes += e.len;
        }
        if (e.flags & MKSNAP_X_CDC) {
            const bool cont = e.flags & MKSNAP_X_CONT, more = e.flags & MKSNAP_X_MORE;
            // a file that spans submits (same contract as the real engine): the pieces are gathered and the WHOLE file
            // is chunked when its last piece arrives -- by definition what the engine's carried open chunk must reproduce
            if (cont && (n_cdc != 0 || !s.file_open))
                return fail(h, MKSNAP_E_STATE, "MKSNAP_X_CONT must be the first CDC extent after a MKSNAP_X_MORE extent");
            if (cont && e.arena_off < 131072)
                return fail(h, MKSNAP_E_INVAL, "a continuation starts at arena offset >= carry_bytes");
            if (!cont && s.file_open)
                return fail(h, MKSNAP_E_STATE, "the previous submit left a file open: its continuation must come first");
            if (saw_more)
                return fail(h, MKSNAP_E_INVAL, "a MKSNAP_X_MORE extent must be the last CDC extent of its submit");
            if (more && (e.len == 0 || e.reserved == 0))
                return fail(h, MKSNAP_E_INVAL, "MKSNAP_X_MORE needs a non-empty piece and the bytes that follow");
            if (cont && s.open_follow != e.len + (more ? e.reserved : 0) && s.open_follow != 0xFFFFFFFFull)
                return fail(h, MKSNAP_E_INVAL, "continuation length disagrees with the bytes announced by the previous piece");
            ++n_cdc;
            s.cdc_bytes += e.len;
            if (!cont)
                s.n_files++;
            s.file.push_back(Piece{s.submitted + e.arena_off, e.len});
            s.file_bytes.insert(s.file_bytes.end(), a + e.arena_off, a + e.arena_off + e.len);
            s.file_open = saw_more = more;
            s.open_follow = more ? e.reserved : 0;
            if (!more)
                chunk_file(p, s);
        } else if (e.flags & (MKSNAP_X_MORE | MKSNAP_X_CONT)) {
            return fail(h, MKSNAP_E_INVAL, "MKSNAP_X_MORE / MKSNAP_X_CONT apply to CDC extents");
        }
    }
    std::set<uint32_t> seen;
    for (uint64_t i = 0; i < n_rng; ++i) { // every range is checked before any stream moves, as on the engine
        const mksnap_range &r = rng[i];
        if (r.arena_off % 16 || r.arena_off + r.len > used)
            return fail(h, MKSNAP_E_INVAL, "range outside the submitted bytes or not 16-byte aligned");
        if (r.stream >= h->cfg.max_extents)
            return fail(h, MKSNAP_E_CAPACITY, "stream slot beyond max_extents");
        if ((r.flags & MKSNAP_R_MORE) && (r.len == 0 || r.len % 64))
            return fail(h, MKSNAP_E_INVAL, "non-final stream piece is empty or not a multiple of 64 bytes");
        if (!seen.insert(r.stream).second)
            return fail(h, MKSNAP_E_INVAL, "two pieces of one stream in one submit");
    }
    for (uint64_t i = 0; i < n_rng; ++i) {
        const mksnap_range &r = rng[i];
        auto it = s.open_streams.find(r.stream);
        if (it == s.open_streams.end()) {
            mko_sha256_ctx c;
            mko_sha256_init(&c);
            it = s.open_streams.emplace(r.stream, c).first;
        }
        mko_sha256_update(&it->second, a + r.arena_off, r.len);
        const bool defer = (r.flags & MKSNAP_R_DEFER) != 0;
        if (r.flags & MKSNAP_R_MORE) {
            s.open_defer[r.stream] = defer;
        } else {
            std::vector<uint8_t> d(32);
            mko_sha256_final(&it->second, d.data());
            s.stream_digest[r.stream] = d;
            s.open_streams.erase(it);
            s.n_streams = std::max<uint64_t>(s.n_streams, (uint64_t)r.stream + 1);
            s.open_defer.erase(r.stream);
        }
        if (!defer || !h->log_cap || r.len > h->log_cap)
            continue; // hashed by its own submit
        uint64_t off = (s.log_used + 15) & ~15ull;
        if (off + r.len > h->log_cap) {
            h->log_flushes++;
            s.log_pending = 0;
            off = 0;
        }
        s.log_used = off + r.len;
        s.log_pending++;
    }
    char line[96];
    snprintf(line, sizeof line, "submit used=%llu cdc=%llu rows=%zu", (unsigned long long)used, (unsigned long long)n_cdc,
             s.digests.size() / 32 - rows0);
    s.log += line + log_tail + "\n";
    s.submitted += used;
    h->acquired[arena_id] = false; // the copy to the device is "done": the arena may be re-acquired
    h->submits++;
    return 0;
}

// ---- gunzip ---------------------------------------------------------------------------------------------------------
// k_gz_scan_*, k_gz_decode(_bits) in count mode, the link, and for an indexed open the cut of long segments
template <bool BITS>
int gz_open(mksnap *h, MockGz &g, const uint64_t *points, uint64_t n_points, mksnap_gunzip_info *info)
{
    const uint8_t *gz = g.gz.data();
    const uint64_t gz_len = g.gz.size();
    mki::LinkState st;
    if (mki::link_start<BITS>(&st, gz, gz_len) != mki::LINK_NEXT)
        return fail(h, MKSNAP_E_DATA, "gunzip: no gzip member header at offset 0");
    const uint64_t body0 = BITS ? st.pos / 8 : st.pos;
    std::vector<uint8_t> kind(gz_len + 1, 0); // k_gz_scan_headers (the device keeps only the member bit)
    for (uint64_t q = 0; q < gz_len; ++q) {
        const int64_t p = mki::member_body(gz, gz_len, q);
        if (p > (int64_t)body0)
            kind[p] |= mki::CAND_MEMBER;
    }
    std::vector<uint64_t> byte_cand{body0}; // k_gz_scan_count / _write
    g_cand_kind.assign(1, mki::CAND_MEMBER);
    for (uint64_t p = body0 + 1; p <= gz_len; ++p) {
        if (mki::flush_end(gz, p))
            kind[p] |= mki::CAND_FLUSH;
        if (kind[p]) {
            byte_cand.push_back(p);
            g_cand_kind.push_back(kind[p]);
        }
    }
    g_cand_off = byte_cand;
    g.cand = BITS ? mki::merge_points(byte_cand, points, n_points) : byte_cand;
    std::vector<mki::Rec> recs(BITS ? mki::REC_CAP : 0);
    unsigned long long n_rec = 0;
    const mki::Recorder recorder{recs.data(), &n_rec, mki::REC_CAP};
    const mki::Recorder *rec = BITS ? &recorder : nullptr;
    std::vector<mki::SegRes> res(g.cand.size());
    mki::Tables t;
    g_consumed = 0;
    g_candidates = g.cand.size();
    for (size_t i = 0; i < g.cand.size(); ++i) { // k_gz_decode(_bits), count mode
        res[i] = mki::decode_segment_t<BITS>(gz, gz_len, g.cand[i], g.cand.data(), g.cand.size(), mki::K_PASS,
                                             nullptr, 0, 0, &t, rec);
        g_consumed += res[i].consumed;
    }
    const auto redecode = [&](uint64_t pos, mki::SegRes *r) {
        *r = mki::decode_segment_t<BITS>(gz, gz_len, pos, g.cand.data(), g.cand.size(), mki::NO_LIMIT, nullptr, 0, 0,
                                         &t, rec);
        g.times.extra_decodes++;
        return 0;
    };
    if (mki::link_all<BITS>(&st, g.cand.data(), res.data(), g.cand.size(), gz, gz_len, redecode, &g.segs, &g.mems) ==
        mki::LINK_ERR)
        return fail(h, MKSNAP_E_DATA, "gunzip: malformed data in member " + std::to_string(st.member));
    if (BITS) {
        g_records = n_rec;
        recs.resize(std::min<uint64_t>(n_rec, mki::REC_CAP));
        const mki::IndexCounts c = mki::split_segments(&g.segs, std::move(recs), &g.cand, byte_cand, points, n_points,
                                                       &g.index);
        g.idx = mksnap_gunzip_index_info{n_points, c.linked, c.recorded, g.index.size()};
    }
    for (uint64_t k = 0; k < g.segs.size();) {
        uint64_t e = k, len = 0;
        while (e < g.segs.size() && (e == k || len + g.segs[e].out_len <= MOCK_WINDOW))
            len += g.segs[e++].out_len;
        g.wins.emplace_back(k, e);
        k = e;
    }
    g.mem_crc.assign(g.mems.size(), 0);
    info->gz_bytes = gz_len;
    info->out_bytes = st.out;
    info->n_members = g.mems.size();
    info->n_segments = g.segs.size();
    return 0;
}

int gz_open_entry(mksnap *h, const void *gz, uint64_t gz_len, const uint64_t *points, uint64_t n_points, bool indexed,
                  mksnap_gunzip_info *info)
{
    if (h->gz)
        return fail(h, MKSNAP_E_STATE, "gunzip: already open (close it first)");
    memset(info, 0, sizeof *info);
    h->gz.reset(new MockGz);
    MockGz &g = *h->gz;
    g.gz.assign((const uint8_t *)gz, (const uint8_t *)gz + gz_len);
    g.indexed = indexed;
    const int rc = indexed ? gz_open<true>(h, g, points, n_points, info) : gz_open<false>(h, g, points, n_points, info);
    if (rc) {
        h->gz.reset();
        memset(info, 0, sizeof *info);
    }
    return rc;
}

// the next window: k_gz_decode(_bits) in write mode, k_gz_resolve, k_gz_narrow, k_gz_hist, member trailer checks
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
    for (uint64_t k = w.first; k < w.second; ++k) {
        const mki::Seg &s = g.segs[k];
        uint16_t *out = sym.data() + (s.out_off - g.win_off);
        const mki::SegRes r =
            g.indexed ? mki::decode_segment_t<true>(g.gz.data(), g.gz.size(), s.start, g.cand.data(), g.cand.size(),
                                                    mki::NO_LIMIT, out, s.out_len, s.member_pos, &t, nullptr)
                      : mki::decode_segment_t<false>(g.gz.data(), g.gz.size(), s.start, g.cand.data(), g.cand.size(),
                                                     mki::NO_LIMIT, out, s.out_len, s.member_pos, &t, nullptr);
        if (r.status != (s.final ? mki::SEG_FINAL : mki::SEG_CAND) || r.end != s.end || r.out_len != s.out_len) {
            g.broken = true;
            return fail(h, MKSNAP_E_DATA, "gunzip: malformed data (a distance reaches before the start of its member)");
        }
    }
    for (uint64_t k = w.first; k < w.second; ++k)
        mki::resolve_segment_tail(sym.data(), g.hist.data(), g.segs[k].out_off - g.win_off, g.segs[k].out_len, 0, 1);
    g.out.assign(len, 0);
    for (uint64_t k = w.first; k < w.second; ++k) {
        const uint64_t o = g.segs[k].out_off - g.win_off;
        for (uint64_t j = 0; j < g.segs[k].out_len; ++j)
            g.out[o + j] = mki::resolve_symbol(sym.data(), g.hist.data(), o, sym[o + j]);
    }
    std::vector<uint8_t> nh(mki::WSIZE);
    for (uint32_t i = 0; i < mki::WSIZE; ++i) {
        const int64_t q = (int64_t)len - (int64_t)mki::WSIZE + i;
        nh[i] = q >= 0 ? g.out[q] : g.hist[mki::WSIZE + q];
    }
    g.hist.swap(nh);
    for (uint64_t k = w.first; k < w.second; ++k) {
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

} // namespace

extern "C" {

int mksnap_abi_version(void) { return MKSNAP_ABI_VERSION; }
const char *mksnap_last_error(const mksnap_t *h) { return h ? h->err.c_str() : g_err.c_str(); }

int mksnap_create(const mksnap_config *cfg, mksnap_t **out)
{
    if (!cfg || !out)
        return MKSNAP_E_INVAL;
    mksnap *h = new mksnap;
    h->cfg = *cfg;
    if (h->cfg.max_extents == 0)
        h->cfg.max_extents = 1 << 16;
    for (uint32_t i = 0; i < cfg->n_host_arenas; ++i) {
        h->arenas.emplace_back((size_t)cfg->host_arena_bytes, (uint8_t)0xAA); // poison: unwritten bytes must not matter
        h->acquired.push_back(false);
    }
    *out = h;
    return 0;
}

void mksnap_destroy(mksnap_t *h) { delete h; }

int mksnap_begin(mksnap_t *h)
{
    if (!h)
        return MKSNAP_E_INVAL;
    h->in_session = true;
    h->finished = false;
    h->ses = Session{};
    std::fill(h->acquired.begin(), h->acquired.end(), false);
    return 0;
}

int mksnap_arena_acquire(mksnap_t *h, void **host_ptr, uint64_t *capacity, int32_t *arena_id)
{
    if (!h || !host_ptr || !capacity || !arena_id)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "arena_acquire outside a session");
    if (h->arenas.empty())
        return fail(h, MKSNAP_E_STATE, "no host arenas configured");
    const uint32_t id = h->next++ % h->arenas.size();
    if (h->acquired[id])
        return fail(h, MKSNAP_E_STATE, "arena still acquired (submit it first)");
    h->acquired[id] = true;
    memset(h->arenas[id].data(), 0xAA, h->arenas[id].size());
    *host_ptr = h->arenas[id].data();
    *capacity = h->arenas[id].size();
    *arena_id = (int32_t)id;
    return 0;
}

int mksnap_arena_release(mksnap_t *h, int32_t arena_id)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->acquired[arena_id])
        return fail(h, MKSNAP_E_STATE, "arena was not acquired");
    h->acquired[arena_id] = false;
    return 0;
}

int mksnap_get_limits(const mksnap_t *h, mksnap_limits *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    memset(out, 0, sizeof *out);
    out->max_extents = out->max_streams = h->cfg.max_extents;
    out->host_arena_bytes = h->cfg.host_arena_bytes;
    out->device_arena_bytes = h->cfg.device_arena_bytes;
    out->n_host_arenas = (uint32_t)h->arenas.size();
    out->carry_bytes = 131072;
    return 0;
}

int mksnap_get_cdc(const mksnap_t *h, mksnap_cdc_params *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    const mko_cdc_params p = cdc_params(h);
    memcpy(out, &p, sizeof p);
    return 0;
}

int mksnap_arena_submit(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
                        const mksnap_range *rng, uint64_t n_rng)
{
    if (!h)
        return MKSNAP_E_INVAL;
    return submit(h, arena_id, used, ext, n_ext, rng, n_rng, "");
}

int mksnap_arena_submit_spans(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_span *spans, uint64_t n_spans,
                              const mksnap_extent *ext, uint64_t n_ext, const mksnap_range *rng, uint64_t n_rng)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->acquired[arena_id] || used > h->arenas[arena_id].size())
        return fail(h, MKSNAP_E_STATE, "arena was not acquired or used exceeds it");
    uint64_t end = 0;
    for (uint64_t k = 0; k < n_spans; ++k) {
        if ((spans[k].off | spans[k].len) % 16 || spans[k].off < end || spans[k].off + spans[k].len > used)
            return fail(h, MKSNAP_E_INVAL, "span not 16-byte aligned, out of order or outside [0, used)");
        end = spans[k].off + spans[k].len;
    }
    auto inside = [&](uint64_t off, uint64_t len) {
        if (len == 0)
            return true;
        for (uint64_t k = 0; k < n_spans; ++k)
            if (off >= spans[k].off && off + len <= spans[k].off + spans[k].len)
                return true;
        return false;
    };
    for (uint64_t i = 0; i < n_ext; ++i)
        if (!inside(ext[i].arena_off, ext[i].len))
            return fail(h, MKSNAP_E_INVAL, "extent " + std::to_string(i) + " is not inside one of the submitted spans");
    for (uint64_t i = 0; i < n_rng; ++i)
        if (!inside(rng[i].arena_off, rng[i].len))
            return fail(h, MKSNAP_E_INVAL, "range " + std::to_string(i) + " is not inside one of the submitted spans");
    uint8_t *a = h->arenas[arena_id].data(); // what the device would hold: zeros outside the spans
    uint64_t at = 0;
    std::string sp;
    for (uint64_t k = 0; k < n_spans; ++k) {
        memset(a + at, 0, spans[k].off - at);
        at = spans[k].off + spans[k].len;
        sp += " " + std::to_string(spans[k].off) + "+" + std::to_string(spans[k].len);
    }
    memset(a + at, 0, used - at);
    return submit(h, arena_id, used, ext, n_ext, rng, n_rng, " spans" + sp);
}

int mksnap_chunks_add(mksnap_t *h, const uint8_t *digests, uint64_t n)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "chunks_add outside begin/finish");
    if (n > MKSNAP_CHUNKS_ADD_MAX)
        return fail(h, MKSNAP_E_CAPACITY, "chunks_add: too many rows in one call");
    Session &s = h->ses;
    if (h->cfg.max_chunks && s.digests.size() / 32 + n > h->cfg.max_chunks) {
        s.overflow = true; // like the device: nothing is written, finish reports the overflow
        return 0;
    }
    s.digests.insert(s.digests.end(), digests, digests + 32 * n);
    s.ends.insert(s.ends.end(), n, UINT64_MAX);
    s.log += "add " + std::to_string(n) + "\n";
    return 0;
}

int mksnap_finish(mksnap_t *h, mksnap_result *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "finish outside a session");
    Session &s = h->ses;
    if (s.overflow)
        return fail(h, MKSNAP_E_CAPACITY, "chunk table overflow (max_chunks)");
    if (!s.open_streams.empty())
        return fail(h, MKSNAP_E_STATE, "a stream was left open (last piece carried MKSNAP_R_MORE)");
    if (s.file_open)
        return fail(h, MKSNAP_E_STATE, "a file was left open (MKSNAP_X_MORE without its continuation)");
    memset(out, 0, sizeof *out);
    out->crc_pure = s.crc_pure ^ s.host_acc;
    out->crc_bytes = s.crc_bytes + s.host_bytes;
    out->cdc_bytes = s.cdc_bytes;
    out->n_files = s.n_files;
    out->n_chunks = s.digests.size() / 32;
    std::vector<uint8_t> table = s.digests;
    const size_t uniq = mko_sort_unique_digests(table.data(), table.size() / 32);
    out->n_unique = uniq;
    mko_merkle_root(table.data(), uniq, out->root);
    out->n_streams = s.n_streams;
    if (s.log_pending)
        h->log_flushes++;
    s.log_pending = s.log_used = 0;
    h->in_session = false;
    h->finished = true;
    return 0;
}

int mksnap_get_chunks(mksnap_t *h, uint64_t *ends, uint8_t *digests, uint64_t capacity)
{
    if (!h || !h->finished)
        return h ? fail(h, MKSNAP_E_STATE, "get_chunks before finish") : MKSNAP_E_INVAL;
    const Session &s = h->ses;
    const uint64_t n = s.digests.size() / 32;
    if (n > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need more rows");
    if (ends && n)
        memcpy(ends, s.ends.data(), n * 8);
    if (digests && n)
        memcpy(digests, s.digests.data(), n * 32);
    return 0;
}

uint32_t mksnap_ctx_crc32(const mksnap_result *r)
{
    return r->crc_pure ^ mko_crc32_mulmod(0xFFFFFFFFu, mko_crc32_xpow8n(r->crc_bytes)) ^ 0xFFFFFFFFu;
}

int mksnap_get_stream_digests(mksnap_t *h, uint8_t *digests, uint64_t capacity)
{
    if (!h || !digests)
        return MKSNAP_E_INVAL;
    const Session &s = h->ses;
    if (s.n_streams > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need more rows");
    for (uint64_t k = 0; k < s.n_streams; ++k) {
        auto it = s.stream_digest.find((uint32_t)k);
        if (it != s.stream_digest.end())
            memcpy(digests + 32 * k, it->second.data(), 32);
        else
            memset(digests + 32 * k, 0xEE, 32); // never-written slot: garbage, like device memory
    }
    return 0;
}

int mksnap_reserve_stream_log(mksnap_t *h, uint64_t bytes)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (h->ses.log_pending)
        return fail(h, MKSNAP_E_STATE, "reserve_stream_log while deferred pieces wait in the log");
    h->log_cap = (bytes + 63) & ~63ull;
    return 0;
}

int mksnap_crc_add(mksnap_t *h, uint32_t pure, uint64_t len, uint64_t crc_suffix)
{
    if (!h || !h->in_session)
        return MKSNAP_E_STATE;
    h->ses.host_acc ^= mko_crc32_mulmod(pure, mko_crc32_xpow8n(crc_suffix));
    h->ses.host_bytes += len;
    return 0;
}

uint32_t mksnap_crc_concat(uint32_t pure_a, uint32_t pure_b, uint64_t len_b) { return mko_crc32_mulmod(pure_a, mko_crc32_xpow8n(len_b)) ^ pure_b; }

int mksnap_get_extent_crcs(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out)
{
    if (!h || !n_out)
        return MKSNAP_E_INVAL;
    const std::vector<uint32_t> &v = h->ses.ext_pure;
    *n_out = v.size();
    if (!pure || capacity < v.size())
        return fail(h, MKSNAP_E_CAPACITY, "need more entries");
    if (!v.empty())
        memcpy(pure, v.data(), v.size() * 4);
    return 0;
}

int mksnap_crc_fold(mksnap_t *h, const mksnap_crc_use *uses, uint64_t n)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "crc_fold outside begin/finish");
    if (n > h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "crc_fold: too many uses in one call");
    Session &s = h->ses;
    if (s.ext_pure.size() > 4 * h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "crc_fold: the session submitted more CRC extents than the per-extent table keeps");
    for (uint64_t i = 0; i < n; ++i)
        if (uses[i].stream >= h->cfg.max_extents || (uses[i].flags & ~MKSNAP_U_VALUE) ||
            (!(uses[i].flags & MKSNAP_U_VALUE) && uses[i].src >= s.ext_pure.size()))
            return fail(h, MKSNAP_E_INVAL, "crc_fold: use " + std::to_string(i) + " names a stream or extent out of range");
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t v = (uses[i].flags & MKSNAP_U_VALUE) ? (uint32_t)uses[i].src : s.ext_pure[uses[i].src];
        s.crc_folds[uses[i].stream] ^= mko_crc32_mulmod(v, mko_crc32_xpow8n(uses[i].suffix));
    }
    return 0;
}

int mksnap_get_crc_streams(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out)
{
    if (!h || !n_out)
        return MKSNAP_E_INVAL;
    if (!h->finished)
        return fail(h, MKSNAP_E_STATE, "get_crc_streams before finish");
    const std::map<uint32_t, uint32_t> &f = h->ses.crc_folds;
    *n_out = f.empty() ? 0 : (uint64_t)f.rbegin()->first + 1;
    if (*n_out > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need more entries");
    for (uint64_t k = 0; k < *n_out; ++k) {
        auto it = f.find((uint32_t)k);
        pure[k] = it != f.end() ? it->second : 0u;
    }
    return 0;
}

uint32_t mksnap_crc_prepend(const void *prefix, uint64_t n, uint32_t pure_rest, uint64_t len_rest)
{
    const uint32_t pure = mko_crc32_mulmod(mko_crc32_pure((const uint8_t *)prefix, n), mko_crc32_xpow8n(len_rest)) ^ pure_rest;
    return pure ^ mko_crc32_mulmod(0xFFFFFFFFu, mko_crc32_xpow8n(n + len_rest)) ^ 0xFFFFFFFFu;
}

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
            return fail(h, MKSNAP_E_INVAL, "gunzip: index point " + std::to_string(k) + " is out of order or past the blob");
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
    if (!h->gz)
        return fail(h, MKSNAP_E_STATE, "gunzip: not open");
    MockGz &g = *h->gz;
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
    h->gz.reset();
    return 0;
}

int mksnap_gunzip_get_times(mksnap_t *h, mksnap_gunzip_times *out)
{
    if (!h || !out || !h->gz)
        return MKSNAP_E_INVAL;
    *out = h->gz->times;
    return 0;
}

// ---- test hooks -----------------------------------------------------------------------------------------------------
uint64_t mock_submits(mksnap_t *h) { return h->submits; }

// the session's submits and appends as text: "submit used=U cdc=N rows=R[ spans off+len ...]" / "add N"
size_t mock_chunk_log(mksnap_t *h, char *out, size_t cap)
{
    const std::string &s = h->ses.log;
    if (s.size() + 1 <= cap)
        memcpy(out, s.c_str(), s.size() + 1);
    return s.size() + 1;
}

// stream-log flushes over the handle's life: a deferred piece that did not fit, or pieces still waiting at finish
uint64_t mock_log_flushes(mksnap_t *h) { return h->log_flushes; }

// count-pass work of the last gunzip open: input bytes all speculative decodes went through, candidate starts
uint64_t mock_gunzip_consumed(void) { return g_consumed; }
uint64_t mock_gunzip_candidates(void) { return g_candidates; }

// byte candidate i of the last open: its offset in *off, and its CAND_FLUSH / CAND_MEMBER bits (0: no such candidate)
uint32_t mock_gunzip_candidate(uint64_t i, uint64_t *off)
{
    if (i >= g_cand_kind.size())
        return 0;
    *off = g_cand_off[i];
    return g_cand_kind[i];
}

// records offered by the count decodes of the last indexed open (before the capacity)
uint64_t mock_gunzip_records(void) { return g_records; }

// the segments of the open gunzip: start and end (bit offsets after an indexed open), decompressed length
uint64_t mock_gunzip_segments(const mksnap_t *h, uint64_t *start, uint64_t *end, uint64_t *out_len, uint64_t cap)
{
    if (!h->gz)
        return 0;
    const auto &s = h->gz->segs;
    for (uint64_t k = 0; k < std::min<uint64_t>(cap, s.size()); ++k) {
        start[k] = s[k].start;
        end[k] = s[k].end;
        out_len[k] = s[k].out_len;
    }
    return s.size();
}

} // extern "C"
