// mock_mksnap.cpp -- TEST INFRASTRUCTURE ONLY: a CPU stand-in for the seven libmksnap entry points libmkhost calls
// (mksnap_begin / arena_acquire / arena_submit / finish / ctx_crc32 / get_stream_digests / last_error, plus
// create/destroy), computing every digest with the oracle (oracle/mkoracle.c).  It exists so that the host-side
// packers of libmkhost (layer commit across several arenas, tar ingest, per-file digests, untar and materialise from
// the arena) can be exercised without a GPU: tests/test_host_mock_engine_cpu.py loads it with RTLD_GLOBAL *before*
// libmkhost in a fresh process, so libmkhost's mksnap_* references bind here.  It is never loaded by the product,
// lives under tests/, and enforces the same contract the real library does (offsets inside `used`, 16-byte aligned
// ranges, non-final stream pieces non-empty multiples of 64 bytes, one piece per stream per submit, stream slot <
// max_extents, no stream left open at finish).
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/mksnap.h"
extern "C" {
#include "../../oracle/mkoracle.h"
}

struct mksnap {
    mksnap_config cfg;
    std::string err;
    std::vector<std::vector<uint8_t>> arenas;
    std::vector<bool> acquired;
    uint32_t next = 0;
    bool in_session = false, finished = false;
    // session
    uint32_t crc_pure = 0;
    uint64_t crc_bytes = 0, cdc_bytes = 0, n_files = 0, n_streams = 0;
    std::vector<uint8_t> digests; // 32 B per chunk, submit order
    std::map<uint32_t, mko_sha256_ctx> open_streams;
    std::map<uint32_t, std::vector<uint8_t>> stream_digest;
    mksnap_result last;
    uint64_t submits = 0;
    std::vector<uint32_t> ext_pure;    // pure(extent) of every CRC extent of the session
    uint32_t host_acc = 0;             // mksnap_crc_add contributions
    uint64_t host_bytes = 0;
    bool file_open = false;            // MKSNAP_X_MORE seen: the next submit must start with the continuation
    uint64_t open_follow = 0;
    std::vector<uint8_t> open_bytes;   // pieces of the file that spans submits
};

static std::string g_err;

static int fail(mksnap *h, int code, const std::string &m)
{
    (h ? h->err : g_err) = m;
    return code;
}

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
    h->crc_pure = 0;
    h->crc_bytes = h->cdc_bytes = h->n_files = h->n_streams = 0;
    h->digests.clear();
    h->open_streams.clear();
    h->stream_digest.clear();
    h->file_open = false;
    h->open_bytes.clear();
    h->ext_pure.clear();
    h->host_acc = 0;
    h->host_bytes = 0;
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

int mksnap_arena_submit(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
                        const mksnap_range *rng, uint64_t n_rng)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (arena_id < 0 || (size_t)arena_id >= h->arenas.size() || !h->acquired[arena_id])
        return fail(h, MKSNAP_E_STATE, "arena was not acquired");
    if (used > h->arenas[arena_id].size())
        return fail(h, MKSNAP_E_CAPACITY, "used exceeds the arena");
    if (n_ext > h->cfg.max_extents || n_rng > h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "too many extents / ranges in one submit");
    const uint8_t *a = h->arenas[arena_id].data();
    mko_cdc_params p;
    mko_cdc_default_params(&p);
    if (h->cfg.cdc.min_size)
        memcpy(&p, &h->cfg.cdc, sizeof p);
    uint64_t n_cdc = 0;
    bool saw_more = false;
    for (uint64_t i = 0; i < n_ext; ++i) {
        const mksnap_extent &e = ext[i];
        if (e.arena_off % 16 || e.arena_off + e.len > used)
            return fail(h, MKSNAP_E_INVAL, "extent outside the submitted bytes or not 16-byte aligned");
        if (e.flags & MKSNAP_X_CRC) {
            const uint32_t pv = mko_crc32_pure(a + e.arena_off, e.len);
            h->ext_pure.push_back(pv);
            h->crc_pure ^= mko_crc32_mulmod(pv, mko_crc32_xpow8n(e.crc_suffix));
            h->crc_bytes += e.len;
        }
        if (e.flags & MKSNAP_X_CDC) {
            const bool cont = e.flags & MKSNAP_X_CONT, more = e.flags & MKSNAP_X_MORE;
            // a file that spans submits (same contract as the real engine): the pieces are buffered and the WHOLE file is
            // chunked when its last piece arrives -- by definition what the engine's carried open chunk must reproduce
            if (cont && (n_cdc != 0 || !h->file_open))
                return fail(h, MKSNAP_E_STATE, "MKSNAP_X_CONT must be the first CDC extent after a MKSNAP_X_MORE extent");
            if (cont && e.arena_off < 131072)
                return fail(h, MKSNAP_E_INVAL, "a continuation starts at arena offset >= carry_bytes");
            if (!cont && h->file_open)
                return fail(h, MKSNAP_E_STATE, "the previous submit left a file open: its continuation must come first");
            if (saw_more)
                return fail(h, MKSNAP_E_INVAL, "a MKSNAP_X_MORE extent must be the last CDC extent of its submit");
            if (more && (e.len == 0 || e.reserved == 0))
                return fail(h, MKSNAP_E_INVAL, "MKSNAP_X_MORE needs a non-empty piece and the bytes that follow");
            ++n_cdc;
            h->cdc_bytes += e.len;
            if (!cont)
                h->n_files++;
            const uint8_t *fp = a + e.arena_off;
            uint64_t flen = e.len;
            if (cont || more) {
                if (cont && h->open_follow != e.len + (more ? e.reserved : 0) && h->open_follow != 0xFFFFFFFFull)
                    return fail(h, MKSNAP_E_INVAL, "continuation length disagrees with the bytes announced by the previous piece");
                h->open_bytes.insert(h->open_bytes.end(), fp, fp + e.len);
                h->file_open = more;
                h->open_follow = more ? e.reserved : 0;
                saw_more = more;
                if (more)
                    continue;
                fp = h->open_bytes.data();
                flen = h->open_bytes.size();
            }
            std::vector<uint64_t> ends((size_t)(flen / p.min_size) + 2);
            const size_t n = mko_cdc_cuts(fp, flen, &p, ends.data(), ends.size());
            uint64_t prev = 0;
            for (size_t j = 0; j < n; ++j) {
                uint8_t d[32];
                mko_sha256(fp + prev, ends[j] - prev, d);
                h->digests.insert(h->digests.end(), d, d + 32);
                prev = ends[j];
            }
            if (cont)
                h->open_bytes.clear();
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
        auto it = h->open_streams.find(r.stream);
        if (it == h->open_streams.end()) {
            mko_sha256_ctx c;
            mko_sha256_init(&c);
            it = h->open_streams.emplace(r.stream, c).first;
        }
        mko_sha256_update(&it->second, a + r.arena_off, r.len);
        if (!(r.flags & MKSNAP_R_MORE)) {
            std::vector<uint8_t> d(32);
            mko_sha256_final(&it->second, d.data());
            h->stream_digest[r.stream] = d;
            h->open_streams.erase(it);
            h->n_streams = std::max<uint64_t>(h->n_streams, (uint64_t)r.stream + 1);
        }
    }
    h->acquired[arena_id] = false; // the copy to the device is "done": the arena may be re-acquired
    h->submits++;
    return 0;
}

int mksnap_finish(mksnap_t *h, mksnap_result *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "finish outside a session");
    if (!h->open_streams.empty())
        return fail(h, MKSNAP_E_STATE, "a stream was left open (last piece carried MKSNAP_R_MORE)");
    if (h->file_open)
        return fail(h, MKSNAP_E_STATE, "a file was left open (MKSNAP_X_MORE without its continuation)");
    memset(out, 0, sizeof *out);
    out->crc_pure = h->crc_pure ^ h->host_acc;
    out->crc_bytes = h->crc_bytes + h->host_bytes;
    out->cdc_bytes = h->cdc_bytes;
    out->n_files = h->n_files;
    out->n_chunks = h->digests.size() / 32;
    std::vector<uint8_t> table = h->digests;
    const size_t uniq = mko_sort_unique_digests(table.data(), table.size() / 32);
    out->n_unique = uniq;
    mko_merkle_root(table.data(), uniq, out->root);
    out->n_streams = h->n_streams;
    h->last = *out;
    h->in_session = false;
    h->finished = true;
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
    if (h->n_streams > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need more rows");
    for (uint64_t s = 0; s < h->n_streams; ++s) {
        auto it = h->stream_digest.find((uint32_t)s);
        if (it != h->stream_digest.end())
            memcpy(digests + 32 * s, it->second.data(), 32);
        else
            memset(digests + 32 * s, 0xEE, 32); // never-written slot: garbage, like device memory
    }
    return 0;
}

int mksnap_crc_add(mksnap_t *h, uint32_t pure, uint64_t len, uint64_t crc_suffix)
{
    if (!h || !h->in_session)
        return MKSNAP_E_STATE;
    h->host_acc ^= mko_crc32_mulmod(pure, mko_crc32_xpow8n(crc_suffix));
    h->host_bytes += len;
    return 0;
}

uint32_t mksnap_crc_concat(uint32_t pure_a, uint32_t pure_b, uint64_t len_b) { return mko_crc32_mulmod(pure_a, mko_crc32_xpow8n(len_b)) ^ pure_b; }

int mksnap_get_extent_crcs(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out)
{
    if (!h || !n_out)
        return MKSNAP_E_INVAL;
    *n_out = h->ext_pure.size();
    if (!pure || capacity < h->ext_pure.size())
        return fail(h, MKSNAP_E_CAPACITY, "need more entries");
    if (!h->ext_pure.empty())
        memcpy(pure, h->ext_pure.data(), h->ext_pure.size() * 4);
    return 0;
}

uint64_t mock_submits(mksnap_t *h) { return h->submits; }

} // extern "C"
