// mock_mksnap_defer.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock engine with gunzip (mock_mksnap_gunzip.cpp) plus
// deferred streams: the MKSNAP_R_DEFER range flag and mksnap_reserve_stream_log.  The mock hashes every piece when it
// is submitted (a deferred stream's digest cannot depend on when it is hashed); what it keeps of the engine is the
// contract -- all pieces of a stream deferred or none (MKSNAP_E_INVAL), no resize while pieces wait in the log
// (MKSNAP_E_STATE) -- and the log's bookkeeping: which deferred pieces the log takes, and when a piece that does not fit
// forces a flush (counted by mock_log_flushes).  tests/test_stream_defer_cpu.py and
// tests/test_host_update_from_tars_cpu.py build this file and load it with RTLD_GLOBAL before libmkhost.
#define mksnap_create mock_defer_base_create
#define mksnap_begin mock_defer_base_begin
#define mksnap_arena_submit mock_defer_base_submit
#define mksnap_finish mock_defer_base_finish
#include "mock_mksnap_gunzip.cpp"
#undef mksnap_create
#undef mksnap_begin
#undef mksnap_arena_submit
#undef mksnap_finish

namespace {
struct DeferState {
    uint64_t log_cap = 0, log_used = 0, pending = 0, flushes = 0;
    std::map<uint32_t, bool> open_defer; // slot of an open stream -> its pieces are deferred
};
std::map<const mksnap *, DeferState> g_defer;
} // namespace

extern "C" {

int mksnap_create(const mksnap_config *cfg, mksnap_t **out)
{
    const int rc = mock_defer_base_create(cfg, out);
    if (rc == 0)
        g_defer[*out] = DeferState();
    return rc;
}

int mksnap_begin(mksnap_t *h)
{
    const int rc = mock_defer_base_begin(h);
    if (rc == 0) {
        DeferState &d = g_defer[h];
        d.log_used = d.pending = 0;
        d.open_defer.clear();
    }
    return rc;
}

int mksnap_reserve_stream_log(mksnap_t *h, uint64_t bytes)
{
    if (!h)
        return MKSNAP_E_INVAL;
    DeferState &d = g_defer[h];
    if (d.pending)
        return fail(h, MKSNAP_E_STATE, "reserve_stream_log while deferred pieces wait in the log");
    d.log_cap = (bytes + 63) & ~63ull;
    return 0;
}

int mksnap_arena_submit(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
                        const mksnap_range *rng, uint64_t n_rng)
{
    if (!h)
        return MKSNAP_E_INVAL;
    DeferState &d = g_defer[h];
    for (uint64_t i = 0; i < n_rng; ++i) {
        auto it = d.open_defer.find(rng[i].stream);
        if (it != d.open_defer.end() && it->second != ((rng[i].flags & MKSNAP_R_DEFER) != 0))
            return fail(h, MKSNAP_E_INVAL, "a stream mixes MKSNAP_R_DEFER and inline pieces");
    }
    const int rc = mock_defer_base_submit(h, arena_id, used, ext, n_ext, rng, n_rng);
    if (rc)
        return rc;
    for (uint64_t i = 0; i < n_rng; ++i) {
        const mksnap_range &r = rng[i];
        const bool defer = (r.flags & MKSNAP_R_DEFER) != 0;
        if (r.flags & MKSNAP_R_MORE)
            d.open_defer[r.stream] = defer;
        else
            d.open_defer.erase(r.stream);
        if (!defer || !d.log_cap || r.len > d.log_cap)
            continue; // hashed by its own submit
        uint64_t off = (d.log_used + 15) & ~15ull;
        if (off + r.len > d.log_cap) {
            d.flushes++;
            d.pending = 0;
            off = 0;
        }
        d.log_used = off + r.len;
        d.pending++;
    }
    return 0;
}

int mksnap_finish(mksnap_t *h, mksnap_result *out)
{
    const int rc = mock_defer_base_finish(h, out);
    if (rc == 0) {
        DeferState &d = g_defer[h];
        if (d.pending)
            d.flushes++;
        d.pending = d.log_used = 0;
    }
    return rc;
}

uint64_t mock_log_flushes(mksnap_t *h) { return g_defer[h].flushes; }

} // extern "C"
