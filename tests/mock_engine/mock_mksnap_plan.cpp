// mock_mksnap_plan.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock engine of mock_mksnap.cpp plus the three entry points of
// plan-level cacheIDs (mksnap_crc_fold / mksnap_get_crc_streams / mksnap_crc_prepend), restated with the oracle's
// arithmetic.  tests/test_host_plan_cache_ids_cpu.py builds this file instead of mock_mksnap.cpp and loads it with
// RTLD_GLOBAL before libmkhost, so the plan code of libmkhost runs against it without a GPU.
//
// The base mock is compiled into this translation unit with its mksnap_begin / mksnap_destroy renamed, so that the
// wrappers below can also reset / drop the stream values a fold leaves behind.
#define mksnap_begin mock_base_begin
#define mksnap_destroy mock_base_destroy
#include "mock_mksnap.cpp"
#undef mksnap_begin
#undef mksnap_destroy

namespace {
// per handle: stream slot -> pure value of the current session
std::map<const mksnap *, std::map<uint32_t, uint32_t>> g_crc_streams;
} // namespace

extern "C" {

int mksnap_begin(mksnap_t *h)
{
    const int rc = mock_base_begin(h);
    if (rc == 0)
        g_crc_streams[h].clear();
    return rc;
}

void mksnap_destroy(mksnap_t *h)
{
    g_crc_streams.erase(h);
    mock_base_destroy(h);
}

// The per-extent table the real engine keeps holds max(4 * max_extents, 2^20) values; this mock keeps 4 * max_extents,
// so that a CPU test can outrun it with a few hundred segments.
int mksnap_crc_fold(mksnap_t *h, const mksnap_crc_use *uses, uint64_t n)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "crc_fold outside begin/finish");
    if (n > h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "crc_fold: too many uses in one call");
    if (h->ext_pure.size() > 4 * h->cfg.max_extents)
        return fail(h, MKSNAP_E_CAPACITY, "crc_fold: the session submitted more CRC extents than the per-extent table keeps");
    for (uint64_t i = 0; i < n; ++i)
        if (uses[i].stream >= h->cfg.max_extents || (uses[i].flags & ~MKSNAP_U_VALUE) ||
            (!(uses[i].flags & MKSNAP_U_VALUE) && uses[i].src >= h->ext_pure.size()))
            return fail(h, MKSNAP_E_INVAL, "crc_fold: use " + std::to_string(i) + " names a stream or extent out of range");
    std::map<uint32_t, uint32_t> &s = g_crc_streams[h];
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t v = (uses[i].flags & MKSNAP_U_VALUE) ? (uint32_t)uses[i].src : h->ext_pure[uses[i].src];
        s[uses[i].stream] ^= mko_crc32_mulmod(v, mko_crc32_xpow8n(uses[i].suffix));
    }
    return 0;
}

int mksnap_get_crc_streams(mksnap_t *h, uint32_t *pure, uint64_t capacity, uint64_t *n_out)
{
    if (!h || !n_out)
        return MKSNAP_E_INVAL;
    if (!h->finished)
        return fail(h, MKSNAP_E_STATE, "get_crc_streams before finish");
    const std::map<uint32_t, uint32_t> &s = g_crc_streams[h];
    *n_out = s.empty() ? 0 : (uint64_t)s.rbegin()->first + 1;
    if (*n_out > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need more entries");
    for (uint64_t k = 0; k < *n_out; ++k) {
        auto it = s.find((uint32_t)k);
        pure[k] = it != s.end() ? it->second : 0u;
    }
    return 0;
}

uint32_t mksnap_crc_prepend(const void *prefix, uint64_t n, uint32_t pure_rest, uint64_t len_rest)
{
    const uint32_t pure = mko_crc32_mulmod(mko_crc32_pure((const uint8_t *)prefix, n), mko_crc32_xpow8n(len_rest)) ^ pure_rest;
    return pure ^ mko_crc32_mulmod(0xFFFFFFFFu, mko_crc32_xpow8n(n + len_rest)) ^ 0xFFFFFFFFu;
}

} // extern "C"
