// mock_mksnap_chunks.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock engine of mock_mksnap.cpp plus the entry points of the
// incremental layer commit (mksnap_chunks_add / mksnap_arena_submit_spans / mksnap_get_cdc) and the chunk table they
// feed (mksnap_get_chunks), restated with the oracle's arithmetic.  tests/test_host_chunk_cache_cpu.py builds this file
// instead of mock_mksnap.cpp and loads it with RTLD_GLOBAL before libmkhost, so the cached commit of libmkhost runs
// against it without a GPU.
//
// The base mock is compiled into this translation unit with the entry points wrapped here renamed.  Like the device,
// a sparse submit sees zeros outside its spans: the mock zeroes those bytes of the arena before the base mock digests
// it, so a packer that left out a byte the engine reads computes a different root than the uncached commit.
#define mksnap_begin mock_base_begin
#define mksnap_destroy mock_base_destroy
#define mksnap_arena_submit mock_base_submit
#define mksnap_finish mock_base_finish
#include "mock_mksnap.cpp"
#undef mksnap_begin
#undef mksnap_destroy
#undef mksnap_arena_submit
#undef mksnap_finish

namespace {
struct Piece {
    uint64_t gbase; // position of the piece's first byte in the concatenation of the submitted arenas
    uint64_t len;
};
struct ChunkState {
    std::vector<uint64_t> ends; // one per row of mksnap::digests
    uint64_t stream_base = 0;   // bytes of the arenas submitted before the current one
    std::vector<Piece> open;    // pieces of the file that spans submits
    std::vector<uint8_t> open_bytes;
    bool overflow = false;
    std::string log; // one line per submit / chunks_add of the session
};
std::map<const mksnap *, ChunkState> g_chunks;
} // namespace

extern "C" {

int mksnap_begin(mksnap_t *h)
{
    const int rc = mock_base_begin(h);
    if (rc == 0)
        g_chunks[h] = ChunkState{};
    return rc;
}

void mksnap_destroy(mksnap_t *h)
{
    g_chunks.erase(h);
    mock_base_destroy(h);
}

int mksnap_get_cdc(const mksnap_t *h, mksnap_cdc_params *out)
{
    if (!h || !out)
        return MKSNAP_E_INVAL;
    mko_cdc_params p;
    mko_cdc_default_params(&p);
    if (h->cfg.cdc.min_size)
        memcpy(&p, &h->cfg.cdc, sizeof p);
    memcpy(out, &p, sizeof p);
    return 0;
}

} // extern "C"

// the base mock digests the chunks; the chunk ends are restated here (the same cut rule over the same bytes)
static int submit_logged(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
                         const mksnap_range *rng, uint64_t n_rng, const std::string &tail)
{
    const size_t rows0 = h ? h->digests.size() / 32 : 0;
    std::vector<uint8_t> arena = h && arena_id >= 0 && (size_t)arena_id < h->arenas.size() ? h->arenas[arena_id] : std::vector<uint8_t>();
    const int rc = mock_base_submit(h, arena_id, used, ext, n_ext, rng, n_rng);
    if (rc)
        return rc;
    ChunkState &cs = g_chunks[h];
    mksnap_cdc_params p;
    mksnap_get_cdc(h, &p);
    uint64_t n_cdc = 0;
    for (uint64_t i = 0; i < n_ext; ++i) {
        const mksnap_extent &e = ext[i];
        if (!(e.flags & MKSNAP_X_CDC))
            continue;
        ++n_cdc;
        cs.open.push_back(Piece{cs.stream_base + e.arena_off, e.len});
        cs.open_bytes.insert(cs.open_bytes.end(), arena.begin() + e.arena_off, arena.begin() + e.arena_off + e.len);
        if (e.flags & MKSNAP_X_MORE)
            continue;
        std::vector<uint64_t> cuts(cs.open_bytes.size() / p.min_size + 2);
        const size_t n = mko_cdc_cuts(cs.open_bytes.data(), cs.open_bytes.size(), (const mko_cdc_params *)&p, cuts.data(), cuts.size());
        for (size_t j = 0; j < n; ++j) { // the piece that holds the chunk's last byte
            uint64_t fstart = 0;
            for (const Piece &pc : cs.open) {
                if (cuts[j] <= fstart + pc.len) {
                    cs.ends.push_back(pc.gbase + (cuts[j] - fstart));
                    break;
                }
                fstart += pc.len;
            }
        }
        cs.open.clear();
        cs.open_bytes.clear();
    }
    if (cs.ends.size() != h->digests.size() / 32)
        return fail(h, MKSNAP_E_STATE, "mock: chunk ends and digests disagree");
    char line[96];
    snprintf(line, sizeof line, "submit used=%llu cdc=%llu rows=%zu", (unsigned long long)used, (unsigned long long)n_cdc,
             h->digests.size() / 32 - rows0);
    cs.log += line + tail + "\n";
    cs.stream_base += used;
    return 0;
}

extern "C" {

int mksnap_arena_submit(mksnap_t *h, int32_t arena_id, uint64_t used, const mksnap_extent *ext, uint64_t n_ext,
                        const mksnap_range *rng, uint64_t n_rng)
{
    return submit_logged(h, arena_id, used, ext, n_ext, rng, n_rng, "");
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
    return submit_logged(h, arena_id, used, ext, n_ext, rng, n_rng, " spans" + sp);
}

int mksnap_chunks_add(mksnap_t *h, const uint8_t *digests, uint64_t n)
{
    if (!h)
        return MKSNAP_E_INVAL;
    if (!h->in_session)
        return fail(h, MKSNAP_E_STATE, "chunks_add outside begin/finish");
    if (n > MKSNAP_CHUNKS_ADD_MAX)
        return fail(h, MKSNAP_E_CAPACITY, "chunks_add: too many rows in one call");
    ChunkState &cs = g_chunks[h];
    if (h->cfg.max_chunks && h->digests.size() / 32 + n > h->cfg.max_chunks) {
        cs.overflow = true; // like the device: nothing is written, finish reports the overflow
        return 0;
    }
    h->digests.insert(h->digests.end(), digests, digests + 32 * n);
    cs.ends.insert(cs.ends.end(), n, UINT64_MAX);
    cs.log += "add " + std::to_string(n) + "\n";
    return 0;
}

int mksnap_finish(mksnap_t *h, mksnap_result *out)
{
    if (h && h->in_session && g_chunks[h].overflow)
        return fail(h, MKSNAP_E_CAPACITY, "chunk table overflow (max_chunks)");
    return mock_base_finish(h, out);
}

int mksnap_get_chunks(mksnap_t *h, uint64_t *ends, uint8_t *digests, uint64_t capacity)
{
    if (!h || !h->finished)
        return h ? fail(h, MKSNAP_E_STATE, "get_chunks before finish") : MKSNAP_E_INVAL;
    const ChunkState &cs = g_chunks[h];
    const uint64_t n = h->digests.size() / 32;
    if (n > capacity)
        return fail(h, MKSNAP_E_CAPACITY, "need more rows");
    if (ends && n)
        memcpy(ends, cs.ends.data(), n * 8);
    if (digests && n)
        memcpy(digests, h->digests.data(), n * 32);
    return 0;
}

// the session's submits and appends as text: "submit used=U cdc=N rows=R[ spans off+len ...]" / "add N"
size_t mock_chunk_log(mksnap_t *h, char *out, size_t cap)
{
    const std::string &s = g_chunks[h].log;
    if (s.size() + 1 <= cap)
        memcpy(out, s.c_str(), s.size() + 1);
    return s.size() + 1;
}

} // extern "C"
