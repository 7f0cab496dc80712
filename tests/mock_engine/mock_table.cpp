// mock_table.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock of libmksnap (mock_mksnap.cpp, compiled into this file
// unchanged) plus mksnap_get_table, the sorted-unique table of a finished session.  The multi-engine batch commit
// (mkhost_memfs_commit_layers_multi) reads it from every engine but engine 0 and appends it to engine 0's session; no
// single-engine path reads it, so the plain mock leaves it out.
#include "mock_mksnap.cpp"

int mksnap_get_table(mksnap_t *h, uint8_t *table, uint64_t capacity_rows)
{
    if (!h || !h->finished || !table)
        return h ? fail(h, MKSNAP_E_STATE, "get_table before finish") : MKSNAP_E_INVAL;
    std::vector<uint8_t> t = h->ses.digests;
    const size_t n = mko_sort_unique_digests(t.data(), t.size() / 32);
    if (n > capacity_rows)
        return fail(h, MKSNAP_E_CAPACITY, "need more rows");
    if (n)
        memcpy(table, t.data(), n * 32);
    return 0;
}
