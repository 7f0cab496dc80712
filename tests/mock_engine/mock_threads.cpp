// mock_threads.cpp -- TEST INFRASTRUCTURE ONLY: the CPU mock of libmksnap with mksnap_get_table (mock_table.cpp, compiled
// into this file unchanged), for calls that drive several mock engines from several threads at once.  The mock keeps
// what its last gunzip open saw (mock_gunzip_candidates, mock_gunzip_records, ...) in process globals that every
// handle's open writes; the device engine has no such state.  Here the two opens take one lock, so concurrent opens on
// different handles are ordered and ThreadSanitizer sees every other access as it is.
#include <mutex>

#define mksnap_gunzip_open mock_gunzip_open_unlocked
#define mksnap_gunzip_open_indexed mock_gunzip_open_indexed_unlocked
#include "mock_table.cpp"
#undef mksnap_gunzip_open
#undef mksnap_gunzip_open_indexed

namespace {
std::mutex g_open_mu; // orders the opens' writes to the mock's last-open globals
} // namespace

extern "C" {

int mksnap_gunzip_open(mksnap_t *h, const void *gz, uint64_t gz_len, mksnap_gunzip_info *info)
{
    std::lock_guard<std::mutex> g(g_open_mu);
    return mock_gunzip_open_unlocked(h, gz, gz_len, info);
}

int mksnap_gunzip_open_indexed(mksnap_t *h, const void *gz, uint64_t gz_len, const uint64_t *points, uint64_t n_points,
                               mksnap_gunzip_info *info)
{
    std::lock_guard<std::mutex> g(g_open_mu);
    return mock_gunzip_open_indexed_unlocked(h, gz, gz_len, points, n_points, info);
}

} // extern "C"
