// mkhost.cpp — host side above the mksnap C-ABI (see include/mkhost.h).
//
// C++ stand-in for the Go code a cgo build of makisu would keep on this path: the filepath.Walk-ordered
// context stream (cacheID), the MemFS copy-op layer (entry order + tar headers) and the arena packer.
// It does no hashing; digests come from libmksnap (GPU).  Reference line numbers are cited per function.
//
// One translation unit: the *.inc files in this directory are fragments of the anonymous namespace below, included in
// dependency order (Go path helpers, Walk/Glob, context stream, file reader pool, tar writer, tar reader, Copier,
// MemFS, arena packers, cache files); this file holds the C entry points and the fields of each cache file.
#include "../../include/mkhost.h"

#include <dirent.h>
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <condition_variable>
#include <exception>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <stdexcept>
#include <chrono>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

namespace {

struct HostError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

std::string errno_str(const std::string &what, const std::string &path)
{
    return what + " " + path + ": " + strerror(errno);
}

#include "gopath.inc"
#include "gowalk.inc"
#include "context_stream.inc"
#include "reads.inc"
#include "tar_writer.inc"
#include "tar_reader.inc"
#include "copier.inc"
#include "memfs.inc"
#include "packer.inc"
#include "cache_file.inc"

} // namespace

// pure(file content) per context file, remembered between builds (incremental cacheID, include/mkhost.h)
struct mkhost_crc_cache {
    struct Entry {
        FileId id;
        uint32_t pure;
    };
    std::map<std::string, Entry> files; // key: absolute path

    // The file (cache_file.inc): "mkhost-crc-cache 1", then per file a line "<dev> <ino> <size> <mtime ns> <ctime ns>
    // <pure as %08x> <path>", path last: it may hold spaces.
    static constexpr const char *name = "crc", *kind = "crc";
    void encode(CacheWriter &w) const
    {
        w.line("mkhost-crc-cache 1");
        for (const auto &kv : files) {
            char pure[16];
            snprintf(pure, sizeof pure, " %08x", kv.second.pure);
            w.entry(file_id_text(kv.second.id) + pure, kv.first);
        }
    }
    void decode(CacheReader &r)
    {
        if (r.line() != "mkhost-crc-cache 1")
            throw HostError("bad header");
        while (!r.at_end()) {
            const std::string s = r.line();
            Entry x;
            int used = 0, used2 = 0;
            if (!parse_file_id(s.c_str(), &x.id, &used) || sscanf(s.c_str() + used, " %x %n", &x.pure, &used2) != 1 ||
                used2 <= 0 || (size_t)(used + used2) >= s.size())
                throw HostError("bad entry");
            files[s.substr(used + used2)] = x;
        }
    }
    void fold(mkhost_crc_cache &&f) // a loaded file merges into the cache
    {
        for (auto &kv : f.files)
            files[kv.first] = kv.second;
    }
};

// block indexes of gzip blobs per caller key, remembered between builds (include/mkhost.h)
struct mkhost_gz_index_cache {
    GzIndexMap map;

    // "mkhost-gz-index-cache 1", then per blob a line "<gz_len> <n_points> <key>" followed by its points, 8 bytes each
    static constexpr const char *name = "gzip index", *kind = "gz-index";
    void encode(CacheWriter &w) const
    {
        w.line("mkhost-gz-index-cache 1");
        for (const auto &kv : map.e) {
            const std::vector<uint64_t> &pts = kv.second.points;
            if (w.entry(std::to_string(kv.second.gz_len) + " " + std::to_string(pts.size()), kv.first))
                w.bytes(pts.data(), 8 * pts.size());
        }
    }
    void decode(CacheReader &r)
    {
        if (r.line() != "mkhost-gz-index-cache 1")
            throw HostError("bad header");
        while (!r.at_end()) {
            const std::string s = r.line();
            unsigned long long len = 0, pts = 0;
            int used = 0;
            if (sscanf(s.c_str(), "%llu %llu %n", &len, &pts, &used) != 2 || used <= 0 || (size_t)used >= s.size())
                throw HostError("bad entry");
            map.e[s.substr(used)] = GzIndexMap::Entry{len, r.values<uint64_t>(pts)};
        }
    }
    void fold(mkhost_gz_index_cache &&f) { map.e.swap(f.map.e); } // a loaded file replaces the cache
};

// chunk digests per source file, remembered between builds (incremental layer commit, include/mkhost.h)
struct mkhost_chunk_cache {
    ChunkMemo memo;

    // "mkhost-chunk-cache 1 <min> <normal> <max> <strict bits> <loose bits>", then per file a line
    // "<dev> <ino> <size> <mtime ns> <ctime ns> <chunks> <path>" followed by its digests, 32 raw bytes per chunk
    static constexpr const char *name = "chunk", *kind = "chunk";
    void encode(CacheWriter &w) const
    {
        std::string h = "mkhost-chunk-cache 1";
        const mksnap_cdc_params &p = memo.cdc;
        for (uint32_t v : {p.min_size, p.normal_size, p.max_size, p.strict_bits, p.loose_bits})
            h += " " + std::to_string(v);
        w.line(h);
        for (const auto &kv : memo.files) {
            const std::vector<uint8_t> &d = kv.second.digests;
            if (w.entry(file_id_text(kv.second.id) + " " + std::to_string(d.size() / 32), kv.first))
                w.bytes(d.data(), d.size());
        }
    }
    void decode(CacheReader &r)
    {
        mksnap_cdc_params &p = memo.cdc;
        const std::string h = r.line();
        int used = 0;
        if (sscanf(h.c_str(), "mkhost-chunk-cache 1 %u %u %u %u %u%n", &p.min_size, &p.normal_size, &p.max_size,
                   &p.strict_bits, &p.loose_bits, &used) != 5 || (size_t)used != h.size())
            throw HostError("bad header");
        while (!r.at_end()) {
            const std::string s = r.line();
            ChunkMemo::Entry x;
            unsigned long long rows = 0;
            int used2 = 0;
            if (!parse_file_id(s.c_str(), &x.id, &used) || sscanf(s.c_str() + used, " %llu %n", &rows, &used2) != 1 ||
                used2 <= 0 || (size_t)(used + used2) >= s.size() || rows > x.id.size) // a chunk holds at least one byte
                throw HostError("bad entry");
            x.digests = r.rows(rows);
            memo.files[s.substr(used + used2)] = std::move(x);
        }
    }
    void fold(mkhost_chunk_cache &&f) // a loaded file merges into the cache, or replaces one cut under other parameters
    {
        if (memcmp(&f.memo.cdc, &memo.cdc, sizeof memo.cdc) != 0) {
            memo.files.clear();
            memo.cdc = f.memo.cdc; // a commit under other parameters starts over (ChunkMemo::bind)
        }
        for (auto &kv : f.memo.files)
            memo.files[kv.first] = std::move(kv.second);
    }
};

// layer ingests per caller key, remembered between builds (incremental layer ingest, include/mkhost.h)
struct mkhost_layer_cache {
    LayerMemo memo;

    // Binary: the line "mkhost-layer-cache 1", the CDC parameters (5 x u32), the entry count (u64), then per entry: key
    // (u32 length + bytes), file identity (dev, ino, size: u64; mtime, ctime ns: i64), u8 bits (1 gunzip, 2 DiffID,
    // 4 file digests), DiffID (32 bytes), tar_bytes (u64), members (u64 count; each: name and linkname as u32 length +
    // bytes, mode, uid, gid, size as i64, mtime ns as two u64 words, low first, typeflag u8, data_len u64), file digests
    // and chunk digests (u64 count + 32 bytes each).  Nothing follows.
    static constexpr const char *name = "layer", *kind = "layer";
    void encode(CacheWriter &w) const
    {
        w.line("mkhost-layer-cache 1");
        const mksnap_cdc_params &p = memo.cdc;
        for (uint32_t v : {p.min_size, p.normal_size, p.max_size, p.strict_bits, p.loose_bits})
            w.put(v);
        w.put<uint64_t>(memo.e.size());
        for (const auto &kv : memo.e) {
            const LayerMemo::Entry &x = kv.second;
            w.str(kv.first);
            w.put(x.id.dev), w.put(x.id.ino), w.put(x.id.size), w.put(x.id.mtime_ns), w.put(x.id.ctime_ns);
            w.put<uint8_t>((x.gunzip ? 1 : 0) | (x.has_diffid ? 2 : 0) | (x.has_file_digests ? 4 : 0));
            w.bytes(x.diffid.data(), 32);
            w.put(x.tar_bytes);
            w.put<uint64_t>(x.members.size());
            for (const TarMember &m : x.members) {
                const Hdr &h = m.hdr;
                w.str(h.name), w.str(h.linkname);
                w.put(h.mode), w.put(h.uid), w.put(h.gid), w.put(h.size);
                w.put((uint64_t)(unsigned __int128)h.mtime_ns), w.put((uint64_t)((unsigned __int128)h.mtime_ns >> 64));
                w.put<uint8_t>((uint8_t)h.typeflag);
                w.put(m.data_len);
            }
            w.rows(x.file_digests);
            w.rows(x.chunks);
        }
    }
    void decode(CacheReader &r)
    {
        if (r.line() != "mkhost-layer-cache 1")
            throw HostError("bad header");
        mksnap_cdc_params &p = memo.cdc;
        for (uint32_t *v : {&p.min_size, &p.normal_size, &p.max_size, &p.strict_bits, &p.loose_bits})
            *v = r.get<uint32_t>();
        // nothing is sized by a count from the file: a count that lies runs out of file, entry by entry
        for (uint64_t k = r.get<uint64_t>(); k > 0; --k) {
            const std::string key = r.str();
            LayerMemo::Entry x;
            x.id.dev = r.get<uint64_t>(), x.id.ino = r.get<uint64_t>(), x.id.size = r.get<uint64_t>();
            x.id.mtime_ns = r.get<int64_t>(), x.id.ctime_ns = r.get<int64_t>();
            const uint8_t bits = r.get<uint8_t>();
            if (bits & ~7u)
                throw HostError("bad entry");
            x.gunzip = bits & 1, x.has_diffid = bits & 2, x.has_file_digests = bits & 4;
            memcpy(x.diffid.data(), r.take(32), 32);
            x.tar_bytes = r.get<uint64_t>();
            for (uint64_t n = r.get<uint64_t>(); n > 0; --n) {
                TarMember m;
                Hdr &h = m.hdr;
                h.name = r.str(), h.linkname = r.str();
                h.mode = r.get<int64_t>(), h.uid = r.get<int64_t>(), h.gid = r.get<int64_t>(), h.size = r.get<int64_t>();
                const uint64_t lo = r.get<uint64_t>(), hi = r.get<uint64_t>();
                h.mtime_ns = (__int128)(((unsigned __int128)hi << 64) | lo);
                h.typeflag = (char)r.get<uint8_t>();
                m.data_len = r.get<uint64_t>();
                x.members.push_back(std::move(m));
            }
            x.file_digests = r.rows();
            x.chunks = r.rows();
            memo.e[key] = std::move(x);
        }
    }
    void fold(mkhost_layer_cache &&f) { memo = std::move(f.memo); } // a loaded file replaces the cache
};

// persistent snapshot.MemFS mirror (layers accumulate in the merged tree, like context.BuildContext.MemFS)
struct mkhost_memfs {
    MemFS fs;
    mkhost_memfs(const std::string &root, std::vector<std::string> bl) : fs(root, 0, std::move(bl)) {}
};

// =====================================================================================================
extern "C" {

size_t mkhost_encode_tar_header(const mkhost_tar_header *h, uint8_t *out, size_t cap)
{
    try {
        Hdr x;
        x.name = h->name ? h->name : "";
        while (!x.name.empty() && x.name[0] == '/') // write.go:57 strings.TrimLeft(h.Name, "/")
            x.name.erase(0, 1);
        x.linkname = h->linkname ? h->linkname : "";
        x.mode = h->mode; x.uid = h->uid; x.gid = h->gid; x.size = h->size; x.mtime_ns = h->mtime_ns;
        x.typeflag = h->typeflag;
        std::string b = encode_header(x);
        if (b.size() > cap)
            return 0;
        memcpy(out, b.data(), b.size());
        return b.size();
    } catch (const std::exception &) {
        return 0;
    }
}

size_t mkhost_describe_context_stream(const char *context_dir, const char *const *from_paths, size_t n_paths, char *out,
                                      size_t cap, char *err, size_t errlen)
{
    try {
        std::string s;
        for (const auto &g : context_segments(go_clean(context_dir), from_paths, n_paths, 4)) { // 4: the parallel walk is what the parity tests see
            if (g.kind == 'F')
                s += "F " + std::to_string(g.size) + " " + g.path + "\n";
            else
                s += std::string(1, g.kind) + " " + g.bytes + "\n";
        }
        if (s.size() + 1 <= cap)
            memcpy(out, s.c_str(), s.size() + 1);
        return s.size() + 1;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("hash context sources: ") + e.what());
        return 0;
    }
}

size_t mkhost_describe_layer(const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops, char *out,
                             size_t cap, char *err, size_t errlen)
{
    try {
        MemFS fs(root_dir, now_unix);
        return emit_text(describe_layer_text(fs.add_layer_by_copy_ops(ops, n_ops)), out, cap);
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("create layer by copy ops: ") + e.what());
        return 0;
    }
}

mkhost_memfs *mkhost_memfs_new(const char *root_dir, const char *const *blacklist, size_t n_blacklist, char *err,
                               size_t errlen)
{
    try {
        std::vector<std::string> bl;
        for (size_t i = 0; i < n_blacklist; ++i)
            bl.emplace_back(blacklist[i]);
        return new mkhost_memfs(root_dir, std::move(bl));
    } catch (const std::exception &e) {
        set_err(err, errlen, e.what());
        return nullptr;
    }
}

void mkhost_memfs_free(mkhost_memfs *m) { delete m; }

int mkhost_memfs_file_digest(mkhost_memfs *m, const char *dst, uint8_t out[32])
{
    return m && dst && m->fs.get_digest(abs_path(dst), out) ? 0 : 1;
}

size_t mkhost_memfs_describe_copy_ops(mkhost_memfs *m, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops, char *out,
                                      size_t cap, char *err, size_t errlen)
{
    try {
        m->fs.set_now(now_unix);
        return emit_text(describe_layer_text(m->fs.add_layer_by_copy_ops(ops, n_ops)), out, cap);
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("create layer by copy ops: ") + e.what());
        return 0;
    }
}

size_t mkhost_memfs_describe_scan(mkhost_memfs *m, int64_t now_unix, char *out, size_t cap, char *err, size_t errlen)
{
    try {
        m->fs.set_now(now_unix);
        return emit_text(describe_layer_text(m->fs.add_layer_by_scan()), out, cap);
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("create layer by scan: ") + e.what());
        return 0;
    }
}

size_t mkhost_eval_symlinks(const char *path, const char *src_root, char *out, size_t cap, char *err, size_t errlen)
{
    try {
        return emit_text(eval_symlinks(path ? path : "", src_root ? src_root : ""), out, cap);
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("eval symlinks for ") + (path ? path : "") + ": " + e.what());
        return 0;
    }
}

int mkhost_copy_op_execute(const mkhost_copy_op *op, uint32_t mode, const char *const *blacklist, size_t n_blacklist,
                           char *err, size_t errlen)
{
    try {
        if (!op || op->n_srcs == 0)
            throw HostError("check copy param: srcs cannot be empty");
        std::vector<std::string> bl;
        for (size_t i = 0; i < n_blacklist; ++i)
            bl.emplace_back(blacklist[i]);
        std::multimap<std::string, DeferredFile> deferred;
        std::vector<Copier> copiers;
        execute_copy_op(*op, mode, bl, (mode & MKHOST_COPY_DEFERRED) ? &deferred : nullptr, &copiers);
        for (const auto &kv : deferred) { // stand-in for the arena: one read of each source, written from memory
            std::vector<uint8_t> buf((size_t)kv.second.st.st_size);
            std::vector<ReadJob> job{ReadJob{kv.first, 0, (uint64_t)buf.size(), buf.data()}};
            run_reads(job, 1);
            copiers[kv.second.copier].finish_regular(kv.second.st, kv.first, kv.second.dst, buf.data(), buf.size());
        }
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, e.what());
        return -1;
    }
}

int mkhost_memfs_commit_copy_ops(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops,
                                 int n_threads, int tar_fd, uint32_t flags, mkhost_layer_result *out, char *err,
                                 size_t errlen)
{
    return mkhost_memfs_commit_copy_ops_cached(m, eng, nullptr, now_unix, ops, n_ops, n_threads, tar_fd, flags, out, nullptr,
                                               err, errlen);
}

int mkhost_memfs_commit_copy_ops_cached(mkhost_memfs *m, mksnap_t *eng, mkhost_chunk_cache *cache, int64_t now_unix,
                                        const mkhost_copy_op *ops, size_t n_ops, int n_threads, int tar_fd, uint32_t flags,
                                        mkhost_layer_result *out, mkhost_chunk_cache_stats *stats, char *err, size_t errlen)
{
    try {
        m->fs.set_now(now_unix);
        ChunkMemo *memo = cache ? &cache->memo : nullptr;
        if (!(flags & MKHOST_MATERIALIZE)) {
            commit_layer(eng, m->fs.add_layer_by_copy_ops(ops, n_ops), n_threads, tar_fd, flags, out, &m->fs, nullptr, memo, stats);
            return 0;
        }
        // SURVEY section 8f-4: the copy onto the file system (CopyOperation.Execute) and the layer share one read of the
        // context.  Directories, symlinks and chmods first; regular files are written from the arena as it fills;
        // what the layer did not need to read (entries the tree already holds) is copied from disk at the end.
        std::multimap<std::string, DeferredFile> deferred;
        std::vector<Copier> copiers;
        const uint32_t mode = (flags & MKHOST_MATERIALIZE_CHOWN) ? MKHOST_COPY_CHOWN : 0u;
        for (size_t i = 0; i < n_ops; ++i) {
            mkhost_copy_op on_disk = ops[i];
            std::string dst = ops[i].dst ? ops[i].dst : "";
            const bool dir_fmt = (!dst.empty() && dst.back() == '/') || dst == "." || dst == "..";
            if (dst.empty() || dst[0] != '/') {
                if (!ops[i].work_dir || ops[i].work_dir[0] != '/')
                    throw HostError("check copy param: dst is not absolute path, must specify absolute working directory");
                dst = go_join(ops[i].work_dir, dst);
            }
            dst = go_join(m->fs.root(), dst) + (dir_fmt ? "/" : ""); // image path -> path under the MemFS root ("/" in a real build)
            on_disk.dst = dst.c_str();
            execute_copy_op(on_disk, mode, m->fs.blacklist(), &deferred, &copiers);
        }
        auto write_from_arena = [&](const std::vector<ReadJob> &jobs) {
            for (const auto &j : jobs) {
                if (j.file_off != 0)
                    continue;
                auto range = deferred.equal_range(j.path);
                if (range.first == range.second || (uint64_t)range.first->second.st.st_size != j.len)
                    continue; // a piece of a file larger than the arena: that file is copied from disk at the end
                for (auto it = range.first; it != range.second; ++it)
                    copiers[it->second.copier].finish_regular(it->second.st, j.path, it->second.dst, j.dst, j.len);
                deferred.erase(range.first, range.second);
            }
        };
        commit_layer(eng, m->fs.add_layer_by_copy_ops(ops, n_ops), n_threads, tar_fd, flags, out, &m->fs, write_from_arena, memo,
                     stats);
        for (const auto &kv : deferred)
            copiers[kv.second.copier].finish_regular(kv.second.st, kv.first, kv.second.dst, nullptr, 0);
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("failed to generate diff layer: ") + e.what());
        return -1;
    }
}

int mkhost_memfs_commit_layers(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_layer_spec *specs, size_t n_layers,
                               int n_threads, uint32_t flags, mkhost_layer_result *outs, char *err, size_t errlen)
{
    return mkhost_memfs_commit_layers_cached(m, eng, nullptr, now_unix, specs, n_layers, n_threads, flags, outs, nullptr, err,
                                             errlen);
}

int mkhost_memfs_commit_layers_cached(mkhost_memfs *m, mksnap_t *eng, mkhost_chunk_cache *cache, int64_t now_unix,
                                      const mkhost_layer_spec *specs, size_t n_layers, int n_threads, uint32_t flags,
                                      mkhost_layer_result *outs, mkhost_chunk_cache_stats *stats, char *err, size_t errlen)
{
    return mkhost_memfs_commit_layers_multi(m, &eng, 1, cache, now_unix, specs, n_layers, n_threads, flags, outs, stats, err,
                                            errlen);
}

int mkhost_memfs_commit_layers_multi(mkhost_memfs *m, mksnap_t *const *engines, size_t n_engines, mkhost_chunk_cache *cache,
                                     int64_t now_unix, const mkhost_layer_spec *specs, size_t n_layers, int n_threads,
                                     uint32_t flags, mkhost_layer_result *outs, mkhost_chunk_cache_stats *stats, char *err,
                                     size_t errlen)
{
    try {
        if (!m || !engines || n_engines == 0 || (!specs && n_layers) || (!outs && n_layers))
            throw HostError("null argument");
        for (size_t k = 0; k < n_engines; ++k)
            if (!engines[k])
                throw HostError("null argument");
        if (flags & ~(uint32_t)(MKHOST_NO_TAR_DIGEST | MKHOST_FILE_DIGESTS))
            throw HostError("commit layers: only MKHOST_NO_TAR_DIGEST and MKHOST_FILE_DIGESTS are supported for a batch");
        m->fs.set_now(now_unix);
        // the layer maps are built in order -- each AddLayerByCopyOps sees the tree its predecessors left
        // (mem_fs.go:276-289) -- and only then packed together
        std::vector<std::map<std::string, MemFile>> maps;
        maps.reserve(n_layers);
        for (size_t i = 0; i < n_layers; ++i)
            maps.push_back(m->fs.add_layer_by_copy_ops(specs[i].ops, specs[i].n_ops));
        std::vector<BatchLayer> bl;
        for (size_t i = 0; i < n_layers; ++i)
            bl.push_back(BatchLayer{&maps[i], specs[i].tar_fd});
        commit_layers_batch(engines, n_engines, bl, n_threads, flags, outs, &m->fs, cache ? &cache->memo : nullptr, stats);
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("failed to generate diff layers: ") + e.what());
        return -1;
    }
}

int mkhost_memfs_commit_scan(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, int n_threads, int tar_fd, uint32_t flags,
                             mkhost_layer_result *out, char *err, size_t errlen)
{
    try {
        m->fs.set_now(now_unix);
        if (!(flags & MKHOST_SCAN_CONTENT)) {
            commit_layer(eng, m->fs.add_layer_by_scan(), n_threads, tar_fd, flags, out, &m->fs);
            return 0;
        }
        // content-aware scan (SURVEY section 8f-3): the reference trusts mtime+size and therefore sync()s and sleeps
        // a second before every scan (mem_fs.go:291-311); here files the metadata calls unchanged are re-hashed on
        // the GPU and compared with the digest remembered when they were committed.
        std::vector<Suspect> suspects;
        std::map<std::string, MemFile> layer = m->fs.add_layer_by_scan(&suspects);
        const std::vector<std::array<uint8_t, 32>> now = digest_files(eng, suspects, n_threads);
        for (size_t k = 0; k < suspects.size(); ++k)
            if (now[k] != suspects[k].known)
                m->fs.add_changed(layer, suspects[k]);
        commit_layer(eng, layer, n_threads, tar_fd, flags, out, &m->fs);
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("failed to generate diff layer: ") + e.what());
        return -1;
    }
}

size_t mkhost_memfs_describe_update_from_tar_ex(mkhost_memfs *m, int64_t now_unix, int tar_fd, uint32_t flags, char *out,
                                                size_t cap, char *err, size_t errlen)
{
    try {
        if (flags & MKHOST_GUNZIP)
            throw HostError("MKHOST_GUNZIP: the describe functions read uncompressed tars only");
        m->fs.set_now(now_unix);
        std::vector<uint8_t> buf;
        uint8_t tmp[65536];
        uint64_t r;
        do {
            r = read_full(tar_fd, tmp, sizeof tmp, "read header");
            buf.insert(buf.end(), tmp, tmp + r);
        } while (r == sizeof tmp);
        MemTarSource src(buf.data(), buf.size());
        if (flags & MKHOST_UNTAR) {
            MemFS::Untar u;
            read_tar(src, [&](const TarMember &mem, const uint8_t *body) { m->fs.untar_member(u, mem, body); });
            return emit_text(describe_layer_text(m->fs.untar_finish(u)), out, cap);
        }
        return emit_text(describe_layer_text(m->fs.update_from_tar(read_tar(src))), out, cap);
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("update memfs from tar: ") + e.what());
        return 0;
    }
}

size_t mkhost_memfs_describe_update_from_tar(mkhost_memfs *m, int64_t now_unix, int tar_fd, char *out, size_t cap, char *err,
                                             size_t errlen)
{
    return mkhost_memfs_describe_update_from_tar_ex(m, now_unix, tar_fd, 0, out, cap, err, errlen);
}

} // extern "C"

namespace {

// mkhost_memfs_update_from_tars; with `cache`, mkhost_memfs_update_from_tars_indexed (keys[i] for layer i); with `lc`,
// mkhost_memfs_update_from_tars_cached.  tar_flags: the range flags of the layers' tar streams (MKSNAP_R_DEFER for a
// run, which then reserves the stream log; 0 for a single layer, whose one stream stays inline).  `what` prefixes errors.
int update_from_tars_impl(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_tar_spec *layers,
                          size_t n_layers, uint32_t flags, uint32_t tar_flags, mkhost_layer_result *outs, GzIndexMap *cache,
                          const char *const *keys, mkhost_gz_index_stats *stats, LayerMemo *lc,
                          mkhost_layer_cache_stats *lstats, const char *what, char *err, size_t errlen)
{
    try {
        if (!m || !eng || (!layers && n_layers) || (!outs && n_layers))
            throw HostError("null argument");
        if (flags & ~(uint32_t)(MKHOST_NO_TAR_DIGEST | MKHOST_FILE_DIGESTS | MKHOST_UNTAR))
            throw HostError("update from tars: flags take MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS and MKHOST_UNTAR; "
                            "MKHOST_GUNZIP goes per layer");
        for (size_t i = 0; i < n_layers; ++i)
            if (layers[i].flags & ~(uint32_t)MKHOST_GUNZIP)
                throw HostError("update from tars: layer " + std::to_string(i) + ": only MKHOST_GUNZIP is a per-layer flag");
        if (n_layers == 0)
            return 0;
        m->fs.set_now(now_unix);
        const bool want_digest = !(flags & MKHOST_NO_TAR_DIGEST);
        const bool file_digests = (flags & MKHOST_FILE_DIGESTS) != 0;
        const mksnap_limits lim = engine_limits(eng);
        if (n_layers + (file_digests ? 1 : 0) > lim.max_streams)
            throw HostError("a run of " + std::to_string(n_layers) + " layers needs a stream slot per layer" +
                            (file_digests ? " and more for the per-file digests" : "") + ": engine max_extents (" +
                            std::to_string(lim.max_streams) + ") is too small");
        // layer i's DiffID is stream slot i; under MKSNAP_R_DEFER the engine keeps its bytes in the stream log and hashes
        // the chains of the whole run together.  Per-file streams are inline, in the slots after the layers.
        const uint32_t file_base = (uint32_t)n_layers;
        if (lc)
            lc->bind(eng);
        mkhost_layer_cache_stats lst{};
        lst.layers = n_layers;
        ck(eng, mksnap_begin(eng), "begin");
        if (want_digest && (tar_flags & MKSNAP_R_DEFER))
            ck(eng, mksnap_reserve_stream_log(eng, RUN_STREAM_LOG_BYTES), "reserve stream log");
        std::vector<uint64_t> entries(n_layers), tar_bytes(n_layers);
        std::vector<uint8_t> d;    // stream-digest rows [0, file_base + most file streams of a layer so far)
        uint32_t max_files = 0;
        // layer cache: the DiffID of each replayed layer, the entry each recorded layer will leave (written after finish,
        // when the DiffIDs exist), and where each layer's submitted bytes start in the session's chunk-end coordinates
        std::vector<std::unique_ptr<std::array<uint8_t, 32>>> replayed(n_layers);
        std::vector<std::unique_ptr<LayerMemo::Entry>> recording(n_layers);
        std::vector<uint64_t> session_at(n_layers + 1, 0);
        for (size_t i = 0; i < n_layers; ++i) {
            // the layers join the tree (and the disk) strictly in order: whiteouts, overwrites and hard links of
            // layer i + 1 act on what layer i left
            const uint32_t lflags = flags | layers[i].flags;
            const char *key = keys ? keys[i] : nullptr;
            FileId id;
            const bool cacheable = lc && key && layer_file_id(layers[i].tar_fd, &id);
            const LayerMemo::Entry *hit = cacheable && !(flags & MKHOST_UNTAR) ? lc->find(key, id, lflags) : nullptr;
            session_at[i + 1] = session_at[i];
            if (hit) { // replay: no read, no gunzip, no submit
                IngestedLayer in;
                in.members = hit->members;
                const std::map<std::string, MemFile> layer = merge_layer(m->fs, flags, in, hit->file_digests.data(), 0);
                const uint64_t n = hit->chunks.size() / 32;
                for (uint64_t r0 = 0; r0 < n; r0 += MKSNAP_CHUNKS_ADD_MAX)
                    ck(eng, mksnap_chunks_add(eng, hit->chunks.data() + 32 * r0, std::min<uint64_t>(MKSNAP_CHUNKS_ADD_MAX, n - r0)),
                       "chunks add");
                replayed[i].reset(new std::array<uint8_t, 32>(hit->diffid));
                entries[i] = layer.size();
                tar_bytes[i] = hit->tar_bytes;
                lst.layers_replayed++;
                lst.chunks_appended += n;
                continue;
            }
            IngestedLayer in;
            const GzIndexUse ix{cache, key, stats};
            ingest_layer(m->fs, eng, layers[i].tar_fd, lflags, (uint32_t)i, tar_flags, file_base, in,
                         cache && ix.key ? &ix : nullptr);
            if (in.n_file_streams) { // inline streams: their rows are final once the submits so far have run
                max_files = std::max(max_files, in.n_file_streams);
                d.assign(((uint64_t)file_base + max_files) * 32, 0);
                ck(eng, mksnap_get_stream_digests(eng, d.data(), file_base + max_files), "stream digests");
            }
            const std::map<std::string, MemFile> layer = merge_layer(m->fs, flags, in, d.data(), file_base);
            entries[i] = layer.size();
            tar_bytes[i] = in.tar_bytes;
            session_at[i + 1] += in.submitted;
            lst.blob_bytes_read += in.blob_bytes;
            if (cacheable) {
                recording[i].reset(new LayerMemo::Entry);
                LayerMemo::Entry &r = *recording[i];
                r.id = id;
                r.gunzip = (lflags & MKHOST_GUNZIP) != 0;
                r.has_diffid = want_digest;
                r.has_file_digests = file_digests;
                r.tar_bytes = in.tar_bytes;
                r.members = std::move(in.members);
                if (in.n_file_streams) // rows file_base .. file_base + n_file_streams - 1 of d are this layer's files
                    r.file_digests.assign(d.begin() + 32 * file_base, d.begin() + 32 * ((uint64_t)file_base + in.n_file_streams));
            }
        }
        mksnap_result res;
        ck(eng, mksnap_finish(eng, &res), "finish");
        std::vector<uint8_t> rows(std::max<uint64_t>(res.n_streams, n_layers) * 32, 0);
        if (want_digest)
            ck(eng, mksnap_get_stream_digests(eng, rows.data(), rows.size() / 32), "stream digests");
        for (size_t i = 0; i < n_layers; ++i) { // root: chunk table of the whole run (one session)
            if (replayed[i])
                memcpy(rows.data() + 32 * i, replayed[i]->data(), 32);
            set_layer_result(&outs[i], res, want_digest ? rows.data() + 32 * i : nullptr, entries[i], tar_bytes[i]);
        }
        if (std::any_of(recording.begin(), recording.end(), [](const auto &r) { return r != nullptr; })) {
            // Every layer submitted arenas of its own, so the chunks it computed end inside its share of the session's
            // bytes, (session_at[i], session_at[i + 1]]; rows appended for replayed layers carry end = UINT64_MAX.
            std::vector<uint64_t> ends(std::max<uint64_t>(1, res.n_chunks));
            std::vector<uint8_t> dig(32 * ends.size());
            if (res.n_chunks)
                ck(eng, mksnap_get_chunks(eng, ends.data(), dig.data(), res.n_chunks), "chunk table");
            for (uint64_t c = 0; c < res.n_chunks; ++c) {
                if (ends[c] == UINT64_MAX)
                    continue;
                if (ends[c] == 0 || ends[c] > session_at[n_layers])
                    throw HostError("internal: the chunk table does not match the layers submitted");
                const size_t i = std::upper_bound(session_at.begin(), session_at.end(), ends[c] - 1) - session_at.begin() - 1;
                if (recording[i])
                    recording[i]->chunks.insert(recording[i]->chunks.end(), dig.begin() + 32 * c, dig.begin() + 32 * (c + 1));
            }
            for (size_t i = 0; i < n_layers; ++i) {
                if (!recording[i])
                    continue;
                if (want_digest)
                    memcpy(recording[i]->diffid.data(), rows.data() + 32 * i, 32);
                lc->e[keys[i]] = std::move(*recording[i]);
                lst.layers_recorded++;
            }
        }
        if (lstats)
            *lstats = lst;
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, what + std::string(e.what()));
        return -1;
    }
}

// mkhost_memfs_update_from_tars_multi (one engine: update_from_tars_impl).  Without MKHOST_UNTAR an ingest never touches the
// tree, so whole layers go to the engines and only their merges keep the run's order:
//  - On this thread, before any engine starts: the layer cache decides which layers are replayed (they need no engine
//    until the end), and the ingested layers go to the engines by LPT over their blob lengths, the layers of one key
//    together (a key's gz index entry is then read and written by one engine, in layer order).
//  - Each engine ingests its share, ascending, in a session of its own on a thread of its own: DiffID streams in slots
//    0..share-1 (MKSNAP_R_DEFER, with its own stream log), per-file streams behind them, their rows taken after each
//    layer.  Its gz lookups see the entries its own earlier layers left, then the cache as the call found it.  An
//    engine stops at its first failing layer.  Every engine finishes its own session on its own thread, so the
//    engines' DiffID chains are hashed at the same time (each finish flushes its stream log), and hands over its
//    DiffIDs, its computed chunk rows and its sorted-unique table.
//  - Then this thread merges the layers in order up to the first that failed (ingest or merge), applies the gz entries
//    of the layers up to that one in order, and reports that layer's failure, as the single call would have.
//  - A last, short session on engine 0 takes every engine's unique table and the replayed layers' chunk rows
//    (mksnap_chunks_add) and finishes: the run's root and n_unique.  Each engine's computed chunk rows go to its own
//    layers through its own session coordinates, and the layer cache is written, as in the single call.
int update_from_tars_sharded(mkhost_memfs *m, mksnap_t *const *engines, size_t n_engines, int64_t now_unix,
                             const mkhost_tar_spec *layers, size_t n_layers, uint32_t flags, mkhost_layer_result *outs,
                             GzIndexMap *cache, const char *const *keys, mkhost_gz_index_stats *stats, LayerMemo *lc,
                             mkhost_layer_cache_stats *lstats, char *err, size_t errlen)
{
    try {
        if (!m || !engines || n_engines == 0 || (!layers && n_layers) || (!outs && n_layers))
            throw HostError("null argument");
        for (size_t k = 0; k < n_engines; ++k)
            if (!engines[k])
                throw HostError("null argument");
        if (flags & ~(uint32_t)(MKHOST_NO_TAR_DIGEST | MKHOST_FILE_DIGESTS | MKHOST_UNTAR))
            throw HostError("update from tars: flags take MKHOST_NO_TAR_DIGEST, MKHOST_FILE_DIGESTS and MKHOST_UNTAR; "
                            "MKHOST_GUNZIP goes per layer");
        for (size_t i = 0; i < n_layers; ++i)
            if (layers[i].flags & ~(uint32_t)MKHOST_GUNZIP)
                throw HostError("update from tars: layer " + std::to_string(i) + ": only MKHOST_GUNZIP is a per-layer flag");
        if (n_engines == 1)
            return update_from_tars_impl(m, engines[0], now_unix, layers, n_layers, flags, MKSNAP_R_DEFER, outs, cache, keys,
                                         stats, lc, lstats, "update memfs from tars: ", err, errlen);
        if (flags & MKHOST_UNTAR)
            throw HostError("update from tars: MKHOST_UNTAR writes the members while the layers are read, so it takes one engine");
        check_same_cdc(engines, n_engines);
        if (n_layers == 0)
            return 0;
        const bool want_digest = !(flags & MKHOST_NO_TAR_DIGEST);
        const bool file_digests = (flags & MKHOST_FILE_DIGESTS) != 0;
        // the layer cache is bound (and cleared when cut under other CDC parameters) only once nothing is refused; a
        // cache that binding would clear replays nothing
        mksnap_cdc_params cdc0;
        ck(engines[0], mksnap_get_cdc(engines[0], &cdc0), "cdc parameters");
        const bool lc_valid = lc && memcmp(&cdc0, &lc->cdc, sizeof cdc0) == 0;
        mkhost_layer_cache_stats lst{};
        lst.layers = n_layers;

        // the plan: replayed layers, and the ingested ones shared out in units of one key
        std::vector<const LayerMemo::Entry *> hit(n_layers, nullptr);
        std::vector<FileId> id(n_layers);
        std::vector<bool> cacheable(n_layers, false);
        std::vector<uint64_t> unit_weight;
        std::vector<std::vector<size_t>> unit_layers;
        std::map<std::string, size_t> unit_of_key;
        for (size_t i = 0; i < n_layers; ++i) {
            const char *key = keys ? keys[i] : nullptr;
            cacheable[i] = lc && key && layer_file_id(layers[i].tar_fd, &id[i]);
            hit[i] = cacheable[i] && lc_valid ? lc->find(key, id[i], flags | layers[i].flags) : nullptr;
            if (hit[i])
                continue;
            struct stat st;
            const uint64_t w = fstat(layers[i].tar_fd, &st) == 0 && S_ISREG(st.st_mode) ? (uint64_t)st.st_size : 0;
            size_t u = unit_weight.size();
            if (key) {
                auto ins = unit_of_key.emplace(key, u);
                u = ins.first->second;
            }
            if (u == unit_weight.size()) {
                unit_weight.push_back(0);
                unit_layers.emplace_back();
            }
            unit_weight[u] += w;
            unit_layers[u].push_back(i);
        }
        const std::vector<std::vector<size_t>> unit_share = lpt_shares(unit_weight, n_engines);

        struct Shard {
            std::vector<size_t> ingests; // its layers, ascending: local stream slot j <-> ingests[j]
            std::vector<uint64_t> at{0}; // where ingests[j]'s submitted bytes start in the session's chunk-end coordinates
            uint32_t max_files = 0;      // most per-file streams of one of its layers so far
            GzIndexMap own;              // gz entries its layers left in this call
            mkhost_gz_index_stats gst{};
            mksnap_result res{};
            std::vector<uint8_t> rows, dig, table; // DiffID rows; computed chunk digests (with ends) and unique table
            std::vector<uint64_t> ends;
            std::exception_ptr failed;             // a failure that belongs to no layer (finish, chunk table)
        };
        std::vector<Shard> sh(n_engines);
        for (size_t k = 0; k < n_engines; ++k) {
            for (size_t u : unit_share[k])
                sh[k].ingests.insert(sh[k].ingests.end(), unit_layers[u].begin(), unit_layers[u].end());
            std::sort(sh[k].ingests.begin(), sh[k].ingests.end());
        }
        size_t n_used = 1; // engines given nothing stay untouched; engine 0 always finishes the run
        for (size_t k = 1; k < n_engines; ++k)
            if (!sh[k].ingests.empty())
                n_used = k + 1;
        for (size_t k = 0; k < n_used; ++k) {
            if (sh[k].ingests.empty())
                continue;
            const mksnap_limits lim = engine_limits(engines[k]);
            const size_t L = sh[k].ingests.size();
            if (L + (file_digests ? 1 : 0) > lim.max_streams)
                throw HostError("engine " + std::to_string(k) + "'s share of " + std::to_string(L) +
                                " layers needs a stream slot per layer" + (file_digests ? " and more for the per-file digests" : "") +
                                ": engine max_extents (" + std::to_string(lim.max_streams) + ") is too small");
        }
        m->fs.set_now(now_unix);
        if (lc)
            lc->bind(engines[0]);

        struct Layer {
            IngestedLayer in;
            std::vector<uint8_t> file_rows; // its per-file digests, member order
            std::unique_ptr<GzIndexMap::Entry> gz;
            bool ran = false;
            std::string failed;
        };
        std::vector<Layer> lay(n_layers);
        for (size_t i = 0; i < n_layers; ++i)
            lay[i].ran = hit[i] != nullptr; // a replayed layer has nothing to run before its merge
        EngineThreads threads(n_used);
        threads.run([&](size_t k) {
            Shard &s = sh[k];
            if (s.ingests.empty())
                return;
            mksnap_t *eng = engines[k];
            const uint32_t file_base = (uint32_t)s.ingests.size();
            try {
                ck(eng, mksnap_begin(eng), "begin");
                if (want_digest)
                    ck(eng, mksnap_reserve_stream_log(eng, RUN_STREAM_LOG_BYTES), "reserve stream log");
            } catch (const std::exception &e) { // the first layer's failure, as in the single call
                lay[s.ingests[0]].failed = e.what();
                return;
            }
            for (size_t j = 0; j < s.ingests.size(); ++j) {
                const size_t i = s.ingests[j];
                Layer &l = lay[i];
                try {
                    const char *key = keys ? keys[i] : nullptr;
                    const GzIndexUse ix{&s.own, key, &s.gst, cache};
                    ingest_layer(m->fs, eng, layers[i].tar_fd, flags | layers[i].flags, (uint32_t)j, MKSNAP_R_DEFER, file_base, l.in,
                                 cache && key ? &ix : nullptr);
                    if (l.in.gz_indexed)
                        l.gz.reset(new GzIndexMap::Entry(s.own.e[key]));
                    if (l.in.n_file_streams) { // inline streams: their rows are final once the submits so far have run
                        s.max_files = std::max(s.max_files, l.in.n_file_streams);
                        std::vector<uint8_t> d(32 * ((uint64_t)file_base + s.max_files));
                        ck(eng, mksnap_get_stream_digests(eng, d.data(), d.size() / 32), "stream digests");
                        l.file_rows.assign(d.begin() + 32 * file_base, d.begin() + 32 * ((uint64_t)file_base + l.in.n_file_streams));
                    }
                    s.at.push_back(s.at.back() + l.in.submitted);
                    l.ran = true;
                } catch (const std::exception &e) {
                    if (l.in.gz_indexed && !l.gz)
                        l.gz.reset(new GzIndexMap::Entry(s.own.e[keys[i]]));
                    l.failed = e.what();
                    return;
                }
            }
            try {
                ck(eng, mksnap_finish(eng, &s.res), "finish");
                s.rows.assign(32 * std::max<uint64_t>(s.res.n_streams, file_base), 0);
                if (want_digest && !s.rows.empty())
                    ck(eng, mksnap_get_stream_digests(eng, s.rows.data(), s.rows.size() / 32), "stream digests");
                s.ends.resize(std::max<uint64_t>(1, s.res.n_chunks));
                s.dig.resize(32 * s.ends.size());
                if (lc && s.res.n_chunks)
                    ck(eng, mksnap_get_chunks(eng, s.ends.data(), s.dig.data(), s.res.n_chunks), "chunk table");
                s.table.resize(32 * s.res.n_unique);
                if (s.res.n_unique)
                    ck(eng, mksnap_get_table(eng, s.table.data(), s.res.n_unique), "chunk table");
            } catch (...) {
                s.failed = std::current_exception();
            }
        });

        // merge in layer order, up to the first layer that failed
        std::vector<uint64_t> entries(n_layers, 0);
        size_t first_bad = n_layers;
        std::string why;
        for (size_t i = 0; i < n_layers && first_bad == n_layers; ++i) {
            Layer &l = lay[i];
            if (!l.ran) {
                first_bad = i;
                why = l.failed;
                break;
            }
            try {
                IngestedLayer replay;
                if (hit[i])
                    replay.members = hit[i]->members;
                const std::map<std::string, MemFile> merged =
                    hit[i] ? merge_layer(m->fs, flags, replay, hit[i]->file_digests.data(), 0) : merge_layer(m->fs, flags, l.in, l.file_rows.data(), 0);
                entries[i] = merged.size();
            } catch (const std::exception &e) {
                first_bad = i;
                why = e.what();
            }
        }
        if (cache)
            for (size_t i = 0; i < n_layers && i <= first_bad; ++i)
                if (lay[i].gz)
                    cache->e[keys[i]] = std::move(*lay[i].gz);
        if (first_bad < n_layers)
            throw HostError(why);
        for (size_t k = 0; k < n_used; ++k)
            if (sh[k].failed)
                std::rethrow_exception(sh[k].failed);
        if (stats)
            for (const Shard &s : sh) {
                stats->blobs += s.gst.blobs;
                stats->blobs_with_index += s.gst.blobs_with_index;
                stats->points_given += s.gst.points_given;
                stats->points_linked += s.gst.points_linked;
                stats->points_recorded += s.gst.points_recorded;
            }

        // One more session on engine 0 holds the run's table: every engine's unique rows and the replayed layers' rows.
        // Its finish sorts, uniques and roots them, so root and n_unique are those of one table over the run; n_chunks
        // counts every engine's computed chunks and every replayed row, as the single call's table does.
        mksnap_t *eng0 = engines[0];
        std::vector<const std::vector<uint8_t> *> tables;
        for (size_t k = 0; k < n_used; ++k)
            tables.push_back(&sh[k].table);
        for (size_t i = 0; i < n_layers; ++i)
            if (hit[i])
                tables.push_back(&hit[i]->chunks);
        ck(eng0, mksnap_begin(eng0), "begin");
        for (const std::vector<uint8_t> *rows : tables) {
            const uint64_t n = rows->size() / 32;
            for (uint64_t r0 = 0; r0 < n; r0 += MKSNAP_CHUNKS_ADD_MAX)
                ck(eng0, mksnap_chunks_add(eng0, rows->data() + 32 * r0, std::min<uint64_t>(MKSNAP_CHUNKS_ADD_MAX, n - r0)),
                   "chunks add");
        }
        mksnap_result res;
        ck(eng0, mksnap_finish(eng0, &res), "finish");
        res.n_chunks = 0;
        for (size_t k = 0; k < n_used; ++k)
            res.n_chunks += sh[k].res.n_chunks;
        for (size_t i = 0; i < n_layers; ++i)
            if (hit[i])
                res.n_chunks += hit[i]->chunks.size() / 32;

        std::vector<std::unique_ptr<LayerMemo::Entry>> recording(n_layers);
        for (size_t k = 0; k < n_used; ++k) {
            const Shard &s = sh[k];
            for (size_t j = 0; j < s.ingests.size(); ++j) {
                const size_t i = s.ingests[j];
                const IngestedLayer &in = lay[i].in;
                set_layer_result(&outs[i], res, want_digest ? s.rows.data() + 32 * j : nullptr, entries[i], in.tar_bytes);
                lst.blob_bytes_read += in.blob_bytes;
                if (!cacheable[i])
                    continue;
                recording[i].reset(new LayerMemo::Entry);
                LayerMemo::Entry &r = *recording[i];
                r.id = id[i];
                r.gunzip = (layers[i].flags & MKHOST_GUNZIP) != 0;
                r.has_diffid = want_digest;
                r.has_file_digests = file_digests;
                r.tar_bytes = in.tar_bytes;
                r.members = std::move(lay[i].in.members);
                r.file_digests = std::move(lay[i].file_rows);
                if (want_digest)
                    memcpy(r.diffid.data(), s.rows.data() + 32 * j, 32);
            }
            if (!lc)
                continue;
            // Every ingested layer submitted arenas of its own, so the chunks it computed end inside its share of this
            // engine's session bytes, (at[j], at[j + 1]].
            for (uint64_t c = 0; c < s.res.n_chunks; ++c) {
                if (s.ends[c] == 0 || s.ends[c] > s.at.back())
                    throw HostError("internal: the chunk table does not match the layers submitted");
                const size_t j = std::upper_bound(s.at.begin(), s.at.end(), s.ends[c] - 1) - s.at.begin() - 1;
                if (recording[s.ingests[j]])
                    recording[s.ingests[j]]->chunks.insert(recording[s.ingests[j]]->chunks.end(), s.dig.begin() + 32 * c,
                                                           s.dig.begin() + 32 * (c + 1));
            }
        }
        for (size_t i = 0; i < n_layers; ++i) {
            if (hit[i]) {
                set_layer_result(&outs[i], res, want_digest ? hit[i]->diffid.data() : nullptr, entries[i], hit[i]->tar_bytes);
                lst.layers_replayed++;
                lst.chunks_appended += hit[i]->chunks.size() / 32;
            } else if (recording[i]) {
                lc->e[keys[i]] = std::move(*recording[i]);
                lst.layers_recorded++;
            }
        }
        if (lstats)
            *lstats = lst;
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("update memfs from tars: ") + e.what());
        return -1;
    }
}

} // namespace

extern "C" {

int mkhost_memfs_update_from_tar(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, int tar_fd, uint32_t flags,
                                 mkhost_layer_result *out, char *err, size_t errlen)
{
    return mkhost_memfs_update_from_tar_indexed(m, eng, nullptr, nullptr, now_unix, tar_fd, flags, out, nullptr, err, errlen);
}

int mkhost_memfs_update_from_tars(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_tar_spec *layers,
                                  size_t n_layers, uint32_t flags, mkhost_layer_result *outs, char *err, size_t errlen)
{
    return mkhost_memfs_update_from_tars_cached(m, eng, nullptr, nullptr, nullptr, now_unix, layers, n_layers, flags, outs,
                                                nullptr, nullptr, err, errlen);
}

// a single layer is a run of one whose DiffID stream stays inline; flag bits the run does not take are ignored
int mkhost_memfs_update_from_tar_indexed(mkhost_memfs *m, mksnap_t *eng, mkhost_gz_index_cache *cache, const char *key,
                                         int64_t now_unix, int tar_fd, uint32_t flags, mkhost_layer_result *out,
                                         mkhost_gz_index_stats *stats, char *err, size_t errlen)
{
    const mkhost_tar_spec layer{tar_fd, flags & MKHOST_GUNZIP};
    return update_from_tars_impl(m, eng, now_unix, &layer, 1, flags & (MKHOST_NO_TAR_DIGEST | MKHOST_FILE_DIGESTS | MKHOST_UNTAR),
                                 0, out, cache ? &cache->map : nullptr, &key, stats, nullptr, nullptr,
                                 "update memfs from tar: ", err, errlen);
}

int mkhost_memfs_update_from_tars_indexed(mkhost_memfs *m, mksnap_t *eng, mkhost_gz_index_cache *cache,
                                          const char *const *keys, int64_t now_unix, const mkhost_tar_spec *layers,
                                          size_t n_layers, uint32_t flags, mkhost_layer_result *outs,
                                          mkhost_gz_index_stats *stats, char *err, size_t errlen)
{
    return mkhost_memfs_update_from_tars_cached(m, eng, nullptr, cache, keys, now_unix, layers, n_layers, flags, outs, nullptr,
                                                stats, err, errlen);
}

int mkhost_memfs_update_from_tars_cached(mkhost_memfs *m, mksnap_t *eng, mkhost_layer_cache *lc, mkhost_gz_index_cache *gz,
                                         const char *const *keys, int64_t now_unix, const mkhost_tar_spec *layers,
                                         size_t n_layers, uint32_t flags, mkhost_layer_result *outs,
                                         mkhost_layer_cache_stats *stats, mkhost_gz_index_stats *gz_stats, char *err,
                                         size_t errlen)
{
    return update_from_tars_impl(m, eng, now_unix, layers, n_layers, flags, MKSNAP_R_DEFER, outs, gz ? &gz->map : nullptr,
                                 keys, gz_stats, lc ? &lc->memo : nullptr, stats, "update memfs from tars: ", err, errlen);
}

int mkhost_memfs_update_from_tars_multi(mkhost_memfs *m, mksnap_t *const *engines, size_t n_engines, mkhost_layer_cache *lc,
                                        mkhost_gz_index_cache *gz, const char *const *keys, int64_t now_unix,
                                        const mkhost_tar_spec *layers, size_t n_layers, uint32_t flags,
                                        mkhost_layer_result *outs, mkhost_layer_cache_stats *stats,
                                        mkhost_gz_index_stats *gz_stats, char *err, size_t errlen)
{
    return update_from_tars_sharded(m, engines, n_engines, now_unix, layers, n_layers, flags, outs, gz ? &gz->map : nullptr,
                                    keys, gz_stats, lc ? &lc->memo : nullptr, stats, err, errlen);
}

mkhost_layer_cache *mkhost_layer_cache_new(void) { return new mkhost_layer_cache; }
void mkhost_layer_cache_free(mkhost_layer_cache *c) { delete c; }
uint64_t mkhost_layer_cache_size(const mkhost_layer_cache *c) { return c ? c->memo.e.size() : 0; }

int mkhost_layer_cache_save(const mkhost_layer_cache *c, const char *path, char *err, size_t errlen)
{
    return save_cache(c, path, err, errlen);
}

int mkhost_layer_cache_load(mkhost_layer_cache *c, const char *path, char *err, size_t errlen)
{
    return load_cache(c, path, err, errlen);
}

mkhost_gz_index_cache *mkhost_gz_index_cache_new(void) { return new mkhost_gz_index_cache; }
void mkhost_gz_index_cache_free(mkhost_gz_index_cache *c) { delete c; }
uint64_t mkhost_gz_index_cache_size(const mkhost_gz_index_cache *c) { return c ? c->map.e.size() : 0; }

int mkhost_gz_index_cache_save(const mkhost_gz_index_cache *c, const char *path, char *err, size_t errlen)
{
    return save_cache(c, path, err, errlen);
}

int mkhost_gz_index_cache_load(mkhost_gz_index_cache *c, const char *path, char *err, size_t errlen)
{
    return load_cache(c, path, err, errlen);
}

// ---- cache.Manager wire format (lib/cache/cache_manager.go:34-35,239-252) ----
size_t mkhost_cache_key(const char *cache_id, int chunk_table, char *out, size_t cap)
{
    return emit_text(std::string("makisu_builder_cache_") + (cache_id ? cache_id : "") + (chunk_table ? "_chunks" : ""), out, cap);
}

size_t mkhost_cache_entry_create(const char *tar_hex, const char *gzip_hex, char *out, size_t cap)
{
    if (!tar_hex) // createEntry(nil)
        return emit_text("MAKISU_CACHE_EMPTY", out, cap);
    return emit_text(std::string(tar_hex) + "," + (gzip_hex ? gzip_hex : ""), out, cap);
}

int mkhost_cache_entry_parse(const char *entry, char *tar_digest, size_t tar_cap, char *gzip_digest, size_t gzip_cap,
                             char *err, size_t errlen)
{
    const std::string e = entry ? entry : "";
    const size_t c = e.find(',');
    if (c == std::string::npos) {
        set_err(err, errlen, "parse redis entry: " + e);
        return -1;
    }
    const std::string t = "sha256:" + e.substr(0, c), g = "sha256:" + e.substr(c + 1); // SplitN(entry, ",", 2)
    if (t.size() + 1 > tar_cap || g.size() + 1 > gzip_cap) {
        set_err(err, errlen, "parse redis entry: output buffer too small");
        return -1;
    }
    memcpy(tar_digest, t.c_str(), t.size() + 1);
    memcpy(gzip_digest, g.c_str(), g.size() + 1);
    return 0;
}

size_t mkhost_cache_chunk_entry_create(const uint8_t root[32], uint64_t n_unique, char *out, size_t cap)
{
    static const char *hx = "0123456789abcdef";
    std::string s;
    for (int i = 0; i < 32; ++i) {
        s += hx[root[i] >> 4];
        s += hx[root[i] & 15];
    }
    return emit_text(s + "," + std::to_string(n_unique), out, cap);
}

int mkhost_cache_chunk_entry_parse(const char *entry, uint8_t root[32], uint64_t *n_unique, char *err, size_t errlen)
{
    const std::string e = entry ? entry : "";
    auto nib = [](char c) { return c >= '0' && c <= '9' ? c - '0' : (c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1); };
    bool ok = e.size() > 65 && e[64] == ',';
    for (int i = 0; ok && i < 64; ++i)
        ok = nib(e[i]) >= 0;
    uint64_t n = 0;
    for (size_t i = 65; ok && i < e.size(); ++i) {
        ok = e[i] >= '0' && e[i] <= '9' && n <= (UINT64_MAX - 9) / 10;
        n = n * 10 + (uint64_t)(e[i] - '0');
    }
    if (!ok) {
        set_err(err, errlen, "parse chunk table entry: " + e);
        return -1;
    }
    for (int i = 0; i < 32; ++i)
        root[i] = (uint8_t)(nib(e[2 * i]) * 16 + nib(e[2 * i + 1]));
    *n_unique = n;
    return 0;
}

} // extern "C"

namespace {

double ms_since(std::chrono::steady_clock::time_point t)
{
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
}

using FileKey = std::tuple<std::string, uint64_t, uint64_t, uint64_t, int64_t, int64_t>; // path, dev, ino, size, mtime, ctime
FileKey file_key(const Seg &g) { return FileKey{g.path, g.id.dev, g.id.ino, g.size, g.id.mtime_ns, g.id.ctime_ns}; }

// One engine session of a cacheID pass as CRC extents, numbered as mksnap_get_extent_crcs returns them: path strings at
// 16-byte alignment, file contents at 512-byte alignment with 4 KiB of room.  CRC is linear, so a file is split across
// arenas at any 16-byte boundary; remember() joins its pieces again after finish.
struct CrcPacker {
    struct Sent { // a file that travelled: its extents [first, first + n)
        const Seg *seg;
        uint64_t first, n;
    };
    ArenaSession s;
    std::vector<uint64_t> len; // length of every CRC extent so far, by extent index
    std::vector<Sent> sent;
    double ms_reads = 0, ms_acquire = 0, ms_submit = 0; // reading files, waiting for an arena, submitting it
    std::chrono::steady_clock::time_point t;

    // begins the session and leases its first arena
    CrcPacker(mksnap_t *eng, int n_threads, ReadPool &pool = ReadPool::get()) : s(eng, n_threads, 1) // cap unrounded: CRC pieces end anywhere
    {
        s.pool = &pool;
        s.after_reads = [this]() {
            ms_reads += ms_since(t);
            t = std::chrono::steady_clock::now();
        };
        ck(eng, mksnap_begin(eng), "begin");
        acquire();
    }
    void acquire()
    {
        t = std::chrono::steady_clock::now();
        s.acquire();
        ms_acquire += ms_since(t);
    }
    void submit()
    {
        t = std::chrono::steady_clock::now();
        s.submit();
        ms_submit += ms_since(t);
    }
    void finish(mksnap_result &res) { ck(s.eng, mksnap_finish(s.eng, &res), "finish"); }
    // offset of `need` bytes at `align` in the current arena, or in a fresh one when the arena or its extent table is full
    uint64_t place(uint64_t align, uint64_t need)
    {
        const uint64_t o = align_up(s.pos, align);
        if (o + need <= s.cap && s.room(1, 0))
            return o;
        submit();
        acquire();
        return 0;
    }
    uint64_t put(uint64_t o, uint64_t n, uint64_t suffix)
    {
        s.ext.push_back(mksnap_extent{o, n, suffix, MKSNAP_X_CRC, 0});
        s.pos = o + n;
        len.push_back(n);
        return len.size() - 1;
    }
    // a path string, link target or prefix of n > 0 bytes; returns its extent
    uint64_t text(const void *p, uint64_t n, uint64_t suffix)
    {
        if (n > s.cap)
            throw HostError("path string larger than the arena");
        const uint64_t o = place(16, n);
        memcpy(s.a + o, p, n);
        return put(o, n, suffix);
    }
    // the content of g, read into the arenas; with `after` (stream bytes behind the file) each piece's crc_suffix is the
    // stream bytes behind that piece, without it 0 (only pure(piece) is wanted)
    Sent file(const Seg &g, std::optional<uint64_t> after)
    {
        Sent f{&g, len.size(), 0};
        for (uint64_t done = 0; done < g.size; ++f.n) {
            const uint64_t o = place(512, 4096);
            const uint64_t n = std::min<uint64_t>(g.size - done, (s.cap - o) / 16 * 16);
            s.jobs.push_back(ReadJob{g.path, done, n, s.a + o});
            done += n;
            put(o, n, after ? *after + g.size - done : 0);
        }
        sent.push_back(f);
        return f;
    }
    // after finish: pure(content) of every file that travelled into `cache` and / or `known`
    void remember(mkhost_crc_cache *cache, std::map<FileKey, uint32_t> *known)
    {
        if (sent.empty() || !(cache || known))
            return;
        std::vector<uint32_t> pure(std::max<size_t>(1, len.size()));
        uint64_t n_got = 0;
        ck(s.eng, mksnap_get_extent_crcs(s.eng, pure.data(), pure.size(), &n_got), "extent crcs");
        if (n_got != len.size())
            throw HostError("internal: extent count mismatch");
        for (const Sent &f : sent) { // pure(A||B) = pure(A) x^(8|B|) ^ pure(B)
            uint32_t v = 0;          // pure of the empty string
            for (uint64_t k = f.first; k < f.first + f.n; ++k)
                v = mksnap_crc_concat(v, pure[k], len[k]);
            if (cache)
                cache->files[f.seg->path] = mkhost_crc_cache::Entry{f.seg->id, v};
            if (known)
                (*known)[file_key(*f.seg)] = v;
        }
    }
};

} // namespace

extern "C" {

// The cacheID over n_engines engines (one engine: the whole stream in one session).  The context is walked once; every
// segment's crc_suffix is its place in the whole stream, so each engine's crc_pure is its segments' share of the value
// and the shares XOR.  Files that travel go to the engines by LPT over their bytes (largest first, each to the least
// loaded engine); a path string or link target goes with the next file in walk order that travels, or to engine 0, as
// do the prefix and every file the cache vouches for (mksnap_crc_add, no bytes).  Each engine packs on a thread of its
// own with a reader pool of its own; the cache is read before they start and written after they have finished.
static int context_crc32_impl(mksnap_t *const *engines, size_t n_engines, mkhost_crc_cache *cache, mkhost_crc_cache_stats *stats,
                              const void *prefix, size_t prefix_len, const char *context_dir, const char *const *from_paths,
                              size_t n_paths, int n_threads, uint32_t *crc_out, uint64_t *stream_len_out, char *err, size_t errlen)
{
    try {
        if (!engines || n_engines == 0 || !crc_out)
            throw HostError("null argument");
        for (size_t k = 0; k < n_engines; ++k)
            if (!engines[k])
                throw HostError("null argument");
        const auto t_start = std::chrono::steady_clock::now();
        std::vector<Seg> segs = context_segments(go_clean(context_dir), from_paths, n_paths, n_threads);
        const double ms_walk = ms_since(t_start);
        uint64_t total = prefix_len;
        for (const auto &g : segs)
            total += g.kind == 'F' ? g.size : g.bytes.size();
        std::vector<uint64_t> after(segs.size()); // stream bytes behind each segment
        std::vector<const mkhost_crc_cache::Entry *> hit(segs.size(), nullptr);
        mkhost_crc_cache_stats st{};
        std::vector<std::pair<uint64_t, size_t>> sent; // (bytes, segment) of every file that travels
        uint64_t a = total - prefix_len;
        for (size_t i = 0; i < segs.size(); ++i) {
            const Seg &g = segs[i];
            a -= g.kind == 'F' ? g.size : g.bytes.size();
            after[i] = a;
            if (g.kind != 'F')
                continue;
            ++st.files_total;
            st.bytes_total += g.size;
            if (cache) { // unchanged since a build that remembered it: fold pure(content) in, send nothing
                auto it = cache->files.find(g.path);
                if (it != cache->files.end() && it->second.id == g.id) {
                    hit[i] = &it->second;
                    ++st.files_reused;
                    continue;
                }
            }
            st.bytes_sent += g.size;
            sent.emplace_back(g.size, i);
        }
        std::vector<size_t> owner(segs.size(), 0);
        if (n_engines > 1) {
            std::stable_sort(sent.begin(), sent.end(), [](const auto &x, const auto &y) { return x.first > y.first; });
            std::vector<uint64_t> load(n_engines, 0);
            for (const auto &f : sent) {
                const size_t k = (size_t)(std::min_element(load.begin(), load.end()) - load.begin());
                load[k] += f.first;
                owner[f.second] = k;
            }
            size_t next = 0; // engine of the next file in walk order that travels
            for (size_t i = segs.size(); i-- > 0;) {
                if (segs[i].kind == 'F' && !hit[i])
                    next = owner[i];
                else
                    owner[i] = segs[i].kind == 'F' ? 0 : next;
            }
        }
        std::vector<std::vector<size_t>> mine(n_engines);
        for (size_t i = 0; i < segs.size(); ++i)
            mine[owner[i]].push_back(i);
        std::vector<size_t> active{0}; // engine 0 and every engine with segments
        for (size_t k = 1; k < n_engines; ++k)
            if (!mine[k].empty())
                active.push_back(k);
        EngineThreads threads(active.size());
        std::vector<std::unique_ptr<CrcPacker>> pks(active.size());
        std::vector<mksnap_result> res(active.size());
        threads.run([&](size_t j) {
            mksnap_t *eng = engines[active[j]];
            pks[j].reset(new CrcPacker(eng, n_threads, threads.pool(j)));
            CrcPacker &pk = *pks[j];
            if (j == 0 && prefix_len)
                pk.text(prefix, prefix_len, total - prefix_len);
            for (size_t i : mine[active[j]]) {
                const Seg &g = segs[i];
                if (g.kind != 'F') {
                    if (!g.bytes.empty())
                        pk.text(g.bytes.data(), g.bytes.size(), after[i]);
                } else if (hit[i]) {
                    ck(eng, mksnap_crc_add(eng, hit[i]->pure, g.size, after[i]), "crc add");
                } else {
                    pk.file(g, after[i]);
                }
            }
            pk.submit();
            pk.finish(res[j]);
        });
        mksnap_result all{};
        for (const mksnap_result &r : res) {
            all.crc_pure ^= r.crc_pure;
            all.crc_bytes += r.crc_bytes;
        }
        if (getenv("MKHOST_TRACE")) { // phase times on stderr, summed over the engines
            double ms_reads = 0, ms_acquire = 0, ms_submit = 0;
            for (const auto &pk : pks)
                ms_reads += pk->ms_reads, ms_acquire += pk->ms_acquire, ms_submit += pk->ms_submit;
            fprintf(stderr, "[mkhost] context crc32: %zu segments, %.1f MiB, %zu engines; walk %.2f ms, reads %.2f, acquire waits %.2f, "
                            "submit %.2f, total %.2f ms\n",
                    segs.size(), (double)total / 1048576.0, active.size(), ms_walk, ms_reads, ms_acquire, ms_submit,
                    ms_since(t_start));
        }
        if (all.crc_bytes != total)
            throw HostError("internal: stream length mismatch");
        *crc_out = mksnap_ctx_crc32(&all);
        if (stream_len_out)
            *stream_len_out = total;
        for (const auto &pk : pks)
            pk->remember(cache, nullptr);
        if (stats)
            *stats = st;
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("hash context sources: ") + e.what());
        return -1;
    }
}

int mkhost_context_crc32(mksnap_t *eng, const void *prefix, size_t prefix_len, const char *context_dir,
                         const char *const *from_paths, size_t n_paths, int n_threads, uint32_t *crc_out,
                         uint64_t *stream_len_out, char *err, size_t errlen)
{
    return context_crc32_impl(&eng, 1, nullptr, nullptr, prefix, prefix_len, context_dir, from_paths, n_paths, n_threads, crc_out,
                              stream_len_out, err, errlen);
}

mkhost_crc_cache *mkhost_crc_cache_new(void) { return new mkhost_crc_cache; }
void mkhost_crc_cache_free(mkhost_crc_cache *c) { delete c; }
uint64_t mkhost_crc_cache_size(const mkhost_crc_cache *c) { return c ? c->files.size() : 0; }

int mkhost_crc_cache_save(const mkhost_crc_cache *c, const char *path, char *err, size_t errlen)
{
    return save_cache(c, path, err, errlen);
}

int mkhost_crc_cache_load(mkhost_crc_cache *c, const char *path, char *err, size_t errlen)
{
    return load_cache(c, path, err, errlen);
}

mkhost_chunk_cache *mkhost_chunk_cache_new(void) { return new mkhost_chunk_cache; }
void mkhost_chunk_cache_free(mkhost_chunk_cache *c) { delete c; }
uint64_t mkhost_chunk_cache_size(const mkhost_chunk_cache *c) { return c ? c->memo.files.size() : 0; }

int mkhost_chunk_cache_save(const mkhost_chunk_cache *c, const char *path, char *err, size_t errlen)
{
    return save_cache(c, path, err, errlen);
}

int mkhost_chunk_cache_load(mkhost_chunk_cache *c, const char *path, char *err, size_t errlen)
{
    return load_cache(c, path, err, errlen);
}

int mkhost_context_crc32_cached(mksnap_t *eng, mkhost_crc_cache *cache, const void *prefix, size_t prefix_len,
                                const char *context_dir, const char *const *from_paths, size_t n_paths, int n_threads,
                                uint32_t *crc_out, uint64_t *stream_len_out, mkhost_crc_cache_stats *stats, char *err, size_t errlen)
{
    if (!cache) {
        set_err(err, errlen, "hash context sources: no cache object");
        return -1;
    }
    return context_crc32_impl(&eng, 1, cache, stats, prefix, prefix_len, context_dir, from_paths, n_paths, n_threads, crc_out,
                              stream_len_out, err, errlen);
}

int mkhost_context_crc32_multi(mksnap_t *const *engines, size_t n_engines, mkhost_crc_cache *cache, const void *prefix,
                               size_t prefix_len, const char *context_dir, const char *const *from_paths, size_t n_paths,
                               int n_threads, uint32_t *crc_out, uint64_t *stream_len_out, mkhost_crc_cache_stats *stats,
                               char *err, size_t errlen)
{
    return context_crc32_impl(engines, n_engines, cache, stats, prefix, prefix_len, context_dir, from_paths, n_paths, n_threads,
                              crc_out, stream_len_out, err, errlen);
}

// One engine session of mkhost_plan_cache_ids: the streams of the walked COPY/ADD steps `batch` (stream slot k = batch[k]).
// Every distinct path string / link target and every file not yet valued travels once as CRC extents (crc_suffix 0:
// only pure(extent) is wanted); each occurrence in a stream becomes a use of those extents, or of a known value.
static void plan_session(mksnap_t *eng, mkhost_crc_cache *cache, const std::vector<std::vector<Seg>> &segs,
                         const std::vector<size_t> &batch, int n_threads, std::map<FileKey, uint32_t> &known,
                         bool remember, std::vector<uint32_t> &pure, std::vector<uint64_t> &slen,
                         mkhost_crc_cache_stats &st, double &ms_fold)
{
    CrcPacker pk(eng, n_threads);
    std::map<std::string, uint64_t> text_ext;   // path string / link target -> its extent
    std::map<FileKey, CrcPacker::Sent> sent_of; // file -> its extents
    std::vector<mksnap_crc_use> uses;           // grouped by stream, as k_crc_fold prefers them
    for (size_t k = 0; k < batch.size(); ++k) {
        const uint32_t slot = (uint32_t)k;
        const std::vector<Seg> &ss = segs[batch[k]];
        uint64_t after = 0; // stream bytes after the segment
        for (const auto &g : ss)
            after += g.kind == 'F' ? g.size : g.bytes.size();
        slen[batch[k]] = after;
        for (const auto &g : ss) {
            if (g.kind != 'F') {
                after -= g.bytes.size();
                if (g.bytes.empty())
                    continue;
                auto it = text_ext.find(g.bytes);
                if (it == text_ext.end())
                    it = text_ext.emplace(g.bytes, pk.text(g.bytes.data(), g.bytes.size(), 0)).first;
                uses.push_back(mksnap_crc_use{after, it->second, slot, 0});
                continue;
            }
            ++st.files_total;
            st.bytes_total += g.size;
            after -= g.size;
            if (g.size == 0)
                continue;
            if (cache) { // unchanged since a build that remembered it: no read
                auto it = cache->files.find(g.path);
                if (it != cache->files.end() && it->second.id == g.id) {
                    ++st.files_reused;
                    uses.push_back(mksnap_crc_use{after, it->second.pure, slot, MKSNAP_U_VALUE});
                    continue;
                }
            }
            const FileKey key = file_key(g);
            auto kn = known.find(key); // valued by an earlier session of this plan
            if (kn != known.end()) {
                uses.push_back(mksnap_crc_use{after, kn->second, slot, MKSNAP_U_VALUE});
                continue;
            }
            auto so = sent_of.find(key);
            if (so == sent_of.end()) {
                so = sent_of.emplace(key, pk.file(g, std::nullopt)).first;
                st.bytes_sent += g.size;
            }
            const CrcPacker::Sent &f = so->second;
            uint64_t a = after + g.size;
            for (uint64_t x = f.first; x < f.first + f.n; ++x) {
                a -= pk.len[x];
                uses.push_back(mksnap_crc_use{a, x, slot, 0});
            }
        }
    }
    pk.submit();
    const auto t_fold = std::chrono::steady_clock::now();
    for (size_t u0 = 0; u0 < uses.size(); u0 += pk.s.lim.max_extents)
        ck(eng, mksnap_crc_fold(eng, uses.data() + u0, std::min<uint64_t>(pk.s.lim.max_extents, uses.size() - u0)), "crc fold");
    mksnap_result res;
    pk.finish(res);
    ms_fold += ms_since(t_fold);
    std::vector<uint32_t> val(batch.size());
    uint64_t n_val = 0;
    ck(eng, mksnap_get_crc_streams(eng, val.data(), val.size(), &n_val), "crc streams");
    for (size_t k = 0; k < batch.size(); ++k)
        pure[batch[k]] = k < n_val ? val[k] : 0u; // a stream nothing was folded into is empty
    pk.remember(cache, remember ? &known : nullptr);
}

int mkhost_plan_cache_ids(mksnap_t *eng, mkhost_crc_cache *cache, const char *seed, const char *context_dir,
                          const mkhost_plan_step *steps, size_t n_steps, int n_threads, uint32_t *ids_out,
                          mkhost_crc_cache_stats *stats, char *err, size_t errlen)
{
    try {
        if (!eng || !seed || !context_dir || (n_steps && (!steps || !ids_out)))
            throw HostError("null argument");
        const auto t_start = std::chrono::steady_clock::now();
        const std::string ctx = go_clean(context_dir);
        std::vector<std::vector<Seg>> segs(n_steps);
        std::vector<size_t> walked; // steps that hash context content, in plan order
        for (size_t i = 0; i < n_steps; ++i) {
            const mkhost_plan_step &p = steps[i];
            if (p.kind < MKHOST_STEP_COPY || p.kind > MKHOST_STEP_REMOTE_FROM)
                throw HostError("step " + std::to_string(i) + ": unknown kind " + std::to_string(p.kind));
            if (p.kind == MKHOST_STEP_COPY && !(p.from_stage && *p.from_stage)) {
                if (p.n_paths && !p.from_paths)
                    throw HostError("step " + std::to_string(i) + ": null from_paths");
                segs[i] = context_segments(ctx, p.from_paths, p.n_paths, n_threads);
                walked.push_back(i);
            }
        }
        const double ms_walk = ms_since(t_start);
        std::vector<uint32_t> pure(n_steps, 0);
        std::vector<uint64_t> slen(n_steps, 0);
        mkhost_crc_cache_stats st{};
        std::map<FileKey, uint32_t> known;
        double ms_fold = 0;
        const uint64_t slots = engine_limits(eng).max_streams;
        size_t n_sessions = 0;
        for (size_t b0 = 0; b0 < walked.size(); b0 += slots, ++n_sessions) {
            const size_t b1 = (size_t)std::min<uint64_t>(walked.size(), b0 + slots);
            const std::vector<size_t> batch(walked.begin() + b0, walked.begin() + b1);
            plan_session(eng, cache, segs, batch, n_threads, known, b1 < walked.size(), pure, slen, st, ms_fold);
        }
        // the seed chain, in plan order (createDockerfileSteps: seed = step.CacheID())
        std::string sd = seed, stage_seed;
        bool in_remote = false;
        for (size_t i = 0; i < n_steps; ++i) {
            const mkhost_plan_step &p = steps[i];
            const std::string dir = p.directive ? p.directive : "", args = p.args ? p.args : "";
            const bool remote = p.kind == MKHOST_STEP_REMOTE_FROM;
            if (remote && !in_remote)
                stage_seed = sd;
            else if (!remote && in_remote)
                sd = stage_seed;
            in_remote = remote;
            std::string prefix;
            if (p.kind == MKHOST_STEP_FROM || remote)
                prefix = sd + "FROM" + args;
            else if (p.kind == MKHOST_STEP_BASE)
                prefix = sd + dir + args + (p.commit ? "true" : "false");
            else
                prefix = sd + dir + args;
            ids_out[i] = mksnap_crc_prepend(prefix.data(), prefix.size(), pure[i], slen[i]);
            char hex[16];
            snprintf(hex, sizeof hex, "%x", ids_out[i]);
            sd = hex;
        }
        if (getenv("MKHOST_TRACE"))
            fprintf(stderr, "[mkhost] plan cacheIDs: %zu steps, %zu walked, %zu sessions; walk %.2f ms, fold + finish %.2f ms, total %.2f ms\n",
                    n_steps, walked.size(), n_sessions, ms_walk, ms_fold, ms_since(t_start));
        if (stats)
            *stats = st;
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("hash context sources: ") + e.what());
        return -1;
    }
}

int mkhost_commit_copy_ops(mksnap_t *eng, const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops, size_t n_ops,
                           int n_threads, mkhost_layer_result *out, char *err, size_t errlen)
{
    return mkhost_commit_copy_ops_to_fd(eng, root_dir, now_unix, ops, n_ops, n_threads, -1, out, err, errlen);
}

int mkhost_commit_copy_ops_to_fd(mksnap_t *eng, const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops,
                                 size_t n_ops, int n_threads, int tar_fd, mkhost_layer_result *out, char *err,
                                 size_t errlen)
{
    return mkhost_commit_copy_ops_ex(eng, root_dir, now_unix, ops, n_ops, n_threads, tar_fd, 0, out, err, errlen);
}

int mkhost_commit_copy_ops_ex(mksnap_t *eng, const char *root_dir, int64_t now_unix, const mkhost_copy_op *ops,
                              size_t n_ops, int n_threads, int tar_fd, uint32_t flags, mkhost_layer_result *out,
                              char *err, size_t errlen)
{
    try {
        MemFS fs(root_dir, now_unix);
        commit_layer(eng, fs.add_layer_by_copy_ops(ops, n_ops), n_threads, tar_fd, flags, out);
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("failed to generate diff layer: ") + e.what());
        return -1;
    }
}

} // extern "C"
