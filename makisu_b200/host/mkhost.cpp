// mkhost.cpp — host side above the mksnap C-ABI (see include/mkhost.h).
//
// C++ stand-in for the Go code a cgo build of makisu would keep on this path: the filepath.Walk-ordered
// context stream (cacheID), the MemFS copy-op layer (entry order + tar headers) and the arena packer.
// It does no hashing; digests come from libmksnap (GPU).  Reference line numbers are cited per function.
//
// One translation unit: the *.inc files in this directory are fragments of the anonymous namespace below, included in
// dependency order (Go path helpers, Walk/Glob, context stream, file reader pool, tar writer, tar reader, Copier,
// MemFS, arena packers); this file holds the C entry points.
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
#include <functional>
#include <map>
#include <memory>
#include <mutex>
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

} // namespace

// pure(file content) per context file, remembered between builds (incremental cacheID, include/mkhost.h)
struct mkhost_crc_cache {
    struct Entry {
        FileId id;
        uint32_t pure;
    };
    std::map<std::string, Entry> files; // key: absolute path
};

// block indexes of gzip blobs per caller key, remembered between builds (include/mkhost.h)
struct mkhost_gz_index_cache {
    GzIndexMap map;
};

// chunk digests per source file, remembered between builds (incremental layer commit, include/mkhost.h)
struct mkhost_chunk_cache {
    ChunkMemo memo;
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
    try {
        if (!m || !eng || (!specs && n_layers) || (!outs && n_layers))
            throw HostError("null argument");
        if (flags & ~(uint32_t)MKHOST_NO_TAR_DIGEST)
            throw HostError("commit layers: only MKHOST_NO_TAR_DIGEST is supported for a batch");
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
        commit_layers_batch(eng, bl, n_threads, flags, outs);
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

// mkhost_memfs_update_from_tar; with `ix`, mkhost_memfs_update_from_tar_indexed
int update_from_tar_impl(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, int tar_fd, uint32_t flags,
                         mkhost_layer_result *out, const GzIndexUse *ix, char *err, size_t errlen)
{
    try {
        m->fs.set_now(now_unix);
        const bool want_digest = !(flags & MKHOST_NO_TAR_DIGEST);
        ck(eng, mksnap_begin(eng), "begin");
        IngestedLayer in;
        ingest_layer(m->fs, eng, tar_fd, flags, 0, 0, 1, in, ix);
        mksnap_result res;
        ck(eng, mksnap_finish(eng, &res), "finish");
        std::vector<uint8_t> d((in.n_file_streams + 1) * 32, 0);
        if (want_digest || in.n_file_streams)
            ck(eng, mksnap_get_stream_digests(eng, d.data(), in.n_file_streams + 1), "stream digests");
        const std::map<std::string, MemFile> layer = merge_layer(m->fs, flags, in, d.data(), 1);
        set_layer_result(out, res, want_digest ? d.data() : nullptr, layer.size(), in.tar_bytes);
        return 0;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("update memfs from tar: ") + e.what());
        return -1;
    }
}

// mkhost_memfs_update_from_tars; with `cache`, mkhost_memfs_update_from_tars_indexed (keys[i] for layer i)
int update_from_tars_impl(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_tar_spec *layers,
                          size_t n_layers, uint32_t flags, mkhost_layer_result *outs, GzIndexMap *cache,
                          const char *const *keys, mkhost_gz_index_stats *stats, char *err, size_t errlen)
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
        // layer i's DiffID is stream slot i, deferred: the engine keeps its bytes in the stream log and hashes the
        // chains of the whole run together.  Per-file streams are inline, in the slots after the layers.
        const uint32_t file_base = (uint32_t)n_layers;
        ck(eng, mksnap_begin(eng), "begin");
        if (want_digest)
            ck(eng, mksnap_reserve_stream_log(eng, RUN_STREAM_LOG_BYTES), "reserve stream log");
        std::vector<uint64_t> entries(n_layers), tar_bytes(n_layers);
        std::vector<uint8_t> d;    // stream-digest rows [0, file_base + most file streams of a layer so far)
        uint32_t max_files = 0;
        for (size_t i = 0; i < n_layers; ++i) {
            // the layers join the tree (and the disk) strictly in order: whiteouts, overwrites and hard links of
            // layer i + 1 act on what layer i left
            IngestedLayer in;
            const GzIndexUse ix{cache, keys ? keys[i] : nullptr, stats};
            ingest_layer(m->fs, eng, layers[i].tar_fd, flags | layers[i].flags, (uint32_t)i, MKSNAP_R_DEFER, file_base, in,
                         cache && ix.key ? &ix : nullptr);
            if (in.n_file_streams) { // inline streams: their rows are final once the submits so far have run
                max_files = std::max(max_files, in.n_file_streams);
                d.assign(((uint64_t)file_base + max_files) * 32, 0);
                ck(eng, mksnap_get_stream_digests(eng, d.data(), file_base + max_files), "stream digests");
            }
            const std::map<std::string, MemFile> layer = merge_layer(m->fs, flags, in, d.data(), file_base);
            entries[i] = layer.size();
            tar_bytes[i] = in.tar_bytes;
        }
        mksnap_result res;
        ck(eng, mksnap_finish(eng, &res), "finish");
        std::vector<uint8_t> rows(std::max<uint64_t>(res.n_streams, n_layers) * 32, 0);
        if (want_digest)
            ck(eng, mksnap_get_stream_digests(eng, rows.data(), rows.size() / 32), "stream digests");
        for (size_t i = 0; i < n_layers; ++i) // root: chunk table of the whole run (one session)
            set_layer_result(&outs[i], res, want_digest ? rows.data() + 32 * i : nullptr, entries[i], tar_bytes[i]);
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
    return update_from_tar_impl(m, eng, now_unix, tar_fd, flags, out, nullptr, err, errlen);
}

int mkhost_memfs_update_from_tars(mkhost_memfs *m, mksnap_t *eng, int64_t now_unix, const mkhost_tar_spec *layers,
                                  size_t n_layers, uint32_t flags, mkhost_layer_result *outs, char *err, size_t errlen)
{
    return update_from_tars_impl(m, eng, now_unix, layers, n_layers, flags, outs, nullptr, nullptr, nullptr, err, errlen);
}

int mkhost_memfs_update_from_tar_indexed(mkhost_memfs *m, mksnap_t *eng, mkhost_gz_index_cache *cache, const char *key,
                                         int64_t now_unix, int tar_fd, uint32_t flags, mkhost_layer_result *out,
                                         mkhost_gz_index_stats *stats, char *err, size_t errlen)
{
    const GzIndexUse ix{cache ? &cache->map : nullptr, key, stats};
    return update_from_tar_impl(m, eng, now_unix, tar_fd, flags, out, cache && key ? &ix : nullptr, err, errlen);
}

int mkhost_memfs_update_from_tars_indexed(mkhost_memfs *m, mksnap_t *eng, mkhost_gz_index_cache *cache,
                                          const char *const *keys, int64_t now_unix, const mkhost_tar_spec *layers,
                                          size_t n_layers, uint32_t flags, mkhost_layer_result *outs,
                                          mkhost_gz_index_stats *stats, char *err, size_t errlen)
{
    return update_from_tars_impl(m, eng, now_unix, layers, n_layers, flags, outs, cache ? &cache->map : nullptr,
                                 keys, stats, err, errlen);
}

mkhost_gz_index_cache *mkhost_gz_index_cache_new(void) { return new mkhost_gz_index_cache; }
void mkhost_gz_index_cache_free(mkhost_gz_index_cache *c) { delete c; }
uint64_t mkhost_gz_index_cache_size(const mkhost_gz_index_cache *c) { return c ? c->map.e.size() : 0; }

// "mkhost-gz-index-cache 1", then per blob a line "<gz_len> <n_points> <key>" followed by its points, 8 bytes each
// (little endian)
int mkhost_gz_index_cache_save(const mkhost_gz_index_cache *c, const char *path, char *err, size_t errlen)
{
    FILE *f = c && path ? fopen(path, "wb") : nullptr;
    if (!f) {
        set_err(err, errlen, std::string("save gzip index cache: ") + strerror(errno));
        return -1;
    }
    fprintf(f, "mkhost-gz-index-cache 1\n");
    for (const auto &kv : c->map.e) { // keys with newlines are not cached
        if (kv.first.find('\n') != std::string::npos)
            continue;
        fprintf(f, "%llu %zu %s\n", (unsigned long long)kv.second.gz_len, kv.second.points.size(), kv.first.c_str());
        fwrite(kv.second.points.data(), 8, kv.second.points.size(), f);
    }
    const bool ok = !ferror(f) && fclose(f) == 0;
    if (!ok)
        set_err(err, errlen, std::string("save gzip index cache: ") + strerror(errno));
    return ok ? 0 : -1;
}

int mkhost_gz_index_cache_load(mkhost_gz_index_cache *c, const char *path, char *err, size_t errlen)
{
    FILE *f = c && path ? fopen(path, "rb") : nullptr;
    if (!f) {
        set_err(err, errlen, std::string("load gzip index cache: ") + strerror(errno));
        return -1;
    }
    struct stat fst;
    const uint64_t fsize = fstat(fileno(f), &fst) == 0 ? (uint64_t)fst.st_size : 0;
    char *line = nullptr;
    size_t cap = 0;
    ssize_t n = getline(&line, &cap, f);
    bool ok = n > 0 && strcmp(line, "mkhost-gz-index-cache 1\n") == 0;
    std::map<std::string, GzIndexMap::Entry> e;
    while (ok && (n = getline(&line, &cap, f)) > 0) {
        if (line[n - 1] == '\n')
            line[--n] = 0;
        unsigned long long len = 0, pts = 0;
        int used = 0;
        if (sscanf(line, "%llu %llu %n", &len, &pts, &used) != 2 || used <= 0 || used >= n || pts > fsize / 8) {
            ok = false; // the points must fit in what is left of the file
            break;
        }
        GzIndexMap::Entry x{len, std::vector<uint64_t>(pts)};
        ok = fread(x.points.data(), 8, pts, f) == pts;
        e[line + used] = std::move(x);
    }
    free(line);
    fclose(f);
    if (!ok) {
        set_err(err, errlen, "load gzip index cache: not a mkhost-gz-index-cache file");
        return -1;
    }
    c->map.e.swap(e);
    return 0;
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

static int context_crc32_impl(mksnap_t *eng, mkhost_crc_cache *cache, mkhost_crc_cache_stats *stats, const void *prefix,
                              size_t prefix_len, const char *context_dir, const char *const *from_paths, size_t n_paths,
                              int n_threads, uint32_t *crc_out, uint64_t *stream_len_out, char *err, size_t errlen)
{
    try {
        const bool trace = getenv("MKHOST_TRACE") != nullptr; // phase times on stderr
        const auto t_start = std::chrono::steady_clock::now();
        auto ms_since = [&](std::chrono::steady_clock::time_point t) {
            return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
        };
        double ms_reads = 0, ms_submit = 0, ms_acquire = 0;
        std::vector<Seg> segs = context_segments(go_clean(context_dir), from_paths, n_paths, n_threads);
        const double ms_walk = ms_since(t_start);
        uint64_t total = prefix_len;
        for (const auto &g : segs)
            total += g.kind == 'F' ? g.size : g.bytes.size();
        ArenaSession s(eng, n_threads, 1); // cap unrounded: CRC pieces end anywhere, files are cut at 16-byte granularity
        auto t = std::chrono::steady_clock::now();
        s.after_reads = [&]() {
            ms_reads += ms_since(t);
            t = std::chrono::steady_clock::now();
        };
        auto acquire = [&]() {
            t = std::chrono::steady_clock::now();
            s.acquire();
            ms_acquire += ms_since(t);
        };
        auto flush = [&]() {
            t = std::chrono::steady_clock::now();
            s.submit();
            ms_submit += ms_since(t);
        };
        ck(eng, mksnap_begin(eng), "begin");
        acquire();
        uint64_t after = total; // stream bytes not yet placed
        uint64_t n_crc_ext = 0; // CRC extents submitted so far in this session (index into mksnap_get_extent_crcs)
        struct Sent {           // a file that travelled: its extents [first, first + pieces) and their lengths
            const Seg *seg;
            uint64_t first;
            std::vector<uint64_t> piece_len;
        };
        std::vector<Sent> sent;
        mkhost_crc_cache_stats st{};
        auto put_bytes = [&](const void *p, size_t n) {
            if (n == 0)
                return;
            uint64_t o = align_up(s.pos, 16);
            if (o + n > s.cap || !s.room(1, 0)) {
                flush();
                acquire();
                o = 0;
            }
            if (n > s.cap)
                throw HostError("path string larger than the arena");
            memcpy(s.a + o, p, n);
            after -= n;
            s.ext.push_back(mksnap_extent{o, n, after, MKSNAP_X_CRC, 0});
            ++n_crc_ext;
            s.pos = o + n;
        };
        put_bytes(prefix, prefix_len);
        for (const auto &g : segs) {
            if (g.kind != 'F') {
                put_bytes(g.bytes.data(), g.bytes.size());
                continue;
            }
            ++st.files_total;
            st.bytes_total += g.size;
            if (cache) { // unchanged since a build that remembered it: fold pure(content) in, send nothing
                auto it = cache->files.find(g.path);
                if (it != cache->files.end() && it->second.id == g.id) {
                    after -= g.size;
                    ck(eng, mksnap_crc_add(eng, it->second.pure, g.size, after), "crc add");
                    ++st.files_reused;
                    continue;
                }
            }
            st.bytes_sent += g.size;
            if (cache)
                sent.push_back(Sent{&g, n_crc_ext, {}});
            uint64_t done = 0; // CRC is linear: a file may be split across arenas at any 16-byte boundary
            while (done < g.size) {
                uint64_t o = align_up(s.pos, 512);
                if (o + 4096 > s.cap || !s.room(1, 0)) {
                    flush();
                    acquire();
                    o = 0;
                }
                uint64_t n = std::min<uint64_t>(g.size - done, (s.cap - o) / 16 * 16);
                s.jobs.push_back(ReadJob{g.path, done, n, s.a + o});
                after -= n;
                s.ext.push_back(mksnap_extent{o, n, after, MKSNAP_X_CRC, 0});
                ++n_crc_ext;
                if (cache)
                    sent.back().piece_len.push_back(n);
                s.pos = o + n;
                done += n;
            }
        }
        flush();
        mksnap_result res;
        const auto t_fin = std::chrono::steady_clock::now();
        ck(eng, mksnap_finish(eng, &res), "finish");
        if (trace)
            fprintf(stderr, "[mkhost] context crc32: %zu segments, %.1f MiB; walk %.2f ms, reads %.2f, acquire waits %.2f, submit %.2f, "
                            "finish %.2f, total %.2f ms\n",
                    segs.size(), (double)total / 1048576.0, ms_walk, ms_reads, ms_acquire, ms_submit, ms_since(t_fin), ms_since(t_start));
        if (res.crc_bytes != total)
            throw HostError("internal: stream length mismatch");
        *crc_out = mksnap_ctx_crc32(&res);
        if (stream_len_out)
            *stream_len_out = total;
        if (cache) { // remember pure(content) of every file that travelled (pieces joined: pure(A||B) = pure(A) x^(8|B|) ^ pure(B))
            std::vector<uint32_t> pure(std::max<uint64_t>(1, n_crc_ext));
            uint64_t n_got = 0;
            ck(eng, mksnap_get_extent_crcs(eng, pure.data(), pure.size(), &n_got), "extent crcs");
            if (n_got != n_crc_ext)
                throw HostError("internal: extent count mismatch");
            for (const Sent &f : sent) {
                uint32_t v = 0; // pure of the empty string
                for (size_t k = 0; k < f.piece_len.size(); ++k)
                    v = mksnap_crc_concat(v, pure[f.first + k], f.piece_len[k]);
                cache->files[f.seg->path] = mkhost_crc_cache::Entry{f.seg->id, v};
            }
        }
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
    return context_crc32_impl(eng, nullptr, nullptr, prefix, prefix_len, context_dir, from_paths, n_paths, n_threads, crc_out,
                              stream_len_out, err, errlen);
}

mkhost_crc_cache *mkhost_crc_cache_new(void) { return new mkhost_crc_cache; }
void mkhost_crc_cache_free(mkhost_crc_cache *c) { delete c; }
uint64_t mkhost_crc_cache_size(const mkhost_crc_cache *c) { return c ? c->files.size() : 0; }

int mkhost_crc_cache_save(const mkhost_crc_cache *c, const char *path, char *err, size_t errlen)
{
    FILE *f = c && path ? fopen(path, "w") : nullptr;
    if (!f) {
        set_err(err, errlen, std::string("save crc cache: ") + strerror(errno));
        return -1;
    }
    fprintf(f, "mkhost-crc-cache 1\n");
    for (const auto &kv : c->files) // path last: it may hold spaces (newlines in file names are not cached)
        if (kv.first.find('\n') == std::string::npos)
            fprintf(f, "%s %08x %s\n", file_id_text(kv.second.id).c_str(), kv.second.pure, kv.first.c_str());
    const bool ok = fclose(f) == 0;
    if (!ok)
        set_err(err, errlen, std::string("save crc cache: ") + strerror(errno));
    return ok ? 0 : -1;
}

int mkhost_crc_cache_load(mkhost_crc_cache *c, const char *path, char *err, size_t errlen)
{
    FILE *f = c && path ? fopen(path, "r") : nullptr;
    if (!f) {
        set_err(err, errlen, std::string("load crc cache: ") + strerror(errno));
        return -1;
    }
    char *line = nullptr;
    size_t cap = 0;
    ssize_t n = getline(&line, &cap, f);
    bool ok = n > 0 && strncmp(line, "mkhost-crc-cache 1", 18) == 0;
    while (ok && (n = getline(&line, &cap, f)) > 0) {
        if (line[n - 1] == '\n')
            line[--n] = 0;
        FileId id;
        unsigned pure;
        int used = 0, used2 = 0;
        if (!parse_file_id(line, &id, &used) || sscanf(line + used, " %x %n", &pure, &used2) != 1 || used2 <= 0 ||
            used + used2 >= n) {
            ok = false;
            break;
        }
        c->files[line + used + used2] = mkhost_crc_cache::Entry{id, (uint32_t)pure};
    }
    free(line);
    fclose(f);
    if (!ok)
        set_err(err, errlen, "load crc cache: not a mkhost-crc-cache file");
    return ok ? 0 : -1;
}

mkhost_chunk_cache *mkhost_chunk_cache_new(void) { return new mkhost_chunk_cache; }
void mkhost_chunk_cache_free(mkhost_chunk_cache *c) { delete c; }
uint64_t mkhost_chunk_cache_size(const mkhost_chunk_cache *c) { return c ? c->memo.files.size() : 0; }

// "mkhost-chunk-cache 1 <min> <normal> <max> <strict bits> <loose bits>", then per file a line
// "<dev> <ino> <size> <mtime ns> <ctime ns> <chunks> <path>" followed by its digests, 32 raw bytes per chunk
int mkhost_chunk_cache_save(const mkhost_chunk_cache *c, const char *path, char *err, size_t errlen)
{
    FILE *f = c && path ? fopen(path, "wb") : nullptr;
    if (!f) {
        set_err(err, errlen, std::string("save chunk cache: ") + strerror(errno));
        return -1;
    }
    const mksnap_cdc_params &p = c->memo.cdc;
    fprintf(f, "mkhost-chunk-cache 1 %u %u %u %u %u\n", p.min_size, p.normal_size, p.max_size, p.strict_bits, p.loose_bits);
    for (const auto &kv : c->memo.files) { // newlines in file names are not cached
        if (kv.first.find('\n') != std::string::npos)
            continue;
        fprintf(f, "%s %zu %s\n", file_id_text(kv.second.id).c_str(), kv.second.digests.size() / 32, kv.first.c_str());
        fwrite(kv.second.digests.data(), 1, kv.second.digests.size(), f);
    }
    const bool ok = !ferror(f) && fclose(f) == 0;
    if (!ok)
        set_err(err, errlen, std::string("save chunk cache: ") + strerror(errno));
    return ok ? 0 : -1;
}

int mkhost_chunk_cache_load(mkhost_chunk_cache *c, const char *path, char *err, size_t errlen)
{
    FILE *f = c && path ? fopen(path, "rb") : nullptr;
    if (!f) {
        set_err(err, errlen, std::string("load chunk cache: ") + strerror(errno));
        return -1;
    }
    char *line = nullptr;
    size_t cap = 0;
    mksnap_cdc_params p{};
    ssize_t n = getline(&line, &cap, f);
    bool ok = n > 0 && sscanf(line, "mkhost-chunk-cache 1 %u %u %u %u %u", &p.min_size, &p.normal_size, &p.max_size,
                              &p.strict_bits, &p.loose_bits) == 5;
    std::map<std::string, ChunkMemo::Entry> files;
    while (ok && (n = getline(&line, &cap, f)) > 0) {
        if (line[n - 1] == '\n')
            line[--n] = 0;
        ChunkMemo::Entry e;
        unsigned long long rows = 0;
        int used = 0, used2 = 0;
        if (!parse_file_id(line, &e.id, &used) || sscanf(line + used, " %llu %n", &rows, &used2) != 1 || used2 <= 0 ||
            used + used2 >= n || rows > (uint64_t)e.id.size) { // a chunk holds at least one byte
            ok = false;
            break;
        }
        e.digests.resize(32 * rows);
        ok = fread(e.digests.data(), 1, e.digests.size(), f) == e.digests.size();
        files[line + used + used2] = std::move(e);
    }
    free(line);
    fclose(f);
    if (!ok) {
        set_err(err, errlen, "load chunk cache: not a mkhost-chunk-cache file");
        return -1;
    }
    if (memcmp(&p, &c->memo.cdc, sizeof p) != 0) { // entries cut under other parameters do not mix with these
        c->memo.files.clear();
        c->memo.cdc = p; // a commit under other parameters starts over (ChunkMemo::bind)
    }
    for (auto &kv : files)
        c->memo.files[kv.first] = std::move(kv.second);
    return 0;
}

int mkhost_context_crc32_cached(mksnap_t *eng, mkhost_crc_cache *cache, const void *prefix, size_t prefix_len,
                                const char *context_dir, const char *const *from_paths, size_t n_paths, int n_threads,
                                uint32_t *crc_out, uint64_t *stream_len_out, mkhost_crc_cache_stats *stats, char *err, size_t errlen)
{
    if (!cache) {
        set_err(err, errlen, "hash context sources: no cache object");
        return -1;
    }
    return context_crc32_impl(eng, cache, stats, prefix, prefix_len, context_dir, from_paths, n_paths, n_threads, crc_out,
                              stream_len_out, err, errlen);
}

// One engine session of mkhost_plan_cache_ids: the streams of the walked COPY/ADD steps `batch` (stream slot k = batch[k]).
// Every distinct path string / link target and every file not yet valued travels once as CRC extents (crc_suffix 0:
// only pure(extent) is wanted); each occurrence in a stream becomes a use of those extents, or of a known value.
using FileKey = std::tuple<std::string, uint64_t, uint64_t, uint64_t, int64_t, int64_t>; // path, dev, ino, size, mtime, ctime
static FileKey file_key(const Seg &g) { return FileKey{g.path, g.id.dev, g.id.ino, g.size, g.id.mtime_ns, g.id.ctime_ns}; }

static void plan_session(mksnap_t *eng, mkhost_crc_cache *cache, const std::vector<std::vector<Seg>> &segs,
                         const std::vector<size_t> &batch, int n_threads, std::map<FileKey, uint32_t> &known,
                         bool remember, std::vector<uint32_t> &pure, std::vector<uint64_t> &slen,
                         mkhost_crc_cache_stats &st, double &ms_fold)
{
    ArenaSession s(eng, n_threads, 1); // cap unrounded, as in the single-step pass
    ck(eng, mksnap_begin(eng), "begin");
    s.acquire();
    uint64_t n_ext = 0; // CRC extents submitted so far (mksnap_get_extent_crcs numbering)
    auto place = [&](uint64_t align, uint64_t need) {
        uint64_t o = align_up(s.pos, align);
        if (o + need > s.cap || !s.room(1, 0)) {
            s.submit();
            s.acquire();
            o = 0;
        }
        return o;
    };
    std::map<std::string, uint64_t> text_ext; // path string / link target -> its extent
    auto put_text = [&](const std::string &b) {
        auto it = text_ext.find(b);
        if (it != text_ext.end())
            return it->second;
        if (b.size() > s.cap)
            throw HostError("path string larger than the arena");
        const uint64_t o = place(16, b.size());
        memcpy(s.a + o, b.data(), b.size());
        s.ext.push_back(mksnap_extent{o, b.size(), 0, MKSNAP_X_CRC, 0});
        s.pos = o + b.size();
        text_ext.emplace(b, n_ext);
        return n_ext++;
    };
    struct Sent { // a file that travelled: extents [first, first + pieces) and their lengths
        const Seg *seg;
        uint64_t first;
        std::vector<uint64_t> piece_len;
    };
    std::vector<Sent> sent;
    std::map<FileKey, size_t> sent_of;
    auto put_file = [&](const Seg &g) { // CRC is linear: a file may be split across arenas at any 16-byte boundary
        Sent f{&g, n_ext, {}};
        for (uint64_t done = 0; done < g.size;) {
            const uint64_t o = place(512, 4096);
            const uint64_t n = std::min<uint64_t>(g.size - done, (s.cap - o) / 16 * 16);
            s.jobs.push_back(ReadJob{g.path, done, n, s.a + o});
            s.ext.push_back(mksnap_extent{o, n, 0, MKSNAP_X_CRC, 0});
            ++n_ext;
            f.piece_len.push_back(n);
            s.pos = o + n;
            done += n;
        }
        st.bytes_sent += g.size;
        sent.push_back(std::move(f));
        return sent.size() - 1;
    };
    std::vector<mksnap_crc_use> uses; // grouped by stream, as k_crc_fold prefers them
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
                if (!g.bytes.empty())
                    uses.push_back(mksnap_crc_use{after, put_text(g.bytes), slot, 0});
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
            const Sent &f = sent[so != sent_of.end() ? so->second : (sent_of[key] = put_file(g))];
            uint64_t a = after + g.size;
            for (size_t p = 0; p < f.piece_len.size(); ++p) {
                a -= f.piece_len[p];
                uses.push_back(mksnap_crc_use{a, f.first + p, slot, 0});
            }
        }
    }
    s.submit();
    const auto t_fold = std::chrono::steady_clock::now();
    for (size_t u0 = 0; u0 < uses.size(); u0 += s.lim.max_extents)
        ck(eng, mksnap_crc_fold(eng, uses.data() + u0, std::min<uint64_t>(s.lim.max_extents, uses.size() - u0)), "crc fold");
    mksnap_result res;
    ck(eng, mksnap_finish(eng, &res), "finish");
    ms_fold += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_fold).count();
    std::vector<uint32_t> val(batch.size());
    uint64_t n_val = 0;
    ck(eng, mksnap_get_crc_streams(eng, val.data(), val.size(), &n_val), "crc streams");
    for (size_t k = 0; k < batch.size(); ++k)
        pure[batch[k]] = k < n_val ? val[k] : 0u; // a stream nothing was folded into is empty
    if (sent.empty() || !(cache || remember))
        return;
    std::vector<uint32_t> ext(n_ext);
    uint64_t n_got = 0;
    ck(eng, mksnap_get_extent_crcs(eng, ext.data(), ext.size(), &n_got), "extent crcs");
    if (n_got != n_ext)
        throw HostError("internal: extent count mismatch");
    for (const Sent &f : sent) { // pure(A||B) = pure(A) x^(8|B|) ^ pure(B)
        uint32_t v = 0;
        for (size_t p = 0; p < f.piece_len.size(); ++p)
            v = mksnap_crc_concat(v, ext[f.first + p], f.piece_len[p]);
        const Seg &g = *f.seg;
        if (cache)
            cache->files[g.path] = mkhost_crc_cache::Entry{g.id, v};
        if (remember)
            known[file_key(g)] = v;
    }
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
        const double ms_walk = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
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
                    n_steps, walked.size(), n_sessions, ms_walk, ms_fold,
                    std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count());
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
