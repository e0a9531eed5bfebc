// lantern_b200 -- reader/writer of the usearch/lantern index file format.
//
// Byte layout (verified against the compiled reference, SURVEY.md Appendix B):
//   index_dense_head_t          U/include/usearch/index_dense.hpp:42-79    80 bytes
//       "usearch" | u16 x3 version 2.8.14 | u8 metric ('e','c','b',...) | u8 scalar kind | u8 key kind (8 = u64)
//       | u8 slot kind (16 = u48) | u64 count_present | u64 count_deleted | u64 dimensions | u8 multi | zero pad
//   index_serialized_header_t   U/include/usearch/index.hpp:1696-1703      40 bytes
//       u64 size, connectivity, connectivity_base, max_level, entry_slot
//   lantern storage             U/include/usearch/lantern_storage.hpp:486-521
//       u64 vector_size_bytes | u64 node_count | per node:
//       u64 key | i16 level | u32 cnt + M0 x uint48 | level x (u32 cnt + M x uint48) | vector bytes or PQ codes
// No padding anywhere (align4 returns 0, lantern_storage.hpp:207-211).  Slots are sequential insertion ids.
// The HBM side keeps u32 ids in fixed-width, 0xFFFFFFFF-padded lists; only this file speaks uint48.
#include <string.h>

#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#include "engine.h"

namespace lb200 {

namespace {

uint8_t metric_char(int m) {
    switch (m) {
    case MK_COS: return 'c';
    case MK_IP: return 'i';
    case MK_L2SQ: return 'e';
    case MK_HAMMING: return 'b';
    default: return 0;
    }
}
uint8_t scalar_code(int k) { // scalar_kind_t, index_plugins.hpp:130-152
    switch (k) {
    case SK_B1: return 1;
    case SK_F64: return 4;
    case SK_F32: return 5;
    case SK_F16: return 6;
    case SK_I8: return 15;
    default: return 0;
    }
}

uint8_t* put_list(uint8_t* p, const uint32_t* ids, size_t width) {
    uint32_t cnt = 0;
    while (cnt < width && ids[cnt] != kNoNeighbor)
        ++cnt;
    memcpy(p, &cnt, 4);
    p += 4;
    memset(p, 0, 6 * width);
    for (uint32_t i = 0; i < cnt; ++i) {
        uint64_t v = ids[i];
        memcpy(p + 6 * i, &v, 6);
    }
    return p + 6 * width;
}

const uint8_t* get_list(const uint8_t* p, uint32_t* ids, size_t width, size_t n_nodes) {
    uint32_t cnt;
    memcpy(&cnt, p, 4);
    if (cnt > width)
        throw CudaError("index file: neighbour count exceeds connectivity");
    p += 4;
    for (size_t i = 0; i < width; ++i) {
        uint64_t v = 0;
        memcpy(&v, p + 6 * i, 6);
        if (i < cnt && v >= n_nodes)
            throw CudaError("index file: neighbour slot out of range (expected sequential ids)");
        ids[i] = i < cnt ? (uint32_t)v : kNoNeighbor;
    }
    return p + 6 * width;
}

} // namespace

// caller holds mu_
size_t Index::serialized_length_locked() {
    if (pending_n_)
        build_pending(*this);
    size_t total = 136;
    for (size_t i = 0; i < n_; ++i)
        total += 10 + (4 + 6 * cfg_.M0) + (size_t)h_levels_[i] * (4 + 6 * cfg_.M) + stored_bytes_;
    return total;
}

size_t Index::serialized_length() {
    flush_staged();
    std::lock_guard<std::mutex> g(mu_);
    return serialized_length_locked();
}

// The 136 bytes in front of the node tapes: dense head, serialized header, vector_size_bytes, node_count.  Caller holds mu_.
void Index::fill_header(uint8_t* p) const {
    memset(p, 0, 80);
    memcpy(p, "usearch", 7);
    const uint16_t ver[3] = {2, 8, 14};
    memcpy(p + 7, ver, 6);
    p[13] = metric_char(cfg_.metric_kind), p[14] = scalar_code(cfg_.scalar_kind), p[15] = 8, p[16] = 16;
    uint64_t v = n_;
    memcpy(p + 17, &v, 8);
    v = 0;
    memcpy(p + 25, &v, 8);
    v = cfg_.dims;
    memcpy(p + 33, &v, 8);
    const uint64_t hdr[7] = {n_, cfg_.M, cfg_.M0, (uint64_t)(max_level_ < 0 ? 0 : max_level_), entry_, vec_bytes_, n_};
    memcpy(p + 80, hdr, 56);
}

// usearch_update_header (U/c/lib.cpp:213-217 -> index_dense.hpp:962-965): the first 136 bytes of a save.
void Index::write_header(void* headerp) {
    flush_staged();
    std::lock_guard<std::mutex> g(mu_);
    if (pending_n_)
        build_pending(*this);
    fill_header((uint8_t*)headerp);
}

size_t Index::save_buffer(void* buffer, size_t length) {
    flush_staged();
    std::lock_guard<std::mutex> g(mu_); // length check and node loop under ONE hold: a concurrent add cannot grow n_ in between
    const size_t need = serialized_length_locked();
    if (length < need)
        throw CudaError("save_buffer: buffer too small (see lb200_serialized_length)");
    const size_t M = cfg_.M, M0 = cfg_.M0;
    std::vector<uint32_t> adj0(n_ * M0), upper_ref(n_), upper_adj(upper_lists_ * M);
    std::vector<uint8_t> rows(n_ * row_bytes_);
    LB_CUDA(cudaDeviceSynchronize());
    if (n_) {
        LB_CUDA(cudaMemcpy(adj0.data(), d_adj0_, adj0.size() * 4, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(upper_ref.data(), d_upper_ref_, upper_ref.size() * 4, cudaMemcpyDeviceToHost));
        if (!upper_adj.empty())
            LB_CUDA(cudaMemcpy(upper_adj.data(), d_upper_adj_, upper_adj.size() * 4, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(rows.data(), d_vectors_, rows.size(), cudaMemcpyDeviceToHost));
    }
    uint8_t* p = (uint8_t*)buffer;
    fill_header(p);
    p += 136;
    for (size_t i = 0; i < n_; ++i) {
        memcpy(p, &h_keys_[i], 8);
        memcpy(p + 8, &h_levels_[i], 2);
        p += 10;
        p = put_list(p, adj0.data() + i * M0, M0);
        for (int l = 1; l <= h_levels_[i]; ++l)
            p = put_list(p, upper_adj.data() + ((size_t)upper_ref[i] + (l - 1)) * M, M);
        memcpy(p, rows.data() + i * row_bytes_, stored_bytes_);
        p += stored_bytes_;
    }
    return (size_t)(p - (uint8_t*)buffer);
}

void save_row_sharded(Index& graph, const std::vector<RowShard>& shards, const std::function<void(const void*, size_t)>& write) {
    const size_t n = graph.n_, M = graph.cfg_.M, M0 = graph.cfg_.M0, row_bytes = graph.row_bytes_, stored = graph.stored_bytes_;
    if (graph.pending_n_)
        throw CudaError("save: the index has rows that are not built yet");
    std::vector<uint32_t> adj0(n * M0), upper_ref(n), upper_adj(graph.upper_lists_ * M);
    LB_CUDA(cudaSetDevice(shards[0].device));
    LB_CUDA(cudaDeviceSynchronize());
    if (n) {
        LB_CUDA(cudaMemcpy(adj0.data(), graph.d_adj0_, adj0.size() * 4, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(upper_ref.data(), graph.d_upper_ref_, upper_ref.size() * 4, cudaMemcpyDeviceToHost));
        if (!upper_adj.empty())
            LB_CUDA(cudaMemcpy(upper_adj.data(), graph.d_upper_adj_, upper_adj.size() * 4, cudaMemcpyDeviceToHost));
    }
    uint8_t head[136];
    graph.fill_header(head);
    write(head, sizeof(head));
    // rows: a block of at most 32 MB at a time, from the rank whose range holds it
    const size_t block = std::max<size_t>(1, ((size_t)32 << 20) / row_bytes);
    std::vector<uint8_t> rows(std::min(block, std::max<size_t>(n, 1)) * row_bytes);
    size_t first = 0, count = 0;
    std::vector<uint8_t> tape(10 + (4 + 6 * M0) + (size_t)std::max(graph.max_level_, 0) * (4 + 6 * M) + stored);
    for (size_t i = 0; i < n; ++i) {
        if (i >= first + count) {
            size_t t = 0;
            while (t + 1 < shards.size() && i >= shards[t].idx->row_hi_)
                ++t;
            const Index& x = *shards[t].idx;
            if (i < x.row_lo_ || i >= x.row_hi_)
                throw CudaError("save: no rank holds row " + std::to_string(i));
            first = i, count = std::min(std::min(block, x.row_hi_ - i), n - i);
            LB_CUDA(cudaSetDevice(shards[t].device));
            LB_CUDA(cudaMemcpy(rows.data(), x.d_vectors_ + (i - x.row_lo_) * row_bytes, count * row_bytes, cudaMemcpyDeviceToHost));
        }
        uint8_t* p = tape.data();
        memcpy(p, &graph.h_keys_[i], 8);
        memcpy(p + 8, &graph.h_levels_[i], 2);
        p += 10;
        p = put_list(p, adj0.data() + i * M0, M0);
        for (int l = 1; l <= graph.h_levels_[i]; ++l)
            p = put_list(p, upper_adj.data() + ((size_t)upper_ref[i] + (l - 1)) * M, M);
        memcpy(p, rows.data() + (i - first) * row_bytes, stored);
        p += stored;
        write(tape.data(), (size_t)(p - tape.data()));
    }
}

void parse_index_file(const IndexConfig& cfg, size_t vec_bytes, size_t stored_bytes, const void* buffer, size_t length,
                      ParsedIndexFile& out) {
    const uint8_t* p = (const uint8_t*)buffer;
    if (length < 136 || memcmp(p, "usearch", 7) != 0)
        throw CudaError("index file: bad magic");
    if (p[15] != 8 || p[16] != 16)
        throw CudaError("index file: expected u64 keys and uint48 slots (lantern storage)");
    if (p[13] != metric_char(cfg.metric_kind) || p[14] != scalar_code(cfg.scalar_kind))
        throw CudaError("index file: metric / scalar kind differ from the index options");
    uint64_t dims;
    memcpy(&dims, p + 33, 8);
    if (dims != cfg.dims)
        throw CudaError("index file: dimensions differ from the index options");
    uint64_t hdr[7];
    memcpy(hdr, p + 80, 56);
    const size_t n = hdr[0], M = cfg.M, M0 = cfg.M0;
    if (hdr[1] != M || hdr[2] != M0)
        throw CudaError("index file: connectivity differs from the index options");
    if (hdr[5] != vec_bytes)
        throw CudaError("index file: vector_size_bytes mismatch");
    if (n >= 0x7FFFFFFFull)
        throw CudaError("index file: more than 2^31-1 nodes in one shard");

    std::vector<uint32_t> adj0(n * M0), upper_ref(n, kNoNeighbor), upper_adj;
    std::vector<int16_t> levels(n);
    std::vector<uint64_t> keys(n), row_off(n);
    const uint8_t* begin = p;
    const uint8_t* end = p + length;
    p += 136;
    std::vector<uint32_t> tmp(M);
    for (size_t i = 0; i < n; ++i) {
        if (p + 10 > end)
            throw CudaError("index file: truncated");
        memcpy(&keys[i], p, 8);
        memcpy(&levels[i], p + 8, 2);
        p += 10;
        if (levels[i] < 0)
            throw CudaError("index file: negative level");
        const size_t tape = (4 + 6 * M0) + (size_t)levels[i] * (4 + 6 * M) + stored_bytes;
        if (p + tape > end)
            throw CudaError("index file: truncated");
        p = get_list(p, adj0.data() + i * M0, M0, n);
        if (levels[i] > 0) {
            upper_ref[i] = (uint32_t)(upper_adj.size() / M);
            for (int l = 1; l <= levels[i]; ++l) {
                p = get_list(p, tmp.data(), M, n);
                upper_adj.insert(upper_adj.end(), tmp.begin(), tmp.end());
            }
        }
        row_off[i] = (uint64_t)(p - begin);
        p += stored_bytes;
    }
    if (n) { // the walk starts at entry_slot on level max_level: both must be consistent or the kernels would read out of bounds
        if (hdr[4] >= n)
            throw CudaError("index file: entry slot out of range");
        if ((int64_t)hdr[3] != (int64_t)levels[hdr[4]])
            throw CudaError("index file: entry node level differs from max_level");
        for (size_t i = 0; i < n; ++i) {
            if (levels[i] > (int16_t)hdr[3])
                throw CudaError("index file: node above max_level");
            for (int l = 1; l <= levels[i]; ++l) { // a level-l link must point to a node that exists on level l
                const uint32_t* list = upper_adj.data() + ((size_t)upper_ref[i] + (l - 1)) * M;
                for (size_t j = 0; j < M && list[j] != kNoNeighbor; ++j)
                    if (levels[list[j]] < l)
                        throw CudaError("index file: link to a node that is missing on that level");
            }
        }
    }
    out.n = n;
    out.max_level = n ? (int32_t)hdr[3] : -1;
    out.entry = (uint32_t)hdr[4];
    out.adj0 = std::move(adj0), out.upper_ref = std::move(upper_ref), out.upper_adj = std::move(upper_adj);
    out.levels = std::move(levels), out.keys = std::move(keys), out.row_off = std::move(row_off);
}

// usearch_load_buffer / usearch_view_buffer (U/c/lib.cpp:295-313): replaces the index contents.
void Index::load_buffer(const void* buffer, size_t length) {
    {
        std::lock_guard<std::mutex> sg(stage_mu_); // loading replaces the contents, staged rows included
        staged_rows_.clear(), staged_keys_.clear();
    }
    std::lock_guard<std::mutex> g(mu_);
    ParsedIndexFile f;
    parse_index_file(cfg_, vec_bytes_, stored_bytes_, buffer, length, f);
    const size_t n = f.n;
    std::vector<uint8_t> rows(n * row_bytes_, 0);
    for (size_t i = 0; i < n; ++i)
        memcpy(rows.data() + i * row_bytes_, (const uint8_t*)buffer + f.row_off[i], stored_bytes_);
    uint32_t pq_max_code = 0;
    if (cfg_.pq) { // codes written by other tools may use all 256 centroids: size the look-up tables accordingly
        for (size_t i = 0; i < n; ++i)
            for (size_t s2 = 0; s2 < stored_bytes_; ++s2) {
                const uint8_t c = rows[i * row_bytes_ + s2];
                if (c >= cfg_.num_centroids)
                    throw CudaError("corrupted centroid id"); // lantern_storage.hpp:141
                pq_max_code = std::max<uint32_t>(pq_max_code, c);
            }
        check_pq_table_fits(pq_lut_width(cfg_.num_centroids, pq_max_code));
    }
    // commit (nothing below throws for a reason that depends on the file contents)
    pq_max_code_ = pq_max_code;
    n_ = 0, pending_n_ = 0;
    ensure_capacity(n ? n : 1);
    reset_screen(); // the screen is chosen again from the loaded rows
    if (n) {
        LB_CUDA(cudaMemcpy(d_vectors_, rows.data(), rows.size(), cudaMemcpyHostToDevice));
        encode_screen(0, n);
    }
    commit_file_graph(f, true);
    decide_screen();
}

// load_buffer's commit of the graph, shared with a group index's load (group.cu)
void Index::commit_file_graph(ParsedIndexFile& f, bool host_mirrors) {
    const size_t n = f.n, M = cfg_.M, M0 = cfg_.M0;
    upper_lists_ = 0;
    alloc_upper(f.upper_adj.size() / M + 1);
    // everything beyond the loaded nodes / lists must read as empty (0xFF): a later insert with level > max_level exposes
    // its still-unwritten upper lists to greedy() before build_insert_kernel has filled them
    LB_CUDA(cudaMemset(d_adj0_, 0xFF, capacity_ * M0 * 4));
    LB_CUDA(cudaMemset(d_upper_ref_, 0xFF, capacity_ * 4));
    LB_CUDA(cudaMemset(d_upper_adj_, 0xFF, upper_lists_cap_ * M * 4));
    if (n) {
        LB_CUDA(cudaMemcpy(d_adj0_, f.adj0.data(), f.adj0.size() * 4, cudaMemcpyHostToDevice));
        LB_CUDA(cudaMemcpy(d_upper_ref_, f.upper_ref.data(), f.upper_ref.size() * 4, cudaMemcpyHostToDevice));
        if (!f.upper_adj.empty())
            LB_CUDA(cudaMemcpy(d_upper_adj_, f.upper_adj.data(), f.upper_adj.size() * 4, cudaMemcpyHostToDevice));
        LB_CUDA(cudaMemcpy(d_keys_, f.keys.data(), f.keys.size() * 8, cudaMemcpyHostToDevice));
    }
    upper_lists_ = f.upper_adj.size() / M;
    if (host_mirrors) {
        h_levels_ = std::move(f.levels);
        h_keys_ = std::move(f.keys);
    } else {
        h_levels_.clear(), h_keys_.clear();
    }
    n_ = n;
    max_level_ = f.max_level;
    entry_ = f.entry;
}

} // namespace lb200
