// lb200_search_daemon -- funnels single-query index scans from many clients into GPU batches.  SURVEY.md 8f-3.
//
// Why: a Postgres backend runs one query at a time (lantern_hnsw/src/hnsw/scan.c:64 num_threads = 1, :220-228 one
// usearch_search_ef per scan) while the engine needs batches of ~1000 queries to reach the HBM roofline.  The daemon owns
// one index handle (loaded from a usearch/lantern index file; with --devices, a row-sharded group of GPUs loaded from it
// instead), accepts connections on a Unix-domain or TCP socket, collects
// the requests that arrive within a short window and serves them with ONE lb200_search_batch call per (k, ef) group.
// It implements ldb_amgettuple's call pattern (scan.c:167-338): first fetch with k = init_k, then `continue` requests that
// return the NEXT k results of the same query (never a row twice), per connection.
//
// Wire format (little-endian; one request -> one response, any number per connection):
//   request : u32 magic 'LBQ1' | u32 k | u32 ef (0 = index default) | u32 flags (bit0 = continue previous query)
//             | u32 nbytes | nbytes of query vector (f32[dims], or packed bits for a b1 index; ignored when continuing)
//   response: u32 status (0 = ok) | u32 found | found x u64 keys | found x f32 distances      (ascending distance)
//             status != 0: u32 length | message
//   stats   : request with magic 'LBQS' (no body) -> u64 requests, u64 batches, u64 largest batch
// The client side for scan.c is a dozen lines (see INTEGRATION.md); lb200d_* helpers below are exported by the daemon's
// own translation unit for tests written in C.
#include <arpa/inet.h>
#include <errno.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <signal.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/lantern_b200.h"

namespace {

constexpr uint32_t kMagicQuery = 0x3151424Cu; // "LBQ1"
constexpr uint32_t kMagicStats = 0x5351424Cu; // "LBQS"

bool read_exact(int fd, void* buf, size_t n) {
    uint8_t* p = (uint8_t*)buf;
    while (n) {
        ssize_t r = ::recv(fd, p, n, 0);
        if (r == 0)
            return false;
        if (r < 0) {
            if (errno == EINTR)
                continue;
            return false;
        }
        p += r, n -= (size_t)r;
    }
    return true;
}
bool write_all(int fd, const void* buf, size_t n) {
    const uint8_t* p = (const uint8_t*)buf;
    while (n) {
        ssize_t w = ::send(fd, p, n, MSG_NOSIGNAL);
        if (w < 0) {
            if (errno == EINTR)
                continue;
            return false;
        }
        p += w, n -= (size_t)w;
    }
    return true;
}

struct Request {
    uint32_t k = 0, ef = 0, want = 0; // want = already returned + k when continuing
    std::vector<uint8_t> query;
    std::vector<uint64_t> keys;
    std::vector<float> dists;
    size_t found = 0;
    std::string error;
    bool done = false;
    std::mutex mu;
    std::condition_variable cv;
};

struct Daemon {
    lb200_index_t idx = nullptr;
    lb200_group_t group = nullptr; // --devices: the index is served by a row-sharded group of GPUs (lb200_group_*)
    lb200_scalar_kind_t in_kind = lb200_scalar_f32_k;
    size_t qbytes = 0;
    size_t max_batch = 1024;
    int window_us = 200;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::shared_ptr<Request>> queue;
    std::atomic<uint64_t> n_requests{0}, n_batches{0}, max_seen{0};
    std::atomic<bool> stop{false};

    void batcher() {
        std::vector<std::shared_ptr<Request>> batch;
        std::vector<uint8_t> qbuf;
        std::vector<uint64_t> keys;
        std::vector<float> dists;
        std::vector<size_t> counts;
        for (;;) {
            batch.clear();
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return stop.load() || !queue.empty(); });
                if (stop.load() && queue.empty())
                    return;
                // give concurrent backends a moment to pile up, unless a full batch is already waiting
                if (queue.size() < max_batch) {
                    auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(window_us);
                    cv.wait_until(lk, deadline, [&] { return queue.size() >= max_batch || stop.load(); });
                }
                // one (want, ef) group per launch: results depend on both (expansion = max(ef, k), index.hpp:2706)
                const uint32_t want = queue.front()->want, ef = queue.front()->ef;
                for (auto it = queue.begin(); it != queue.end() && batch.size() < max_batch;) {
                    if ((*it)->want == want && (*it)->ef == ef) {
                        batch.push_back(*it);
                        it = queue.erase(it);
                    } else
                        ++it;
                }
            }
            const size_t n = batch.size(), want = batch[0]->want;
            qbuf.resize(n * qbytes), keys.resize(n * want), dists.resize(n * want), counts.resize(n);
            for (size_t i = 0; i < n; ++i)
                memcpy(qbuf.data() + i * qbytes, batch[i]->query.data(), qbytes);
            lb200_error_t err = nullptr;
            if (group)
                lb200_group_search_batch(group, qbuf.data(), n, qbytes, in_kind, want, batch[0]->ef, keys.data(), dists.data(),
                                         counts.data(), &err);
            else
                lb200_search_batch(idx, qbuf.data(), n, qbytes, in_kind, want, batch[0]->ef, keys.data(), dists.data(),
                                   counts.data(), &err);
            n_batches++;
            uint64_t prev = max_seen.load();
            while (n > prev && !max_seen.compare_exchange_weak(prev, n)) {
            }
            for (size_t i = 0; i < n; ++i) {
                Request& r = *batch[i];
                std::lock_guard<std::mutex> g(r.mu);
                if (err)
                    r.error = err;
                else {
                    r.found = counts[i];
                    r.keys.assign(keys.begin() + i * want, keys.begin() + i * want + counts[i]);
                    r.dists.assign(dists.begin() + i * want, dists.begin() + i * want + counts[i]);
                }
                r.done = true;
                r.cv.notify_one();
            }
        }
    }

    void serve(int fd) {
        std::vector<uint8_t> last_query;
        std::vector<uint64_t> returned; // keys handed out for last_query (scan.c streaming)
        for (;;) {
            uint32_t magic;
            if (!read_exact(fd, &magic, 4))
                break;
            if (magic == kMagicStats) {
                uint64_t st[3] = {n_requests.load(), n_batches.load(), max_seen.load()};
                if (!write_all(fd, st, sizeof(st)))
                    break;
                continue;
            }
            uint32_t hdr[4];
            if (magic != kMagicQuery || !read_exact(fd, hdr, sizeof(hdr)))
                break;
            const uint32_t k = hdr[0], ef = hdr[1], flags = hdr[2], nbytes = hdr[3];
            if (nbytes > std::max<size_t>(qbytes, 1u << 16)) { // never size a buffer from an unchecked wire field
                const std::string msg = "query body too large for this index";
                uint32_t head[2] = {1u, (uint32_t)msg.size()};
                if (write_all(fd, head, sizeof(head)))
                    write_all(fd, msg.data(), msg.size());
                break; // the stream cannot be resynchronised without reading the body: drop the connection
            }
            std::vector<uint8_t> body(nbytes);
            if (nbytes && !read_exact(fd, body.data(), nbytes))
                break;
            std::string error;
            const bool cont = flags & 1u;
            if (!cont) {
                if (nbytes != qbytes)
                    error = "query has the wrong size for this index";
                else
                    last_query = body, returned.clear();
            } else if (last_query.empty())
                error = "continue without a preceding query on this connection";
            if (k == 0 || returned.size() + k > 4096)
                error = "k out of range";
            auto req = std::make_shared<Request>();
            if (error.empty()) {
                req->k = k, req->ef = ef, req->want = (uint32_t)(returned.size() + k);
                req->query = last_query;
                n_requests++;
                {
                    std::lock_guard<std::mutex> g(mu);
                    queue.push_back(req);
                }
                cv.notify_all();
                std::unique_lock<std::mutex> lk(req->mu);
                req->cv.wait(lk, [&] { return req->done; });
                error = req->error;
            }
            if (!error.empty()) {
                uint32_t head[2] = {1u, (uint32_t)error.size()};
                if (!write_all(fd, head, sizeof(head)) || !write_all(fd, error.data(), error.size()))
                    break;
                continue;
            }
            // hand out the closest k results not returned before on this connection (filter by key: a wider beam may
            // rank earlier results differently)
            std::vector<uint64_t> seen(returned);
            std::sort(seen.begin(), seen.end());
            std::vector<uint64_t> ok;
            std::vector<float> od;
            for (size_t i = 0; i < req->found && ok.size() < k; ++i) {
                if (std::binary_search(seen.begin(), seen.end(), req->keys[i]))
                    continue;
                ok.push_back(req->keys[i]), od.push_back(req->dists[i]);
                returned.push_back(req->keys[i]);
            }
            uint32_t head[2] = {0u, (uint32_t)ok.size()};
            if (!write_all(fd, head, sizeof(head)) || !write_all(fd, ok.data(), ok.size() * 8) ||
                !write_all(fd, od.data(), od.size() * 4))
                break;
        }
        close(fd);
    }
};

int parse_metric(const std::string& s) {
    if (s == "cos")
        return lb200_metric_cos_k;
    if (s == "hamming")
        return lb200_metric_hamming_k;
    return lb200_metric_l2sq_k;
}
int parse_quant(const std::string& s) {
    if (s == "f16")
        return lb200_scalar_f16_k;
    if (s == "i8")
        return lb200_scalar_i8_k;
    if (s == "b1")
        return lb200_scalar_b1_k;
    return lb200_scalar_f32_k;
}

} // namespace

int main(int argc, char** argv) {
    std::string index_path, sock_path, metric = "l2sq", quant = "f32", devices;
    int port = 0;
    size_t dims = 0, m = 16, efc = 128, ef = 64;
    Daemon d;
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto next = [&]() -> const char* { return i + 1 < argc ? argv[++i] : ""; };
        if (a == "--index")
            index_path = next();
        else if (a == "--socket")
            sock_path = next();
        else if (a == "--port")
            port = atoi(next());
        else if (a == "--dim")
            dims = (size_t)atol(next());
        else if (a == "--metric")
            metric = next();
        else if (a == "--quant")
            quant = next();
        else if (a == "--m")
            m = (size_t)atol(next());
        else if (a == "--ef-construction")
            efc = (size_t)atol(next());
        else if (a == "--ef")
            ef = (size_t)atol(next());
        else if (a == "--max-batch")
            d.max_batch = (size_t)atol(next());
        else if (a == "--window-us")
            d.window_us = atoi(next());
        else if (a == "--devices") // e.g. 0,1,2,3,4,5,6,7: serve the index from a row-sharded group of these GPUs
            devices = next();
        else {
            fprintf(stderr,
                    "usage: %s --index FILE --dim D [--metric l2sq|cos|hamming] [--quant f32|f16|i8|b1] [--m M] [--ef EF]\n"
                    "          (--socket PATH | --port P) [--max-batch N] [--window-us U] [--devices 0,1,...]\n",
                    argv[0]);
            return 2;
        }
    }
    d.max_batch = std::max<size_t>(d.max_batch, 1);
    if (index_path.empty() || !dims || (sock_path.empty() && !port)) {
        fprintf(stderr, "need --index, --dim and one of --socket / --port\n");
        return 2;
    }
    signal(SIGPIPE, SIG_IGN);
    lb200_init_options_t o;
    memset(&o, 0, sizeof(o));
    o.metric_kind = (lb200_metric_kind_t)parse_metric(metric);
    o.quantization = (lb200_scalar_kind_t)parse_quant(quant);
    o.dimensions = dims, o.connectivity = m, o.expansion_add = efc, o.expansion_search = ef;
    lb200_error_t err = nullptr;
    d.in_kind = o.quantization == lb200_scalar_b1_k ? lb200_scalar_b1_k : lb200_scalar_f32_k;
    d.qbytes = d.in_kind == lb200_scalar_b1_k ? (dims + 7) / 8 : dims * 4;
    size_t vectors = 0;
    if (devices.empty()) {
        d.idx = lb200_init(&o, nullptr, &err);
        if (err) {
            fprintf(stderr, "lb200_init: %s\n", err);
            return 1;
        }
        lb200_load(d.idx, index_path.c_str(), &err);
        if (err) {
            fprintf(stderr, "lb200_load: %s\n", err);
            return 1;
        }
        vectors = lb200_size(d.idx, &err);
    } else {
        // one graph over several GPUs: rows sharded by range, distances evaluated on the owning GPU, results identical to the
        // single-GPU search (csrc/group.cu).  Every GPU reads its rows and the graph straight from the file: no GPU holds
        // the whole index, so the file may be larger than one GPU.
        std::vector<int> devs;
        for (size_t at = 0; at < devices.size();) {
            devs.push_back(atoi(devices.c_str() + at));
            const size_t comma = devices.find(',', at);
            if (comma == std::string::npos)
                break;
            at = comma + 1;
        }
        d.group = lb200_group_create_local(devs.data(), (int)devs.size(), &err);
        if (!err) // streaming scans ask for up to 1000 rows per query (scan.c:249-252)
            lb200_group_load(d.group, &o, index_path.c_str(), 0, d.max_batch, d.max_batch * 1000, &err);
        if (err) {
            fprintf(stderr, "lb200_group: %s\n", err);
            return 1;
        }
        fprintf(stderr, "lb200_search_daemon: serving from %zu GPUs (row-sharded group)\n", devs.size());
        for (size_t r = 0; r < devs.size(); ++r) {
            lb200_group_rank_info_t info;
            lb200_group_rank_info(d.group, (int)r, &info, &err);
            if (err) {
                fprintf(stderr, "lb200_group_rank_info: %s\n", err);
                return 1;
            }
            vectors = std::max<size_t>(vectors, info.rows_end);
            fprintf(stderr,
                    "lb200_search_daemon: rank %d on GPU %d: rows [%llu, %llu), device MB: rows %.1f, graph %.1f, scratch %.1f, "
                    "mailbox %.1f\n",
                    info.rank, devs[r], (unsigned long long)info.rows_begin, (unsigned long long)info.rows_end,
                    info.bytes_rows / 1e6, info.bytes_graph / 1e6, info.bytes_scratch / 1e6, info.bytes_mailbox / 1e6);
        }
    }

    int ls;
    if (!sock_path.empty()) {
        ls = socket(AF_UNIX, SOCK_STREAM, 0);
        sockaddr_un addr;
        memset(&addr, 0, sizeof(addr));
        addr.sun_family = AF_UNIX;
        strncpy(addr.sun_path, sock_path.c_str(), sizeof(addr.sun_path) - 1);
        unlink(sock_path.c_str());
        if (bind(ls, (sockaddr*)&addr, sizeof(addr)) != 0 || listen(ls, 256) != 0) {
            fprintf(stderr, "cannot listen on %s: %s\n", sock_path.c_str(), strerror(errno));
            return 1;
        }
    } else {
        ls = socket(AF_INET, SOCK_STREAM, 0);
        int one = 1;
        setsockopt(ls, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
        sockaddr_in addr;
        memset(&addr, 0, sizeof(addr));
        addr.sin_family = AF_INET, addr.sin_port = htons((uint16_t)port);
        inet_pton(AF_INET, "127.0.0.1", &addr.sin_addr);
        if (bind(ls, (sockaddr*)&addr, sizeof(addr)) != 0 || listen(ls, 256) != 0) {
            fprintf(stderr, "cannot listen on 127.0.0.1:%d: %s\n", port, strerror(errno));
            return 1;
        }
    }
    fprintf(stderr, "lb200_search_daemon: %zu vectors, batching up to %zu queries per %d us window\n", vectors, d.max_batch,
            d.window_us);
    std::thread batcher([&] { d.batcher(); });
    for (;;) {
        int fd = accept(ls, nullptr, nullptr);
        if (fd < 0) {
            if (errno == EINTR)
                continue;
            break;
        }
        int one = 1;
        setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
        std::thread([&d, fd] {
            try {
                d.serve(fd);
            } catch (const std::exception& e) { // e.g. bad_alloc: lose the connection, not the daemon
                fprintf(stderr, "lb200_search_daemon: connection dropped: %s\n", e.what());
                close(fd);
            }
        }).detach();
    }
    d.stop = true;
    d.cv.notify_all();
    batcher.join();
    return 0;
}
