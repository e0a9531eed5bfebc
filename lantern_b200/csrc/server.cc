// lb200_index_server -- GPU external-indexing server speaking Lantern's wire protocol (SURVEY.md 8b "B2", 8f-1).
//
// Drop-in for `lantern_cli start-indexing-server` (lantern_cli/src/external_index/server.rs:311-435, 526-584) as seen by
// the Postgres side (lantern_hnsw/src/hnsw/external_index_socket.{h,c}): `CREATE INDEX ... WITH (external=true)` then
// builds on the GPU with no change to Postgres.  Protocol, little-endian only (external_index_socket.c:337):
//   <- u32 protocol_version = 1, u32 server_type = 1                               server.rs:182-183
//   -> u32 INIT_MSG 0x13333337 + 11 x u32 {pq, metric_kind, quantization, dim, m, ef_construction, ef, num_centroids,
//      num_subvectors, estimated_capacity, element_bits}                           external_index_socket.h:25-39
//   -> [pq] num_centroids frames of dim x f32, then u32 END_MSG 0x31333337           server.rs:109-130
//   <- u8 0 (ready)                                                                server.rs:206
//   -> per row [u64 label][vector bytes]: dim x element_bits/8 bytes, or ceil(dim/8) bytes when element_bits < 8
//      (hamming: dim already counts bits)                                          server.rs:226-263
//   -> u32 END_MSG ; <- u64 rows indexed, u64 file size, index file bytes (usearch/lantern format)   server.rs:388-422
//   errors: <- u32 ERR_MSG 0x37333337, u32 length, text                            server.rs:563-573
// The library underneath is the C ABI of include/lantern_b200.h; rows are handed to the GPU in blocks
// (lb200_add_batch) instead of being fanned out over CPU threads (server.rs:317-359).  TLS and the router role
// (server_type 2) are not implemented.  With --devices 0,1,... every session's index is built on a single-process group
// of those GPUs (lb200_group_build, same file as the one-GPU build); the index lives on the first listed device.
#include <arpa/inet.h>
#include <dlfcn.h>
#include <errno.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <signal.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/time.h>
#include <unistd.h>

#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/lantern_b200.h"

namespace {

constexpr uint32_t kProtocolVersion = 1, kServerType = 1;
constexpr uint32_t kInitMsg = 0x13333337u, kEndMsg = 0x31333337u, kErrMsg = 0x37333337u;
constexpr size_t kBlockRows = 65536;

struct Conn {
    int fd;
    void read_exact(void* buf, size_t n) {
        uint8_t* p = (uint8_t*)buf;
        while (n) {
            ssize_t r = ::recv(fd, p, n, 0);
            if (r == 0)
                throw std::runtime_error("connection closed by peer");
            if (r < 0) {
                if (errno == EINTR)
                    continue;
                throw std::runtime_error(std::string("socket read failed: ") + strerror(errno));
            }
            p += r, n -= (size_t)r;
        }
    }
    void write_all(const void* buf, size_t n) {
        const uint8_t* p = (const uint8_t*)buf;
        while (n) {
            ssize_t w = ::send(fd, p, n, MSG_NOSIGNAL);
            if (w < 0) {
                if (errno == EINTR)
                    continue;
                throw std::runtime_error(std::string("socket write failed: ") + strerror(errno));
            }
            p += w, n -= (size_t)w;
        }
    }
};

void check(lb200_error_t err) {
    if (err)
        throw std::runtime_error(err);
}

// Makes `device` the current CUDA device of this thread through the driver API (the engine's runtime adopts the current
// context), so that lb200_init allocates there.  Loaded at run time: without --devices the server needs no driver.
bool make_device_current(int device) {
    void* cu = dlopen("libcuda.so.1", RTLD_NOW);
    if (!cu)
        return false;
    typedef int (*init_fn)(unsigned);
    typedef int (*get_fn)(int*, int);
    typedef int (*retain_fn)(void**, int);
    typedef int (*set_fn)(void*);
    init_fn cu_init = (init_fn)dlsym(cu, "cuInit");
    get_fn cu_device_get = (get_fn)dlsym(cu, "cuDeviceGet");
    retain_fn cu_retain = (retain_fn)dlsym(cu, "cuDevicePrimaryCtxRetain");
    set_fn cu_set = (set_fn)dlsym(cu, "cuCtxSetCurrent");
    int dev = 0;
    void* ctx = nullptr;
    return cu_init && cu_device_get && cu_retain && cu_set && cu_init(0) == 0 && cu_device_get(&dev, device) == 0 &&
           cu_retain(&ctx, dev) == 0 && cu_set(ctx) == 0;
}

void serve(Conn& c, bool verbose, lb200_group_t group) {
    const uint32_t hello[2] = {kProtocolVersion, kServerType};
    c.write_all(hello, sizeof(hello));

    uint32_t init[12];
    c.read_exact(init, sizeof(init));
    if (init[0] != kInitMsg)
        throw std::runtime_error("send init message first");
    const uint32_t pq = init[1], metric_kind = init[2], quantization = init[3], dim = init[4], m = init[5], efc = init[6],
                   ef = init[7], num_centroids = init[8], num_subvectors = init[9], capacity = init[10], element_bits = init[11];
    if (quantization > 5)
        throw std::runtime_error("Invalid scalar quantization");
    // everything below sizes buffers from these fields: refuse nonsense before allocating (the library re-checks the rest)
    if (dim == 0 || dim > 65536)
        throw std::runtime_error("vector dimensions must be in [1, 65536]");
    if (element_bits >= 8 && element_bits != 32)
        throw std::runtime_error("only 32-bit float rows (or packed bits) are accepted");
    if (pq == 1 && (num_centroids == 0 || num_centroids > 256 || num_subvectors == 0))
        throw std::runtime_error("pq needs 1..256 centroids and a nonzero number of subvectors");

    std::vector<float> codebook;
    if (pq == 1) { // frames of dim floats until END_MSG (server.rs:109-130)
        std::vector<uint8_t> frame((size_t)dim * 4);
        for (;;) {
            c.read_exact(frame.data(), 4);
            uint32_t head;
            memcpy(&head, frame.data(), 4);
            if (head == kEndMsg)
                break;
            if (codebook.size() >= (size_t)num_centroids * dim)
                throw std::runtime_error("codebook has more rows than num_centroids");
            c.read_exact(frame.data() + 4, frame.size() - 4);
            const float* f = (const float*)frame.data();
            codebook.insert(codebook.end(), f, f + dim);
        }
        if (codebook.size() != (size_t)num_centroids * dim)
            throw std::runtime_error("codebook size does not match num_centroids x dim");
    }

    lb200_init_options_t o;
    memset(&o, 0, sizeof(o));
    o.metric_kind = (lb200_metric_kind_t)metric_kind;
    o.quantization = quantization <= 1 ? lb200_scalar_f32_k : (lb200_scalar_kind_t)quantization; // server.rs:96-103
    o.dimensions = dim;
    o.connectivity = m, o.expansion_add = efc, o.expansion_search = ef;
    o.pq = pq == 1, o.num_centroids = num_centroids, o.num_subvectors = num_subvectors;
    lb200_error_t err = nullptr;
    lb200_index_t idx = lb200_init(&o, codebook.empty() ? nullptr : codebook.data(), &err);
    check(err);
    struct Guard {
        lb200_index_t h;
        ~Guard() {
            lb200_error_t e = nullptr;
            lb200_free(h, &e);
        }
    } guard{idx};
    lb200_reserve(idx, capacity ? capacity : 1, &err);
    check(err);
    const uint8_t ready = 0;
    c.write_all(&ready, 1);

    // rows (server.rs:226-263): element_bits < 8 -> packed bits, else dim * element_bits/8 bytes
    const size_t vec_bytes = element_bits < 8 ? ((size_t)dim + 7) / 8 : (size_t)dim * (element_bits / 8);
    const lb200_scalar_kind_t in_kind = element_bits < 8 ? lb200_scalar_b1_k : lb200_scalar_f32_k;
    const size_t frame_bytes = 8 + vec_bytes;
    std::vector<uint8_t> frame(frame_bytes);
    std::vector<uint64_t> keys;
    std::vector<uint8_t> rows;
    keys.reserve(kBlockRows), rows.reserve(kBlockRows * vec_bytes);
    size_t received = 0, cap = capacity ? capacity : 1;
    auto flush = [&]() {
        if (keys.empty())
            return;
        if (received > cap) { // server.rs:246-249: grow by doubling
            while (cap < received)
                cap *= 2;
            lb200_reserve(idx, cap, &err);
            check(err);
        }
        lb200_add_batch(idx, keys.data(), rows.data(), keys.size(), vec_bytes, in_kind, &err);
        check(err);
        keys.clear(), rows.clear();
    };
    for (;;) {
        c.read_exact(frame.data(), 4);
        uint32_t head;
        memcpy(&head, frame.data(), 4);
        if (head == kEndMsg)
            break;
        c.read_exact(frame.data() + 4, frame_bytes - 4);
        uint64_t label;
        memcpy(&label, frame.data(), 8);
        keys.push_back(label);
        rows.insert(rows.end(), frame.begin() + 8, frame.end());
        ++received;
        if (keys.size() == kBlockRows)
            flush();
    }
    flush();
    if (group)
        lb200_group_build(group, idx, 0, &err);
    else
        lb200_build(idx, &err);
    check(err);

    const uint64_t count = lb200_size(idx, &err);
    check(err);
    const size_t len = lb200_serialized_length(idx, &err);
    check(err);
    std::vector<uint8_t> file(len);
    lb200_save_buffer(idx, file.data(), file.size(), &err);
    check(err);
    const uint64_t file_size = file.size();
    c.write_all(&count, 8);
    c.write_all(&file_size, 8);
    c.write_all(file.data(), file.size());
    if (verbose)
        fprintf(stderr, "lb200_index_server: indexed %llu rows, sent %llu bytes\n", (unsigned long long)count,
                (unsigned long long)file_size);
}

} // namespace

int main(int argc, char** argv) {
    const char* host = "127.0.0.1";
    int port = 8998; // lantern_extras/src/lib.rs:172-237 hosts the reference server on 127.0.0.1:8998
    int max_sessions = -1;
    bool verbose = true;
    std::vector<int> devices;
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        if (a == "--host" && i + 1 < argc)
            host = argv[++i];
        else if (a == "--port" && i + 1 < argc)
            port = atoi(argv[++i]);
        else if (a == "--sessions" && i + 1 < argc)
            max_sessions = atoi(argv[++i]);
        else if (a == "--quiet")
            verbose = false;
        else if (a == "--devices" && i + 1 < argc) { // e.g. 0,1,2,3: build every index on a group of these GPUs
            const std::string list = argv[++i];
            for (size_t at = 0; at < list.size();) {
                devices.push_back(atoi(list.c_str() + at));
                const size_t comma = list.find(',', at);
                if (comma == std::string::npos)
                    break;
                at = comma + 1;
            }
        } else {
            fprintf(stderr, "usage: %s [--host H] [--port P] [--sessions N] [--quiet] [--devices 0,1,...]\n", argv[0]);
            return 2;
        }
    }
    signal(SIGPIPE, SIG_IGN);
    lb200_group_t group = nullptr;
    if (!devices.empty()) {
        if (!make_device_current(devices[0])) {
            fprintf(stderr, "cannot make CUDA device %d current\n", devices[0]);
            return 1;
        }
        lb200_error_t err = nullptr;
        group = lb200_group_create_local(devices.data(), (int)devices.size(), &err);
        if (err) {
            fprintf(stderr, "lb200_group: %s\n", err);
            return 1;
        }
        fprintf(stderr, "lb200_index_server: building on %zu GPUs (single-process group)\n", devices.size());
    }
    int ls = socket(AF_INET, SOCK_STREAM, 0);
    if (ls < 0) {
        fprintf(stderr, "cannot create a socket: %s\n", strerror(errno));
        return 1;
    }
    int one = 1;
    setsockopt(ls, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
    sockaddr_in addr;
    memset(&addr, 0, sizeof(addr));
    addr.sin_family = AF_INET;
    addr.sin_port = htons((uint16_t)port);
    if (inet_pton(AF_INET, host, &addr.sin_addr) != 1) {
        fprintf(stderr, "bad host %s\n", host);
        return 2;
    }
    if (bind(ls, (sockaddr*)&addr, sizeof(addr)) != 0 || listen(ls, 16) != 0) {
        fprintf(stderr, "cannot listen on %s:%d: %s\n", host, port, strerror(errno));
        return 1;
    }
    if (verbose)
        fprintf(stderr, "External Indexing Server (lantern_b200, %s) started on %s:%d\n", lb200_version(), host, port);
    for (int served = 0; max_sessions < 0 || served < max_sessions; ++served) {
        int fd = accept(ls, nullptr, nullptr);
        if (fd < 0) {
            if (errno == EINTR)
                continue;
            break;
        }
        setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
        timeval tv{600, 0}; // generous: the client disables its own read timeout while we build
        setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
        Conn c{fd};
        try {
            serve(c, verbose, group);
        } catch (const std::exception& e) { // server.rs:563-573
            std::string msg = e.what();
            if (verbose)
                fprintf(stderr, "Indexing error: %s\n", msg.c_str());
            std::vector<uint8_t> out(8 + msg.size());
            uint32_t len = (uint32_t)msg.size();
            memcpy(out.data(), &kErrMsg, 4);
            memcpy(out.data() + 4, &len, 4);
            memcpy(out.data() + 8, msg.data(), msg.size());
            try {
                c.write_all(out.data(), out.size());
            } catch (...) {
            }
        }
        close(fd);
    }
    close(ls);
    if (group) {
        lb200_error_t err = nullptr;
        lb200_group_free(group, &err);
    }
    return 0;
}
