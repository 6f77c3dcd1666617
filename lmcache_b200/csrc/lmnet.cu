// lmnet.cu -- the lm:// wire protocol in C++: client (what LMCRemoteBackend talks through) and server.
// Host-only code (no device work); it lives in libb200kv.so so that the engine's remote tier has one native library.
//
// Replaces (reference paths relative to the LMCache v0.1.2 tree):
//   lmcache/storage_backend/connector/lm_connector.py:15-84   blocking Python socket client, recv loop into bytearrays
//   lmcache/server/__main__.py:29-104                         Python thread-per-client server; EXIST = `key in list_keys()`
//   lmcache/protocol.py:4-70                                   the headers below, byte for byte
//
// Wire format (little-endian, as Python's struct "ii150s" / "ii" produce on x86 / aarch64):
//   client -> server  int32 command | int32 payload length | char key[150] (space padded)      158 bytes [+ payload]
//   server -> client  int32 status  | int32 payload length                                        8 bytes [+ payload]
//   PUT has no reply (server/__main__.py:46-48); GET miss = FAIL with length 0; EXIST = SUCCESS / FAIL with length 0;
//   LIST = SUCCESS + keys joined by '\n'.
//
// Ranged reads (this project's servers only; the reference server ignores an unknown command -- no reply, and the body
// is read as the next header -- so a client that sent one would wait forever: a client sends them only after EXIST on
// kRangesProbe has answered SUCCESS -- the reference answers FAIL):
//   OPEN  (5)  key, length = prefix bytes wanted -> SUCCESS, 16 + n: u32 handle | u32 0 | u64 value size | the first
//              n = min(prefix, size) bytes; a miss, or a connection already holding kMaxHandles, is FAIL with length 0
//   READ  (6)  length = 24 m, body m x {u32 handle | u32 0 | u64 offset | u64 nbytes} -> SUCCESS, sum nbytes, then the
//              ranges in request order; an unknown handle or a range out of bounds is FAIL with length 0 (the connection
//              stays in step)
//   CLOSE (7)  length = 4 m, body m x u32 handle -> SUCCESS, 0 (unknown handles are ignored)
// A handle holds the value as it was at OPEN (the stored Blob is shared, never mutated: a PUT replaces it), so every
// byte read through it comes from one stored value.  A connection's handles are dropped when it closes.
//
// What is different from the reference, on purpose: payloads go from / into caller memory with one send / recv loop
// (pinned slabs and Python bytes alike: no intermediate copies), the server keeps values in a hash map behind a
// reader-writer lock (EXIST and GET are O(1) and concurrent), and a connection serialises whole request / response
// exchanges (the reference locks sends only, its TODO:1).
#include <arpa/inet.h>
#include <netdb.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/socket.h>
#include <sys/types.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cerrno>
#include <cstring>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace b200kv {
namespace {

constexpr int kKeyLen = 150;
constexpr int kClientHdr = 8 + kKeyLen;     // struct "ii150s"
constexpr int kServerHdr = 8;               // struct "ii"
enum { kPut = 1, kGet = 2, kExist = 3, kList = 4, kOpen = 5, kRead = 6, kClose = 7, kSuccess = 200, kFail = 400 };
constexpr const char* kRangesProbe = "b200kv-ranges-v1";    // EXIST on it: SUCCESS from a server that has OPEN / READ / CLOSE
constexpr size_t kMaxHandles = 4096;                         // open handles per connection
constexpr int64_t kMaxReply = INT32_MAX;                    // a reply's length is an int32
constexpr size_t kIoChunk = 1u << 20;      // bytes per send / recv call

bool send_all(int fd, const void* p, size_t n) {
    const char* c = static_cast<const char*>(p);
    while (n) {
        const ssize_t k = ::send(fd, c, n < kIoChunk ? n : kIoChunk, MSG_NOSIGNAL);
        if (k < 0) {
            if (errno == EINTR) continue;
            return false;
        }
        c += k;
        n -= (size_t)k;
    }
    return true;
}

bool recv_all(int fd, void* p, size_t n) {
    char* c = static_cast<char*>(p);
    while (n) {
        const ssize_t k = ::recv(fd, c, n < kIoChunk ? n : kIoChunk, 0);
        if (k == 0) return false;
        if (k < 0) {
            if (errno == EINTR) continue;
            return false;
        }
        c += k;
        n -= (size_t)k;
    }
    return true;
}

void tune(int) {}     // kernel defaults (as the reference's Python sockets): autotuned buffers, Nagle on -- measured fastest

// An OPEN or READ reply is corked while its pieces are sent and uncorked at the end, which pushes its last partial
// segment at once: under Nagle alone that tail would wait for the peer's (delayed) ACK of the reply's earlier segments,
// on every round trip of a layer-by-layer fetch.
struct Corked {
    int fd;
    explicit Corked(int f) : fd(f) { set(1); }
    ~Corked() { set(0); }
    void set(int on) { setsockopt(fd, IPPROTO_TCP, TCP_CORK, &on, sizeof on); }
};

void pack_client(char* hdr, int32_t cmd, int32_t len, const char* key) {
    memcpy(hdr, &cmd, 4);
    memcpy(hdr + 4, &len, 4);
    memset(hdr + 8, ' ', kKeyLen);
    memcpy(hdr + 8, key, strlen(key));
}

// Python: key.decode().strip()
std::string unpack_key(const char* raw) {
    int a = 0, b = kKeyLen;
    auto ws = [](char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\f' || c == '\v' || c == 0; };
    while (a < b && ws(raw[a])) ++a;
    while (b > a && ws(raw[b - 1])) --b;
    return std::string(raw + a, raw + b);
}

struct Blob {
    std::unique_ptr<char[]> data;
    int32_t len = 0;
};

struct Server {
    int lfd = -1;
    int port = 0;
    std::atomic<bool> stop{false};
    std::thread acceptor;
    std::mutex conn_mu;
    std::vector<int> conns;                 // open client sockets (a worker removes its own on exit)
    std::atomic<int> active{0};             // running worker threads (detached; stop() waits for zero)
    std::shared_mutex mu;
    std::unordered_map<std::string, std::shared_ptr<Blob>> store;
    std::atomic<int64_t> handles_open{0};   // OPEN handles of every connection (b200kv_lm_server_num_handles)

    std::shared_ptr<Blob> find(const std::string& key) {
        std::shared_lock<std::shared_mutex> lk(mu);
        auto it = store.find(key);
        return it == store.end() ? nullptr : it->second;
    }

    void serve(int fd) {
        tune(fd);
        std::unordered_map<uint32_t, std::shared_ptr<Blob>> handles;     // this connection's snapshots
        uint32_t next_handle = 1;
        std::vector<char> body;
        char hdr[kClientHdr];
        while (!stop.load(std::memory_order_relaxed) && recv_all(fd, hdr, kClientHdr)) {
            int32_t cmd, len;
            memcpy(&cmd, hdr, 4);
            memcpy(&len, hdr + 4, 4);
            const std::string key = unpack_key(hdr + 8);
            char rep[kServerHdr];
            auto reply = [&](int32_t code, int32_t n) {
                memcpy(rep, &code, 4);
                memcpy(rep + 4, &n, 4);
                return send_all(fd, rep, kServerHdr);
            };
            if (cmd == kPut) {
                if (len < 0) break;
                auto blob = std::make_shared<Blob>();
                blob->data.reset(new char[len > 0 ? len : 1]);
                blob->len = len;
                if (!recv_all(fd, blob->data.get(), (size_t)len)) break;
                std::unique_lock<std::shared_mutex> lk(mu);
                store[key] = std::move(blob);
            } else if (cmd == kGet) {
                std::shared_ptr<Blob> blob;
                {
                    std::shared_lock<std::shared_mutex> lk(mu);
                    auto it = store.find(key);
                    if (it != store.end()) blob = it->second;
                }
                if (!blob) {
                    if (!reply(kFail, 0)) break;
                } else {
                    if (!reply(kSuccess, blob->len) || !send_all(fd, blob->data.get(), (size_t)blob->len)) break;
                }
            } else if (cmd == kExist) {
                bool ok = key == kRangesProbe;
                if (!ok) {
                    std::shared_lock<std::shared_mutex> lk(mu);
                    ok = store.find(key) != store.end();
                }
                if (!reply(ok ? kSuccess : kFail, 0)) break;
            } else if (cmd == kOpen) {
                std::shared_ptr<Blob> blob = len >= 0 && handles.size() < kMaxHandles ? find(key) : nullptr;
                if (!blob) {
                    if (!reply(kFail, 0)) break;
                    continue;
                }
                while (handles.count(next_handle) || next_handle == 0) ++next_handle;
                const uint32_t h = next_handle++;
                handles[h] = blob;
                handles_open.fetch_add(1);
                const int32_t n = len < blob->len ? len : blob->len;
                char meta[16];
                const uint32_t zero = 0;
                const uint64_t size = (uint64_t)blob->len;
                memcpy(meta, &h, 4);
                memcpy(meta + 4, &zero, 4);
                memcpy(meta + 8, &size, 8);
                Corked cork(fd);
                if (!reply(kSuccess, 16 + n) || !send_all(fd, meta, 16) || !send_all(fd, blob->data.get(), (size_t)n)) break;
            } else if (cmd == kRead || cmd == kClose) {
                const int unit = cmd == kRead ? 24 : 4;
                if (len < 0) break;
                body.resize((size_t)len);
                if (!recv_all(fd, body.data(), (size_t)len)) break;
                const size_t m = (size_t)len / unit;
                if (cmd == kClose) {
                    for (size_t i = 0; i < m; ++i) {
                        uint32_t h;
                        memcpy(&h, body.data() + 4 * i, 4);
                        if (handles.erase(h)) handles_open.fetch_sub(1);
                    }
                    if (!reply(kSuccess, 0)) break;
                    continue;
                }
                // every entry is checked before a byte is sent: a refused READ sends nothing but its header
                std::vector<const char*> src(m);
                int64_t total = 0;
                bool ok = len % unit == 0;
                for (size_t i = 0; ok && i < m; ++i) {
                    uint32_t h;
                    uint64_t off, nb;
                    memcpy(&h, body.data() + 24 * i, 4);
                    memcpy(&off, body.data() + 24 * i + 8, 8);
                    memcpy(&nb, body.data() + 24 * i + 16, 8);
                    auto it = handles.find(h);
                    ok = it != handles.end() && off <= (uint64_t)it->second->len &&
                         nb <= (uint64_t)it->second->len - off && total + (int64_t)nb <= kMaxReply;
                    if (ok) {
                        src[i] = it->second->data.get() + off;
                        total += (int64_t)nb;
                    }
                }
                if (!ok) {
                    if (!reply(kFail, 0)) break;
                    continue;
                }
                Corked cork(fd);
                if (!reply(kSuccess, (int32_t)total)) break;
                bool sent = true;
                for (size_t i = 0; sent && i < m; ++i) {
                    uint64_t nb;
                    memcpy(&nb, body.data() + 24 * i + 16, 8);
                    sent = send_all(fd, src[i], (size_t)nb);
                }
                if (!sent) break;
            } else if (cmd == kList) {
                std::string all;
                {
                    std::shared_lock<std::shared_mutex> lk(mu);
                    for (const auto& kv : store) {
                        if (!all.empty()) all.push_back('\n');
                        all += kv.first;
                    }
                }
                if (!reply(kSuccess, (int32_t)all.size()) || !send_all(fd, all.data(), all.size())) break;
            } else {
                break;      // unknown command: drop the connection, as the reference does by raising
            }
        }
        handles_open.fetch_sub((int64_t)handles.size());
        {
            std::lock_guard<std::mutex> lk(conn_mu);
            for (size_t i = 0; i < conns.size(); ++i)
                if (conns[i] == fd) {
                    conns[i] = conns.back();
                    conns.pop_back();
                    break;
                }
            ::close(fd);
        }
        active.fetch_sub(1);
    }

    void accept_loop() {
        for (;;) {
            const int fd = ::accept(lfd, nullptr, nullptr);
            if (fd < 0) {
                if (errno == EINTR) continue;
                break;                                  // listening socket closed: shutting down
            }
            if (stop.load()) {
                ::close(fd);
                break;
            }
            {
                std::lock_guard<std::mutex> lk(conn_mu);
                conns.push_back(fd);
            }
            active.fetch_add(1);
            std::thread([this, fd] { serve(fd); }).detach();
        }
    }
};

struct Conn {
    int fd = -1;
    std::mutex mu;          // one request / response exchange at a time
    int64_t pending = 0;    // payload bytes of a begun GET / LIST not yet read
};

int resolve(const char* host, int port, sockaddr_in* out) {
    memset(out, 0, sizeof *out);
    out->sin_family = AF_INET;
    out->sin_port = htons((uint16_t)port);
    if (host == nullptr || host[0] == 0 || strcmp(host, "0.0.0.0") == 0) {
        out->sin_addr.s_addr = htonl(INADDR_ANY);
        return 0;
    }
    if (strcmp(host, "localhost") == 0) host = "127.0.0.1";
    if (inet_pton(AF_INET, host, &out->sin_addr) == 1) return 0;
    addrinfo hints{}, *res = nullptr;
    hints.ai_family = AF_INET;
    hints.ai_socktype = SOCK_STREAM;
    if (getaddrinfo(host, nullptr, &hints, &res) != 0 || res == nullptr) return -1;
    out->sin_addr = reinterpret_cast<sockaddr_in*>(res->ai_addr)->sin_addr;
    freeaddrinfo(res);
    return 0;
}

}  // namespace
}  // namespace b200kv

using namespace b200kv;

extern "C" {

int b200kv_lm_server_start(const char* host, int32_t port, void** server) {
    B2_REQUIRE(server != nullptr && port >= 0 && port < 65536, "bad server arguments");
    sockaddr_in addr;
    B2_REQUIRE(resolve(host, port, &addr) == 0, "cannot resolve host");
    const int fd = ::socket(AF_INET, SOCK_STREAM, 0);
    B2_REQUIRE(fd >= 0, "socket() failed");
    int one = 1;
    setsockopt(fd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof one);
    if (::bind(fd, reinterpret_cast<sockaddr*>(&addr), sizeof addr) != 0 || ::listen(fd, 128) != 0) {
        const std::string why = strerror(errno);
        ::close(fd);
        set_error("bind/listen failed: " + why);
        return -1;
    }
    socklen_t sl = sizeof addr;
    getsockname(fd, reinterpret_cast<sockaddr*>(&addr), &sl);
    Server* s = new Server();
    s->lfd = fd;
    s->port = ntohs(addr.sin_port);
    s->acceptor = std::thread([s] { s->accept_loop(); });
    *server = s;
    return 0;
}

int32_t b200kv_lm_server_port(void* server) { return server ? static_cast<Server*>(server)->port : -1; }

int64_t b200kv_lm_server_num_keys(void* server) {
    if (!server) return -1;
    Server* s = static_cast<Server*>(server);
    std::shared_lock<std::shared_mutex> lk(s->mu);
    return (int64_t)s->store.size();
}

int64_t b200kv_lm_server_num_handles(void* server) {
    return server ? static_cast<Server*>(server)->handles_open.load() : -1;
}

int b200kv_lm_server_stop(void* server) {
    B2_REQUIRE(server != nullptr, "server is NULL");
    Server* s = static_cast<Server*>(server);
    s->stop.store(true);
    ::shutdown(s->lfd, SHUT_RDWR);
    ::close(s->lfd);
    if (s->acceptor.joinable()) s->acceptor.join();
    {
        std::lock_guard<std::mutex> lk(s->conn_mu);
        for (int fd : s->conns) ::shutdown(fd, SHUT_RDWR);       // wakes workers blocked in recv
    }
    while (s->active.load() != 0) std::this_thread::sleep_for(std::chrono::milliseconds(1));
    delete s;
    return 0;
}

int b200kv_lm_connect(const char* host, int32_t port, void** conn) {
    B2_REQUIRE(conn != nullptr && port > 0 && port < 65536, "bad connect arguments");
    sockaddr_in addr;
    B2_REQUIRE(resolve(host, port, &addr) == 0, "cannot resolve host");
    const int fd = ::socket(AF_INET, SOCK_STREAM, 0);
    B2_REQUIRE(fd >= 0, "socket() failed");
    if (::connect(fd, reinterpret_cast<sockaddr*>(&addr), sizeof addr) != 0) {
        const std::string why = strerror(errno);
        ::close(fd);
        set_error("connect failed: " + why);
        return -1;
    }
    tune(fd);
    Conn* c = new Conn();
    c->fd = fd;
    *conn = c;
    return 0;
}

int b200kv_lm_close(void* conn) {
    if (!conn) return 0;
    Conn* c = static_cast<Conn*>(conn);
    ::shutdown(c->fd, SHUT_RDWR);
    ::close(c->fd);
    delete c;
    return 0;
}

// connection.set(key, obj): header + payload straight from caller memory (Python bytes, a pinned slab, ...)
int b200kv_lm_put(void* conn, const char* key, const void* data, int64_t len) {
    B2_REQUIRE(conn && key && strlen(key) <= (size_t)kKeyLen, "bad key / connection");
    B2_REQUIRE(len >= 0 && len <= INT32_MAX && (data != nullptr || len == 0), "payload must be 0 .. 2^31-1 bytes");
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    B2_REQUIRE(c->pending == 0, "a GET payload is still pending on this connection");
    char hdr[kClientHdr];
    pack_client(hdr, kPut, (int32_t)len, key);
    if (!send_all(c->fd, hdr, kClientHdr) || !send_all(c->fd, data, (size_t)len)) {
        set_error("lm:// send failed");
        return -1;
    }
    return 0;
}

// 1 = present, 0 = absent, < 0 = error
int b200kv_lm_exists(void* conn, const char* key) {
    B2_REQUIRE(conn && key && strlen(key) <= (size_t)kKeyLen, "bad key / connection");
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    B2_REQUIRE(c->pending == 0, "a GET payload is still pending on this connection");
    char hdr[kClientHdr], rep[kServerHdr];
    pack_client(hdr, kExist, 0, key);
    if (!send_all(c->fd, hdr, kClientHdr) || !recv_all(c->fd, rep, kServerHdr)) {
        set_error("lm:// exchange failed");
        return -1;
    }
    int32_t code;
    memcpy(&code, rep, 4);
    return code == kSuccess ? 1 : 0;
}

// GET / LIST are two calls because the caller allocates the destination once the length is known:
//   n = b200kv_lm_get_begin(conn, key)   -> payload length (>= 0), -1 = miss, < -1 = error; the connection is held
//   b200kv_lm_read(conn, dst, n)         -> payload into caller memory (n may be 0)
static int64_t begin(void* conn, int32_t cmd, const char* key) {
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->pending != 0) {
        set_error("invalid argument: a GET payload is still pending on this connection");
        return -2;
    }
    char hdr[kClientHdr], rep[kServerHdr];
    pack_client(hdr, cmd, 0, key);
    if (!send_all(c->fd, hdr, kClientHdr) || !recv_all(c->fd, rep, kServerHdr)) {
        set_error("lm:// exchange failed");
        return -3;
    }
    int32_t code, len;
    memcpy(&code, rep, 4);
    memcpy(&len, rep + 4, 4);
    if (code != kSuccess) return -1;
    c->pending = len;
    return len;
}

int64_t b200kv_lm_get_begin(void* conn, const char* key) {
    if (!conn || !key || strlen(key) > (size_t)kKeyLen) {
        set_error("invalid argument: bad key / connection");
        return -2;
    }
    return begin(conn, kGet, key);
}

int64_t b200kv_lm_list_begin(void* conn) {
    if (!conn) {
        set_error("invalid argument: connection is NULL");
        return -2;
    }
    return begin(conn, kList, "");
}

int b200kv_lm_read(void* conn, void* dst, int64_t len) {
    B2_REQUIRE(conn != nullptr, "connection is NULL");
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    B2_REQUIRE(len == c->pending && (dst != nullptr || len == 0), "length does not match the pending payload");
    c->pending = 0;
    if (!recv_all(c->fd, dst, (size_t)len)) {
        set_error("lm:// receive failed");
        return -1;
    }
    return 0;
}

// OPEN: n = b200kv_lm_open_begin(conn, key, prefix, &handle, &size) -> prefix bytes pending (min(prefix, size)),
// -1 = miss (or the server's handle cap), < -1 = error; the prefix then comes through b200kv_lm_read(conn, dst, n)
int64_t b200kv_lm_open_begin(void* conn, const char* key, int64_t prefix, uint32_t* handle, int64_t* size) {
    if (!conn || !key || strlen(key) > (size_t)kKeyLen || prefix < 0 || prefix > INT32_MAX - 16 || !handle || !size) {
        set_error("invalid argument: bad key / connection / prefix");
        return -2;
    }
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->pending != 0) {
        set_error("invalid argument: a GET payload is still pending on this connection");
        return -2;
    }
    char hdr[kClientHdr], rep[kServerHdr], meta[16];
    pack_client(hdr, kOpen, (int32_t)prefix, key);
    if (!send_all(c->fd, hdr, kClientHdr) || !recv_all(c->fd, rep, kServerHdr)) {
        set_error("lm:// exchange failed");
        return -3;
    }
    int32_t code, len;
    memcpy(&code, rep, 4);
    memcpy(&len, rep + 4, 4);
    if (code != kSuccess) return -1;
    if (len < 16 || !recv_all(c->fd, meta, 16)) {
        set_error("lm:// OPEN reply malformed or cut short");
        return -3;
    }
    memcpy(handle, meta, 4);
    memcpy(size, meta + 8, 8);
    c->pending = len - 16;
    return len - 16;
}

// READ: the m ranges (handles[i], offsets[i], sizes[i]) straight into dst[i] (caller memory, e.g. slab blocks).
// 0 = done, 1 = refused by the server (unknown handle / out of bounds: nothing was written), < 0 = error.
int b200kv_lm_read_ranges(void* conn, int32_t m, const uint32_t* handles, const uint64_t* offsets, const uint64_t* sizes,
                          void* const* dst) {
    B2_REQUIRE(conn != nullptr && m >= 0 && (int64_t)m * 24 <= INT32_MAX &&
               (m == 0 || (handles && offsets && sizes && dst)), "bad READ arguments");
    int64_t total = 0;
    for (int32_t i = 0; i < m; ++i) {
        B2_REQUIRE(sizes[i] <= (uint64_t)kMaxReply && (sizes[i] == 0 || dst[i] != nullptr), "bad READ range");
        total += (int64_t)sizes[i];
    }
    B2_REQUIRE(total <= kMaxReply, "a READ reply must stay below 2^31 bytes: split the request");
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    B2_REQUIRE(c->pending == 0, "a GET payload is still pending on this connection");
    std::vector<char> req(kClientHdr + 24 * (size_t)m);
    pack_client(req.data(), kRead, 24 * m, "");
    for (int32_t i = 0; i < m; ++i) {
        char* e = req.data() + kClientHdr + 24 * (size_t)i;
        const uint32_t zero = 0;
        memcpy(e, &handles[i], 4);
        memcpy(e + 4, &zero, 4);
        memcpy(e + 8, &offsets[i], 8);
        memcpy(e + 16, &sizes[i], 8);
    }
    char rep[kServerHdr];
    if (!send_all(c->fd, req.data(), req.size()) || !recv_all(c->fd, rep, kServerHdr)) {
        set_error("lm:// exchange failed");
        return -3;
    }
    int32_t code, len;
    memcpy(&code, rep, 4);
    memcpy(&len, rep + 4, 4);
    if (code != kSuccess) return 1;
    if (len != total) {
        set_error("lm:// READ reply length does not match the request");
        return -3;
    }
    for (int32_t i = 0; i < m; ++i)
        if (!recv_all(c->fd, dst[i], (size_t)sizes[i])) {
            set_error("lm:// receive failed");
            return -3;
        }
    return 0;
}

int b200kv_lm_close_handles(void* conn, int32_t m, const uint32_t* handles) {
    B2_REQUIRE(conn != nullptr && m >= 0 && (int64_t)m * 4 <= INT32_MAX && (m == 0 || handles), "bad CLOSE arguments");
    Conn* c = static_cast<Conn*>(conn);
    std::lock_guard<std::mutex> lk(c->mu);
    B2_REQUIRE(c->pending == 0, "a GET payload is still pending on this connection");
    std::vector<char> req(kClientHdr + 4 * (size_t)m);
    pack_client(req.data(), kClose, 4 * m, "");
    if (m) memcpy(req.data() + kClientHdr, handles, 4 * (size_t)m);
    char rep[kServerHdr];
    if (!send_all(c->fd, req.data(), req.size()) || !recv_all(c->fd, rep, kServerHdr)) {
        set_error("lm:// exchange failed");
        return -3;
    }
    return 0;
}

}  // extern "C"
