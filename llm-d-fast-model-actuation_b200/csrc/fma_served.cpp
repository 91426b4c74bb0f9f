// fma_served.cpp — a native inference-server stand-in that speaks the dual-pods controller's wire contract (B1) and moves
// REAL bytes through the engine's C-ABI: the compiled host side of the path.
//
// north_star asks for the host code in Go over cgo; this image has no Go toolchain (DESIGN.md §1), and the reference's
// code on this path IS compiled (Go): the controller's call sites (pkg/controller/dual-pods/inference-server.go:1329-1339
// POST /sleep, :1118-1137 POST /wake_up, :1595-1607 GET /is_sleeping) and its executable spec of the server side,
// cmd/test-server/main.go:56-91 — a fake vLLM that flips an atomic bool.  This program is that server with the bool replaced
// by engines: it allocates a synthetic model (segments of given tags and sizes, one engine per listed GPU = one per
// tensor-parallel rank), and then
//
//   GET  /health                          200 "OK" once the startup delay has passed, 503 before     (main.go:58-68)
//   GET  /is_sleeping                     200 {"is_sleeping":bool}                                    (main.go:69-81, pkg/api/interface.go:131-133)
//   POST /sleep[?level=1|2][&mode=...]    200, empty body, after EVERY rank has finished              (main.go:82-86; vllm api_router.py:22-33)
//   POST /wake_up[?tags=a&tags=b]         200; no tags = wake everything; safe to retry               (main.go:87-91; api_router.py:36-49)
//   GET  /stats                           200 JSON: last sleep / wake seconds and bytes per rank      (no counterpart)
//   GET  /digests                         200 JSON: K3 digest of every weights segment per rank, 409 while asleep
//
// with the executor's state machine (vllm:v1/executor/abstract.py:322-360): sleeping while asleep and waking while awake are
// no-ops, sleeping_tags = {weights, kv_cache}, waking a tag that is not asleep is refused with a warning (still 200).
// Ranks run concurrently (one thread per engine, no collective), the answer waits for the slowest.
//
// Plain POSIX sockets, HTTP/1.1 with Connection: close, one thread per connection; engine calls are serialised by a mutex
// while /is_sleeping and /health never take it (the controller polls them while a sleep is in flight).
//
//   fma_served --port 8005 --device 0 [--device 1 ...] --seg weights:1002 --seg weights:48 ... --seg kv_cache:32768
//              [--tier host|local] [--pack 1] [--incremental 1] [--seed 1234] [--startup-delay 0] [--host 127.0.0.1]
//   (sizes in MiB; port 0 picks a free port; "listening on <port>" is printed once it serves)
#include <arpa/inet.h>
#include <netinet/in.h>
#include <signal.h>
#include <sys/socket.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "../../include/fma_engine.h"

namespace {

struct SegSpec { std::string tag; size_t bytes; };
struct Rank {
    int device = 0;
    fma_engine_t* e = nullptr;
    int tag_weights = 0;
    std::vector<int> weight_segments;
};

std::vector<Rank> g_ranks;
std::mutex g_engine_mu;                       // one actuation at a time
std::atomic<bool> g_sleeping{false};          // Executor.is_sleeping
std::set<std::string> g_sleeping_tags;        // guarded by g_engine_mu
std::chrono::steady_clock::time_point g_healthy_at;
int g_tier = FMA_TIER_HOST;
std::atomic<bool> g_stop{false};
int g_listen_fd = -1;

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// run f on every rank concurrently; first error wins
template <class F>
int each_rank(F f, std::string* err) {
    std::vector<int> rc(g_ranks.size(), 0);
    std::vector<std::string> msg(g_ranks.size());
    std::vector<std::thread> th;
    for (size_t i = 0; i < g_ranks.size(); ++i)
        th.emplace_back([&, i] {
            rc[i] = f(g_ranks[i]);
            if (rc[i] != 0) msg[i] = fma_last_error();   // thread-local in the library: read it on the thread that failed
        });
    for (auto& t : th) t.join();
    for (size_t i = 0; i < rc.size(); ++i)
        if (rc[i] != 0) {
            *err = "rank " + std::to_string(i) + ": " + msg[i];
            return rc[i];
        }
    return 0;
}

// ---- the executor-level state machine (abstract.py:322-360) over the engines ----
int do_sleep(int level, std::string* err) {
    std::lock_guard<std::mutex> lk(g_engine_mu);
    if (g_sleeping.load()) {
        fprintf(stderr, "[fma_served] Executor is already sleeping.\n");
        return 0;
    }
    const double t0 = now_s();
    int rc = each_rank([&](Rank& r) {
        const uint64_t mask = level == 1 ? (1ull << r.tag_weights) : 0ull;   // Worker.sleep: level 1 offloads ("weights",), level 2 nothing
        return fma_sleep(r.e, mask, g_tier, 0);
    }, err);
    if (rc != 0) return rc;
    g_sleeping_tags = {"weights", "kv_cache"};
    g_sleeping.store(true);
    fprintf(stderr, "[fma_served] It took %.6f seconds to fall asleep.\n", now_s() - t0);
    return 0;
}

int do_wake(const std::vector<std::string>& tags, std::string* err) {
    std::lock_guard<std::mutex> lk(g_engine_mu);
    if (!g_sleeping.load()) {
        fprintf(stderr, "[fma_served] Executor is not sleeping.\n");
        return 0;
    }
    for (const std::string& t : tags)
        if (!g_sleeping_tags.count(t)) {
            fprintf(stderr, "[fma_served] Tag %s is not in sleeping tags\n", t.c_str());
            return 0;
        }
    const double t0 = now_s();
    int rc = each_rank([&](Rank& r) {
        uint64_t mask = 0;
        for (const std::string& t : tags) {
            const int id = fma_tag_intern(r.e, t.c_str());
            if (id < 0) return id;
            mask |= 1ull << id;
        }
        return fma_wake(r.e, mask, 0);   // mask 0 = every tag
    }, err);
    if (rc != 0) return rc;
    fprintf(stderr, "[fma_served] It took %.6f seconds to wake up.\n", now_s() - t0);
    if (tags.empty()) g_sleeping_tags.clear();
    for (const std::string& t : tags) g_sleeping_tags.erase(t);
    if (g_sleeping_tags.empty()) g_sleeping.store(false);
    return 0;
}

// ---- HTTP ----
void respond(int fd, int code, const char* reason, const char* ctype, const std::string& body) {
    char head[256];
    const int n = snprintf(head, sizeof(head), "HTTP/1.1 %d %s\r\nContent-Type: %s\r\nContent-Length: %zu\r\nConnection: close\r\n\r\n", code, reason, ctype,
                           body.size());
    std::string out(head, (size_t)n);
    out += body;
    size_t off = 0;
    while (off < out.size()) {
        const ssize_t w = send(fd, out.data() + off, out.size() - off, MSG_NOSIGNAL);
        if (w <= 0) break;
        off += (size_t)w;
    }
}

std::string url_decode(const std::string& s) {
    std::string o;
    for (size_t i = 0; i < s.size(); ++i) {
        if (s[i] == '%' && i + 2 < s.size() && isxdigit((unsigned char)s[i + 1]) && isxdigit((unsigned char)s[i + 2])) {
            o += (char)strtol(s.substr(i + 1, 2).c_str(), nullptr, 16);
            i += 2;
        } else if (s[i] == '+') {
            o += ' ';
        } else {
            o += s[i];
        }
    }
    return o;
}

std::vector<std::pair<std::string, std::string>> parse_query(const std::string& q) {
    std::vector<std::pair<std::string, std::string>> out;
    size_t i = 0;
    while (i < q.size()) {
        size_t j = q.find('&', i);
        if (j == std::string::npos) j = q.size();
        const std::string kv = q.substr(i, j - i);
        const size_t eq = kv.find('=');
        if (!kv.empty()) out.emplace_back(url_decode(kv.substr(0, eq)), eq == std::string::npos ? "" : url_decode(kv.substr(eq + 1)));
        i = j + 1;
    }
    return out;
}

std::string stats_json() {
    std::lock_guard<std::mutex> lk(g_engine_mu);
    std::ostringstream o;
    o << "{\"is_sleeping\":" << (g_sleeping.load() ? "true" : "false") << ",\"ranks\":[";
    for (size_t i = 0; i < g_ranks.size(); ++i) {
        fma_stats_t st;
        memset(&st, 0, sizeof(st));
        fma_stats(g_ranks[i].e, &st);
        o << (i ? "," : "") << "{\"device\":" << g_ranks[i].device << ",\"sleep_seconds\":" << st.sleep_seconds << ",\"wake_seconds\":" << st.wake_seconds
          << ",\"sleep_bytes_offloaded\":" << st.sleep_bytes_offloaded << ",\"wake_bytes_restored\":" << st.wake_bytes_restored
          << ",\"image_store_bytes\":" << st.image_store_bytes << ",\"sleep_bytes_copied\":" << st.sleep_bytes_copied << ",\"image_packed\":" << st.image_packed << ",\"hbm_mapped_bytes\":" << st.hbm_mapped_bytes << ",\"resident_bytes\":" << st.resident_bytes << "}";
    }
    o << "]}";
    return o.str();
}

int digests_json(std::string* out) {
    std::lock_guard<std::mutex> lk(g_engine_mu);
    if (g_sleeping.load()) return 409;
    std::ostringstream o;
    o << "[";
    for (size_t i = 0; i < g_ranks.size(); ++i) {
        o << (i ? "," : "") << "[";
        for (size_t k = 0; k < g_ranks[i].weight_segments.size(); ++k) {
            uint64_t d = 0;
            if (fma_digest_segment(g_ranks[i].e, g_ranks[i].weight_segments[k], &d) != 0) return 500;
            o << (k ? "," : "") << "\"" << std::hex << d << std::dec << "\"";
        }
        o << "]";
    }
    o << "]";
    *out = o.str();
    return 200;
}

void handle(int fd) {
    std::string req;
    char buf[4096];
    while (req.find("\r\n\r\n") == std::string::npos && req.size() < (64u << 10)) {
        const ssize_t n = recv(fd, buf, sizeof(buf), 0);
        if (n <= 0) break;
        req.append(buf, (size_t)n);
    }
    const size_t eol = req.find("\r\n");
    if (eol == std::string::npos) {
        close(fd);
        return;
    }
    std::istringstream first(req.substr(0, eol));
    std::string method, target, version;
    first >> method >> target >> version;
    const size_t qm = target.find('?');
    const std::string path = target.substr(0, qm), query = qm == std::string::npos ? "" : target.substr(qm + 1);
    // a request body (the controller sends none) is drained so the peer never sees a reset
    size_t content_length = 0;
    {
        std::string lower = req;
        for (char& c : lower) c = (char)tolower((unsigned char)c);
        const size_t p = lower.find("content-length:");
        if (p != std::string::npos) content_length = (size_t)strtoul(lower.c_str() + p + 15, nullptr, 10);
    }
    size_t have = req.size() - (req.find("\r\n\r\n") + 4);
    while (have < content_length && have < (1u << 20)) {
        const ssize_t n = recv(fd, buf, sizeof(buf), 0);
        if (n <= 0) break;
        have += (size_t)n;
    }

    std::string err;
    if (path == "/health") {
        if (method != "GET") respond(fd, 405, "Method Not Allowed", "text/plain", "Method Not Allowed\n");
        else if (std::chrono::steady_clock::now() >= g_healthy_at) respond(fd, 200, "OK", "text/plain", "OK\n");
        else respond(fd, 503, "Service Unavailable", "text/plain", "Service Unavailable\n");
    } else if (path == "/is_sleeping") {
        if (method != "GET") respond(fd, 405, "Method Not Allowed", "text/plain", "Method Not Allowed\n");
        else respond(fd, 200, "OK", "application/json", std::string("{\"is_sleeping\":") + (g_sleeping.load() ? "true" : "false") + "}");
    } else if (path == "/sleep") {
        if (method != "POST") {
            respond(fd, 405, "Method Not Allowed", "text/plain", "Method Not Allowed\n");
        } else {
            int level = 1;
            bool bad = false;
            for (auto& kv : parse_query(query))
                if (kv.first == "level") {
                    char* end = nullptr;
                    level = (int)strtol(kv.second.c_str(), &end, 10);
                    bad = kv.second.empty() || *end != 0;
                }
            if (bad) respond(fd, 422, "Unprocessable Entity", "text/plain", "level must be an integer\n");
            else if (do_sleep(level, &err) == 0) respond(fd, 200, "OK", "text/plain", "");   // exactly 200, empty body (inference-server.go:1335)
            else respond(fd, 500, "Internal Server Error", "text/plain", err + "\n");
        }
    } else if (path == "/wake_up") {
        if (method != "POST") {
            respond(fd, 405, "Method Not Allowed", "text/plain", "Method Not Allowed\n");
        } else {
            std::vector<std::string> tags;
            for (auto& kv : parse_query(query))
                if (kv.first == "tags") tags.push_back(kv.second);
            if (do_wake(tags, &err) == 0) respond(fd, 200, "OK", "text/plain", "");
            else respond(fd, 500, "Internal Server Error", "text/plain", err + "\n");
        }
    } else if (path == "/stats" && method == "GET") {
        respond(fd, 200, "OK", "application/json", stats_json());
    } else if (path == "/digests" && method == "GET") {
        std::string body;
        const int code = digests_json(&body);
        if (code == 200) respond(fd, 200, "OK", "application/json", body);
        else if (code == 409) respond(fd, 409, "Conflict", "text/plain", "asleep: weights are not mapped\n");
        else respond(fd, 500, "Internal Server Error", "text/plain", std::string(fma_last_error()) + "\n");
    } else {
        respond(fd, 404, "Not Found", "text/plain", "Not Found\n");
    }
    shutdown(fd, SHUT_RDWR);
    close(fd);
}

void on_signal(int) {
    g_stop.store(true);
    if (g_listen_fd >= 0) shutdown(g_listen_fd, SHUT_RDWR);
}

int die(const char* what) {
    fprintf(stderr, "fma_served: %s: %s\n", what, fma_last_error());
    return 1;
}

}  // namespace

int main(int argc, char** argv) {
    int port = 8005, pack = 0, incremental = 0;
    std::string host = "127.0.0.1";
    std::vector<int> devices;
    std::vector<SegSpec> segs;
    uint64_t seed = 1234;
    double startup_delay = 0;
    for (int i = 1; i < argc; ++i) {
        const std::string a = argv[i];
        auto val = [&]() -> const char* { return i + 1 < argc ? argv[++i] : ""; };
        if (a == "--port") port = atoi(val());
        else if (a == "--host") host = val();
        else if (a == "--device") devices.push_back(atoi(val()));
        else if (a == "--seed") seed = strtoull(val(), nullptr, 0);
        else if (a == "--pack") pack = atoi(val());
        else if (a == "--incremental") incremental = atoi(val());
        else if (a == "--startup-delay") startup_delay = atof(val());
        else if (a == "--tier") {
            const std::string t = val();
            g_tier = t == "local" ? FMA_TIER_LOCAL : FMA_TIER_HOST;
        } else if (a == "--seg") {
            const std::string s = val();
            const size_t c = s.find(':');
            if (c == std::string::npos || atol(s.c_str() + c + 1) <= 0) { fprintf(stderr, "fma_served: --seg wants tag:MiB\n"); return 2; }
            segs.push_back(SegSpec{s.substr(0, c), (size_t)atol(s.c_str() + c + 1) << 20});
        } else {
            fprintf(stderr, "fma_served: unknown argument %s\n", a.c_str());
            return 2;
        }
    }
    if (devices.empty()) devices.push_back(0);
    if (segs.empty()) segs = {{"weights", (size_t)48 << 20}, {"weights", (size_t)32 << 20}, {"weights", (size_t)2 << 20}, {"kv_cache", (size_t)64 << 20}};

    for (size_t r = 0; r < devices.size(); ++r) {
        Rank rk;
        rk.device = devices[r];
        fma_config_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.abi_version = FMA_ABI_VERSION;
        cfg.numa_bind = -1;
        cfg.pack = pack;
        if (fma_engine_create(rk.device, &cfg, &rk.e) != 0) return die("fma_engine_create");
        if (incremental && fma_set_option(rk.e, "incremental", 1) != 0) return die("fma_set_option");
        rk.tag_weights = fma_tag_intern(rk.e, "weights");
        uint64_t first_word = 0;
        for (const SegSpec& s : segs) {
            const int tag = fma_tag_intern(rk.e, s.tag.c_str());
            void* p = nullptr;
            if (tag < 0 || fma_alloc(rk.e, s.bytes, tag, &p) != 0) return die("fma_alloc");
            const int idx = fma_segment_find(rk.e, p);
            if (s.tag == "weights") {
                if (fma_fill_segment(rk.e, idx, seed + r, first_word) != 0) return die("fma_fill_segment");   // K0: seed 1234 + rank
                first_word += s.bytes / 8;
                rk.weight_segments.push_back(idx);
            }
        }
        g_ranks.push_back(rk);
    }
    g_healthy_at = std::chrono::steady_clock::now() + std::chrono::milliseconds((long)(startup_delay * 1e3));

    g_listen_fd = socket(AF_INET, SOCK_STREAM, 0);
    int one = 1;
    setsockopt(g_listen_fd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
    sockaddr_in addr;
    memset(&addr, 0, sizeof(addr));
    addr.sin_family = AF_INET;
    addr.sin_port = htons((uint16_t)port);
    if (inet_pton(AF_INET, host.c_str(), &addr.sin_addr) != 1) { fprintf(stderr, "fma_served: bad --host %s\n", host.c_str()); return 2; }
    if (bind(g_listen_fd, (sockaddr*)&addr, sizeof(addr)) != 0 || listen(g_listen_fd, 64) != 0) { perror("fma_served: bind/listen"); return 1; }
    socklen_t alen = sizeof(addr);
    getsockname(g_listen_fd, (sockaddr*)&addr, &alen);
    struct sigaction sa;
    memset(&sa, 0, sizeof(sa));
    sa.sa_handler = on_signal;
    sigaction(SIGTERM, &sa, nullptr);
    sigaction(SIGINT, &sa, nullptr);
    printf("listening on %d\n", (int)ntohs(addr.sin_port));
    fflush(stdout);

    std::atomic<int> inflight{0};
    while (!g_stop.load()) {
        const int fd = accept(g_listen_fd, nullptr, nullptr);
        if (fd < 0) {
            if (g_stop.load()) break;
            continue;
        }
        ++inflight;
        std::thread([fd, &inflight] {
            handle(fd);
            --inflight;
        }).detach();
    }
    for (int i = 0; i < 3000 && inflight.load() > 0; ++i) std::this_thread::sleep_for(std::chrono::milliseconds(10));   // let answers finish
    close(g_listen_fd);
    {
        std::lock_guard<std::mutex> lk(g_engine_mu);
        for (Rank& r : g_ranks) fma_engine_destroy(r.e);
    }
    return 0;
}
