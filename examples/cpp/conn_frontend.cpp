// The routes of examples/cpp/conn_routes.cpp (the reference's TestGofr_ServerRoutes, pkg/gofr/gofr_test.go:40-105, plus the
// handlers of examples/http-server/main.go:29-43) served the way net/http serves them: one thread per group of connections,
// each connection's requests pipelined into one byte stream and delivered as reads cut at arbitrary byte positions.  Each
// read goes through gofr::ConnFrontend (the threads' reads are batched together on the GPU) and the thread keeps the tail
// on GOFR_HTTP_CONN_MORE.  The handlers the GPU runs itself are registered with their fused kinds (a static string,
// c.Param formatting, a static error, nil, a panic); the two closures (two path parameters, the body echoed) are GOFR_H_HOST
// routes, so their requests come back as holes, and the thread answers each through a gofr::App that holds those closures,
// under the trace id the front-end returned for it.  Exits non-zero when a response is not what the reference's test
// expects, when a response's X-Correlation-Id is not the trace id returned for it, when a connection ends in another state
// than its stream, or when a trace id repeats.
//   g++ -std=c++17 -Iinclude examples/cpp/conn_frontend.cpp gofr_b200/libgofr_b200.so -lpthread -o conn_frontend
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <random>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "gofr_b200.hpp"

static std::string head_of(const std::string& wire) { return wire.substr(0, wire.find("\r\n\r\n")); }
static std::string body_of(const std::string& wire) {
    const size_t p = wire.find("\r\n\r\n");
    return p == std::string::npos ? wire : wire.substr(p + 4);
}
static std::string hex(const std::array<uint8_t, 16>& id) {
    static const char* d = "0123456789abcdef";
    std::string s;
    for (uint8_t b : id) { s += d[b >> 4]; s += d[b & 15]; }
    return s;
}

int main(int argc, char** argv) {
    const int threads = argc > 1 ? atoi(argv[1]) : 8, conns_per_thread = argc > 2 ? atoi(argv[2]) : 6;
    // the closures, run on the host for the holes
    gofr::App g;
    g.GET("/users/{id:[0-9]+}/posts/{slug}", [](gofr::Context& c) -> gofr::Result {
        return "user " + c.PathParam("id") + " post " + c.PathParam("slug");
    });
    g.POST("/echo", [](gofr::Context& c) -> gofr::Result { return c.Body(); });
    g.Run(0);
    // the table the front-end serves: every route in the reference's registration order
    struct Route { uint32_t method; const char* pattern; uint32_t kind; const char *s0, *s1, *s2, *s3; };
    const Route routes[] = {
        {GOFR_M_GET, "/hello", GOFR_H_STATIC_STRING, "Hello World!", "", "", ""},
        {GOFR_M_GET, "/hello2", GOFR_H_STATIC_STRING, "Hello World!", "", "", ""},
        {GOFR_M_PUT, "/hello", GOFR_H_STATIC_STRING, "Hello World!", "", "", ""},
        {GOFR_M_POST, "/hello", GOFR_H_STATIC_STRING, "Hello World!", "", "", ""},
        {GOFR_M_GET, "/params", GOFR_H_PARAM_FORMAT, "name", "", "Hello ", "!"},
        {GOFR_M_DELETE, "/delete", GOFR_H_STATIC_STRING, "Success", "", "", ""},
        {GOFR_M_GET, "/greet", GOFR_H_PARAM_FORMAT, "name", "World", "Hello ", "!"},
        {GOFR_M_GET, "/error", GOFR_H_STATIC_ERROR, "some error occurred", "", "", ""},
        {GOFR_M_GET, "/users/{id:[0-9]+}/posts/{slug}", GOFR_H_HOST, "", "", "", ""},
        {GOFR_M_GET, "/nil", GOFR_H_NIL, "", "", "", ""},
        {GOFR_M_GET, "/panic", GOFR_H_PANIC, "", "", "", ""},
        {GOFR_M_POST, "/echo", GOFR_H_HOST, "", "", "", ""},
    };
    auto ck = [](int rc, const char* what) {
        if (rc) { fprintf(stderr, "%s: %s\n", what, gofr_last_error()); exit(1); }
    };
    gofr_table* table = nullptr;
    ck(gofr_table_create(&table, GOFR_FRAME_WIRE), "gofr_table_create");
    for (const Route& r : routes) {
        gofr_handler_desc h;
        memset(&h, 0, sizeof h);
        h.kind = r.kind;
        h.s0 = r.s0; h.s0_len = (uint32_t)strlen(r.s0); h.s1 = r.s1; h.s1_len = (uint32_t)strlen(r.s1);
        h.s2 = r.s2; h.s2_len = (uint32_t)strlen(r.s2); h.s3 = r.s3; h.s3_len = (uint32_t)strlen(r.s3);
        uint32_t id = 0;
        ck(gofr_table_add_route(table, r.method, r.pattern, (uint32_t)strlen(r.pattern), &h, &id), "gofr_table_add_route");
    }
    ck(gofr_table_add_default_routes(table, nullptr, 0), "gofr_table_add_default_routes");
    ck(gofr_table_seal(table), "gofr_table_seal");
    gofr_engine* engine = nullptr;
    ck(gofr_engine_create(&engine, table, 0), "gofr_engine_create");

    struct Case { const char* method; const char* target; const char* body; int status; const char* want; };
    const std::vector<Case> cases = {
        {"GET", "/hello", "", 200, "{\"data\":\"Hello World!\"}\n"},
        {"GET", "/hello2", "", 200, "{\"data\":\"Hello World!\"}\n"},
        {"PUT", "/hello", "", 200, "{\"data\":\"Hello World!\"}\n"},
        {"POST", "/hello", "", 200, "{\"data\":\"Hello World!\"}\n"},
        {"GET", "/params?name=Vikash", "", 200, "{\"data\":\"Hello Vikash!\"}\n"},
        {"DELETE", "/delete", "", 200, "{\"data\":\"Success\"}\n"},
        {"GET", "/greet", "", 200, "{\"data\":\"Hello World!\"}\n"},
        {"GET", "/greet?name=a%26b+c&name=second", "", 200, "{\"data\":\"Hello a\\u0026b c!\"}\n"},
        {"GET", "/error", "", 500, "{\"error\":{\"message\":\"some error occurred\"}}\n"},
        {"GET", "/users/42/posts/hello-world", "", 200, "{\"data\":\"user 42 post hello-world\"}\n"},
        {"GET", "/users/4x2/posts/p", "", 404, "{\"error\":{\"message\":\"http: no such file\"}}\n"},
        {"GET", "/nil", "", 200, "{}\n"},
        {"GET", "/panic", "", 500, "{\"code\":500,\"message\":\"Some unexpected error has occurred\",\"status\":\"ERROR\"}\n"},
        {"POST", "/echo", "line1\n\"quoted\" <tag>", 200, "{\"data\":\"line1\\n\\\"quoted\\\" \\u003ctag\\u003e\"}\n"},
        {"GET", "/hello/", "", 404, "{\"error\":{\"message\":\"http: no such file\"}}\n"},
        {"GET", "/a/../hello", "", 301, nullptr},
        {"OPTIONS", "/hello", "", 200, ""},
        {"PATCH", "/hello", "", 404, "{\"error\":{\"message\":\"http: no such file\"}}\n"},
        {"GET", "/.well-known/health", "", 200, "{\"data\":{}}\n"},
    };
    auto wire = [](const Case& c) {
        std::string m = std::string(c.method) + " " + c.target + " HTTP/1.1\r\nHost: localhost:8000\r\nUser-Agent: curl/8.4.0\r\n";
        const std::string body = c.body;
        if (!body.empty() || std::string(c.method) == "POST" || std::string(c.method) == "PUT")
            m += "Content-Length: " + std::to_string(body.size()) + "\r\n";
        return m + "\r\n" + body;
    };

    gofr::ConnFrontend* fe = new gofr::ConnFrontend(engine, table, 64, 200, 64 << 10);
    std::mutex app_mu;  // the holes' closures run through App::ServeHTTP one at a time
    std::mutex ids_mu;
    std::set<std::string> ids;
    std::atomic<int> bad{0}, reads{0}, requests{0}, holes{0}, headers{0};
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++)
        th.emplace_back([&, t] {
            std::mt19937 rng(1000u + (unsigned)t);
            for (int k = 0; k < conns_per_thread; k++) {
                const int c = t * conns_per_thread + k;
                // the connection's stream: every case once, from a different first case per connection; odd connections end
                // in the first part of one more request, which stays the kept tail
                std::vector<const Case*> order;
                std::string stream;
                for (size_t i = 0; i < cases.size(); i++) {
                    order.push_back(&cases[(c + i) % cases.size()]);
                    stream += wire(*order.back());
                }
                const std::string tail = c % 2 ? std::string("GET /hello HTTP/1.1\r\nHost: loc") : std::string();
                stream += tail;
                std::vector<size_t> cuts;
                for (int j = 0; j < 1 + c % 7; j++) cuts.push_back(1 + rng() % (stream.size() - 1));
                cuts.push_back(stream.size());
                std::sort(cuts.begin(), cuts.end());
                const std::string remote = "10.0.0." + std::to_string(c) + ":5" + std::to_string(1000 + c);
                std::string held;
                size_t pos = 0, q = 0;
                uint32_t status = GOFR_HTTP_CONN_DONE;
                for (size_t cut : cuts) {
                    held += stream.substr(pos, cut - pos);
                    pos = cut;
                    const gofr::ConnFrontend::Read r = fe->Serve(held, remote);
                    reads++;
                    if (r.rc != GOFR_OK) { bad++; fprintf(stderr, "connection %d: rc %d\n", c, r.rc); break; }
                    for (size_t j = 0; j < r.meta.size(); j++, q++) {
                        const Case& want = *order[q];
                        std::string resp = r.bytes.substr(r.out_off[j], r.out_off[j + 1] - r.out_off[j]);
                        int st = (int)(r.meta[j] & 0xFFFF);
                        if (st == 0) {  // a hole: the route's closure runs here, under the trace id the front-end gave it
                            gofr::App::Request req;
                            req.method = want.method;
                            req.target = want.target;
                            req.body = want.body;
                            req.trace_id = r.trace_ids[j];
                            std::lock_guard<std::mutex> lk(app_mu);
                            const gofr::App::Response a = g.ServeHTTP(req);
                            resp = a.bytes;
                            st = a.status;
                            holes++;
                        }
                        requests++;
                        if (st != want.status || (want.want && body_of(resp) != want.want)) {
                            bad++;
                            fprintf(stderr, "connection %d, %s %s: status %d body %s\n", c, want.method, want.target, st, body_of(resp).c_str());
                        }
                        const std::string h = head_of(resp), key = "\r\nX-Correlation-Id: ";
                        const size_t at = h.find(key);
                        if (at != std::string::npos) {
                            headers++;
                            if (h.substr(at + key.size(), 32) != hex(r.trace_ids[j])) { bad++; fprintf(stderr, "connection %d: X-Correlation-Id\n", c); }
                        }
                        std::lock_guard<std::mutex> lk(ids_mu);
                        if (!ids.insert(hex(r.trace_ids[j])).second) { bad++; fprintf(stderr, "connection %d: a trace id repeats\n", c); }
                    }
                    held = held.substr(r.consumed);
                    status = r.conn_status;
                    if (status == GOFR_HTTP_CONN_DEFER) break;
                }
                const uint32_t want_status = tail.empty() ? GOFR_HTTP_CONN_DONE : GOFR_HTTP_CONN_MORE;
                if (q != order.size() || status != want_status || held != tail) {
                    bad++;
                    fprintf(stderr, "connection %d: %zu of %zu requests answered, status %u, %zu bytes kept\n", c, q, order.size(), status, held.size());
                }
            }
        });
    for (auto& x : th) x.join();
    const auto s = fe->Stats();
    delete fe;
    gofr_engine_destroy(engine);
    gofr_table_destroy(table);
    printf("%d threads, %d reads in %llu batches, %d requests (%d holes), %d X-Correlation-Id headers: %s\n", threads, reads.load(),
           (unsigned long long)s[0], requests.load(), holes.load(), headers.load(), bad.load() ? "MISMATCH" : "ok");
    return bad.load() || headers.load() == 0 ? 1 : 0;
}
