// The routes of examples/cpp/conn_routes.cpp (the reference's TestGofr_ServerRoutes, pkg/gofr/gofr_test.go:40-105, plus the
// handlers of examples/http-server/main.go:29-43), every one of them a closure of gofr::App, served the way net/http serves
// them: one thread per connection, each connection's requests pipelined into one byte stream and delivered as reads cut at
// arbitrary byte positions.  Each read goes through App::ServeRead: routed and bound on the GPU with the other threads' reads,
// its closures run on the connection's own thread, its responses answered on the GPU; the thread keeps the tail on
// GOFR_HTTP_CONN_MORE.  Exits non-zero when a response is not what the reference's test expects, when a response's
// X-Correlation-Id is not the trace id returned for it, when a connection ends in another state than its stream, or when
// a trace id repeats.
//   g++ -std=c++17 -Iinclude examples/cpp/conn_app_frontend.cpp gofr_b200/libgofr_b200.so -lpthread -o conn_app_frontend
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
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
static int status_of(const std::string& resp) { return resp.size() > 12 ? atoi(resp.c_str() + 9) : 0; }  // "HTTP/1.1 200"

int main(int argc, char** argv) {
    const int threads = argc > 1 ? atoi(argv[1]) : 8, conns_per_thread = argc > 2 ? atoi(argv[2]) : 6;
    const std::string helloWorld = "Hello World!";
    gofr::App g;
    g.GET("/hello", [&](gofr::Context&) -> gofr::Result { return helloWorld; });
    g.add("GET", "/hello2", [&](gofr::Context&) -> gofr::Result { return helloWorld; });
    g.PUT("/hello", [&](gofr::Context&) -> gofr::Result { return helloWorld; });
    g.POST("/hello", [&](gofr::Context&) -> gofr::Result { return helloWorld; });
    g.GET("/params", [](gofr::Context& c) -> gofr::Result { return "Hello " + c.Param("name") + "!"; });
    g.DELETE("/delete", [](gofr::Context&) -> gofr::Result { return "Success"; });
    g.GET("/greet", [](gofr::Context& c) -> gofr::Result {
        std::string name = c.Param("name");
        if (name.empty()) name = "World";
        return "Hello " + name + "!";
    });
    g.GET("/error", [](gofr::Context&) -> gofr::Result { return gofr::Error{"some error occurred"}; });
    auto& person = g.Struct("main.Person").Int("ID", "id").String("Name", "name").Bool("Admin", "admin", true);
    g.GET("/users/{id:[0-9]+}/posts/{slug}", [](gofr::Context& c) -> gofr::Result {
        return "user " + c.PathParam("id") + " post " + c.PathParam("slug");
    });
    g.GET("/person/{name}", [&](gofr::Context& c) -> gofr::Result {
        const std::string n = c.PathParam("name");
        if (n == "nobody") return gofr::Result(person({int64_t(0), n, false}), gofr::Error{"partial <result>"});
        return gofr::Data(person({int64_t(n.size()), n, n == "root"}));
    }, &person);
    g.GET("/nil", [](gofr::Context&) -> gofr::Result { return gofr::Result(); });
    g.GET("/file", [](gofr::Context&) -> gofr::Result { return gofr::ErrMissingFile(); });
    g.GET("/panic", [](gofr::Context&) -> gofr::Result { throw std::runtime_error("boom"); });
    g.POST("/echo", [](gofr::Context& c) -> gofr::Result { return c.Body(); });
    g.POST("/people", [](gofr::Context& c) -> gofr::Result {
        gofr::StructValue p;
        if (auto err = c.Bind(&p)) return *err;
        return gofr::Data(p);
    }, &person);
    g.Binds(person);
    g.GET("/raw", [](gofr::Context&) -> gofr::Result { return gofr::Raw("just <text>"); });
    g.GET("/rawerr", [](gofr::Context&) -> gofr::Result { return gofr::Result(gofr::Raw("x"), gofr::Error{"ignored"}); });
    g.Run(0);
    g.ServeReads(64, 200, 64 << 10, 0x5EED);

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
        {"GET", "/person/root", "", 200, "{\"data\":{\"id\":4,\"name\":\"root\",\"admin\":true}}\n"},
        {"GET", "/person/al%20ice", "", 200, "{\"data\":{\"id\":6,\"name\":\"al ice\"}}\n"},
        {"GET", "/person/nobody", "", 500, "{\"error\":{\"message\":\"partial \\u003cresult\\u003e\"},\"data\":{\"id\":0,\"name\":\"nobody\"}}\n"},
        {"GET", "/nil", "", 200, "{}\n"},
        {"GET", "/file", "", 404, "{\"error\":{\"message\":\"http: no such file\"}}\n"},
        {"GET", "/panic", "", 500, "{\"code\":500,\"message\":\"Some unexpected error has occurred\",\"status\":\"ERROR\"}\n"},
        {"POST", "/echo", "line1\n\"quoted\" <tag>", 200, "{\"data\":\"line1\\n\\\"quoted\\\" \\u003ctag\\u003e\"}\n"},
        {"GET", "/hello/", "", 404, "{\"error\":{\"message\":\"http: no such file\"}}\n"},
        {"GET", "/a/../hello", "", 301, nullptr},
        {"OPTIONS", "/hello", "", 200, ""},
        {"PATCH", "/hello", "", 404, "{\"error\":{\"message\":\"http: no such file\"}}\n"},
        {"GET", "/.well-known/health", "", 200, "{\"data\":{}}\n"},
        {"POST", "/people", "{\"id\":1,\"name\":\"Bob\"}", 200, "{\"data\":{\"id\":1,\"name\":\"Bob\"}}\n"},
        {"POST", "/people", "{\"id\":\"x\"}", 500, "{\"error\":{\"message\":\"json: cannot unmarshal string into Go struct field Person.id of type int\"}}\n"},
        {"POST", "/people", "", 500, "{\"error\":{\"message\":\"unexpected end of JSON input\"}}\n"},
        {"GET", "/raw", "", 200, "\"just \\u003ctext\\u003e\"\n"},
        {"GET", "/rawerr", "", 500, "\"x\"\n"},
    };
    auto wire = [](const Case& c) {
        std::string m = std::string(c.method) + " " + c.target + " HTTP/1.1\r\nHost: localhost:8000\r\nUser-Agent: curl/8.4.0\r\n";
        const std::string body = c.body;
        if (!body.empty() || std::string(c.method) == "POST" || std::string(c.method) == "PUT")
            m += "Content-Length: " + std::to_string(body.size()) + "\r\n";
        return m + "\r\n" + body;
    };

    std::mutex ids_mu;
    std::set<std::string> ids;
    std::atomic<int> bad{0}, reads{0}, requests{0}, headers{0};
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
                    const gofr::App::ReadResponse r = g.ServeRead(held, remote);
                    reads++;
                    if (r.rc != GOFR_OK) { bad++; fprintf(stderr, "connection %d: rc %d\n", c, r.rc); break; }
                    std::vector<std::string> resps;
                    for (size_t j = 0; j + 1 < r.out_off.size(); j++) resps.push_back(r.bytes.substr(r.out_off[j], r.out_off[j + 1] - r.out_off[j]));
                    if (resps.size() != r.trace_ids.size()) { bad++; fprintf(stderr, "connection %d: %zu responses for %zu ids\n", c, resps.size(), r.trace_ids.size()); break; }
                    for (size_t j = 0; j < resps.size(); j++, q++) {
                        const Case& want = *order[q];
                        const std::string& resp = resps[j];
                        const int st = status_of(resp);
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
    const gofr_conn_app_stats s = g.ReadStats();
    printf("%d threads, %d reads in %llu route and %llu respond batches, %d requests, %d X-Correlation-Id headers: %s\n", threads,
           reads.load(), (unsigned long long)s.route_batches, (unsigned long long)s.respond_batches, requests.load(), headers.load(),
           bad.load() ? "MISMATCH" : "ok");
    return bad.load() || headers.load() == 0 ? 1 : 0;
}
