// The routes of examples/cpp/server_routes.cpp (the reference's TestGofr_ServerRoutes, pkg/gofr/gofr_test.go:40-105, plus
// the handlers of examples/http-server/main.go:29-43), with the requests sent as raw HTTP/1.1 bytes the way a socket delivers
// them: pipelined over a few connections, the last one ending in the first part of one more request.  App::ServeConnections
// routes them on the GPU, runs the closures and answers every request on the GPU.  Exits non-zero when a response is not
// what the reference's test expects, when a connection's bytes are not the concatenation of what App::Serve returns for the
// same requests (same trace ids and date), or when consumed / the connection status are wrong.
//   g++ -std=c++17 -Iinclude examples/cpp/conn_routes.cpp gofr_b200/libgofr_b200.so -o conn_routes
#include <cstdio>
#include <string>
#include <vector>

#include "gofr_b200.hpp"

static std::string body_of(const std::string& wire) {
    const size_t p = wire.find("\r\n\r\n");
    return p == std::string::npos ? wire : wire.substr(p + 4);
}

// include/gofr_b200.h, gofr_conn_batch_submit: the trace id of request j of connection c
static uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static std::array<uint8_t, 16> trace_id(uint64_t seed, uint32_t c, uint32_t j) {
    const uint64_t x = splitmix64(seed ^ splitmix64(c)), lo = splitmix64(x + 2ull * j), hi = splitmix64(x + 2ull * j + 1);
    std::array<uint8_t, 16> id{};
    for (int k = 0; k < 8; k++) { id[k] = (uint8_t)(lo >> (8 * k)); id[8 + k] = (uint8_t)(hi >> (8 * k)); }
    return id;
}

int main() {
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

    struct Case { const char* method; const char* target; const char* body; int status; const char* want; };
    const Case cases[] = {
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
    const size_t n_cases = sizeof cases / sizeof cases[0];
    auto wire = [](const Case& c) {
        std::string m = std::string(c.method) + " " + c.target + " HTTP/1.1\r\nHost: localhost:8000\r\nUser-Agent: curl/8.4.0\r\n";
        const std::string body = c.body;
        if (!body.empty() || std::string(c.method) == "POST" || std::string(c.method) == "PUT")
            m += "Content-Length: " + std::to_string(body.size()) + "\r\n";
        return m + "\r\n" + body;
    };
    // four connections: 1, 3, 7 and the rest of the cases pipelined; the last one ends in half a request
    const size_t split[] = {0, 1, 4, 11, n_cases};
    const std::string tail = "GET /hello HTTP/1.1\r\nHost: loc";
    std::vector<std::string> buffers;
    std::vector<std::vector<size_t>> conn_cases;
    for (int c = 0; c < 4; c++) {
        std::string b;
        conn_cases.emplace_back();
        for (size_t i = split[c]; i < split[c + 1]; i++) { b += wire(cases[i]); conn_cases.back().push_back(i); }
        buffers.push_back(b);
    }
    buffers.back() += tail;
    const uint64_t seed = 0x5EEDu;
    const int64_t now = 1700000000;
    const auto got = g.ServeConnections(buffers, seed, now);
    int bad = 0;
    for (size_t c = 0; c < buffers.size(); c++) {
        const bool last = c + 1 == buffers.size();
        const uint32_t want_consumed = (uint32_t)(buffers[c].size() - (last ? tail.size() : 0));
        const uint32_t want_status = last ? GOFR_HTTP_CONN_MORE : GOFR_HTTP_CONN_DONE;
        if (got[c].consumed != want_consumed || got[c].conn_status != want_status) {
            bad++;
            fprintf(stderr, "connection %zu: consumed %u status %u\n", c, got[c].consumed, got[c].conn_status);
        }
        // the same requests through App::Serve, with the trace ids the connection call gives them
        std::vector<gofr::App::Request> reqs;
        for (size_t j = 0; j < conn_cases[c].size(); j++) {
            const Case& k = cases[conn_cases[c][j]];
            gofr::App::Request r;
            r.method = k.method;
            r.target = k.target;
            r.body = k.body;
            r.trace_id = trace_id(seed, (uint32_t)c, (uint32_t)j);
            reqs.push_back(r);
        }
        const auto resp = g.Serve(reqs, now);
        std::string joined;
        for (auto& r : resp) joined += r.bytes;
        if (joined != got[c].bytes) { bad++; fprintf(stderr, "connection %zu: bytes differ from App::Serve\n", c); }
        for (size_t j = 0; j < resp.size(); j++) {
            const Case& k = cases[conn_cases[c][j]];
            const std::string body = body_of(resp[j].bytes);
            if (resp[j].status != k.status || (k.want && body != k.want)) {
                bad++;
                fprintf(stderr, "case %s %s: status %d body %s\n", k.method, k.target, resp[j].status, body.c_str());
            }
        }
    }
    printf("%zu connections, %zu requests, %s\n", buffers.size(), n_cases, bad ? "MISMATCH" : "ok");
    return bad ? 1 : 0;
}
