// Context.Bind through the three serve entries of gofr::App (Serve, ServeConnections, ServeRead): the same bodies, the
// closure's view of c.Bind(&v) and the response bodies, for tests/test_bind_unmarshal.py to hold against its json.Unmarshal
// model.  Input: one group of bodies per line, hex, comma separated.  Per group, the bodies go through Serve as one batch,
// through ServeConnections as one connection each, and through ServeRead as one read with the requests pipelined.
// Output, per entry, group and request: "<entry> <group> <k> <bind> <response body>", all hex; bind is "O" + the struct as
// a GOFR_H_ROW row, or "E" + err.Error().
#include <cstdio>
#include <iostream>
#include <mutex>
#include <sstream>
#include <string>
#include <vector>

#include "gofr_b200.hpp"

static std::string hex(const std::string& s) {
    static const char* d = "0123456789abcdef";
    std::string o;
    for (unsigned char c : s) { o += d[c >> 4]; o += d[c & 15]; }
    return o.empty() ? "-" : o;
}
static std::string unhex(const std::string& h) {
    std::string o;
    for (size_t i = 0; i + 1 < h.size(); i += 2) o += (char)std::stoi(h.substr(i, 2), nullptr, 16);
    return o;
}
static std::string wire(const std::string& body) {
    return "POST /bind HTTP/1.1\r\nHost: t\r\nContent-Length: " + std::to_string(body.size()) + "\r\n\r\n" + body;
}
// the body of each HTTP/1.1 response in `bytes`, in order
static std::vector<std::string> bodies_of(const std::string& bytes) {
    std::vector<std::string> out;
    size_t at = 0;
    while (at < bytes.size()) {
        const size_t h = bytes.find("\r\n\r\n", at);
        const size_t cl = bytes.find("Content-Length: ", at);
        if (h == std::string::npos || cl == std::string::npos || cl > h) throw std::runtime_error("unframed response");
        const size_t n = std::stoul(bytes.substr(cl + 16, bytes.find("\r\n", cl) - cl - 16));
        out.push_back(bytes.substr(h + 4, n));
        at = h + 4 + n;
    }
    return out;
}

int main() {
    gofr::App app;
    auto& t = app.Struct("main.T").Int64("ID", "id").String("Name", "name").Bool("OK", "ok").Int32("N", "n");
    std::mutex mu;
    std::vector<std::string> seen;  // what each closure's Bind gave, in call order
    app.POST("/bind", [&](gofr::Context& c) -> gofr::Result {
        gofr::StructValue v;
        std::string got;
        const auto err = c.Bind(&v);
        if (err) got = "E" + err->message;
        else {
            std::string words, strs;
            for (size_t k = 0; k < v.fields.size(); k++) {  // id int64, name string, ok bool, n int32 (little-endian host)
                const gofr::Value& f = v.fields[k];
                if (auto* s = std::get_if<std::string>(&f.v)) { const uint32_t n = (uint32_t)s->size(); words.append((const char*)&n, 4); strs += *s; }
                else if (auto* b = std::get_if<bool>(&f.v)) { const uint32_t x = *b; words.append((const char*)&x, 4); }
                else { const int64_t x = std::get<int64_t>(f.v); words.append((const char*)&x, k == 3 ? 4 : 8); }
            }
            got = "O" + words + strs;
        }
        std::lock_guard<std::mutex> g(mu);
        seen.push_back(got);
        if (err) return *err;
        return gofr::Data(v);
    }, &t);
    app.Binds(t);
    app.Run(0);
    app.ServeReads(8, 50, 1u << 22, 7);
    const int64_t now = 1700000000;
    std::string line;
    int group = 0;
    while (std::getline(std::cin, line)) {
        std::vector<std::string> bodies;
        std::stringstream ss(line);
        for (std::string h; std::getline(ss, h, ',');) bodies.push_back(h == "-" ? std::string() : unhex(h));
        std::vector<gofr::App::Request> reqs;
        std::vector<std::string> bufs;
        std::string read;
        for (auto& b : bodies) {
            gofr::App::Request r;
            r.method = "POST";
            r.target = "/bind";
            r.body = b;
            reqs.push_back(r);
            bufs.push_back(wire(b));
            read += wire(b);
        }
        auto emit = [&](const char* entry, const std::vector<std::string>& resp) {
            if (seen.size() != bodies.size() || resp.size() != bodies.size()) throw std::runtime_error(std::string(entry) + ": request count");
            for (size_t k = 0; k < bodies.size(); k++)
                printf("%s %d %zu %s %s\n", entry, group, k, hex(seen[k]).c_str(), hex(resp[k]).c_str());
            seen.clear();
        };
        std::vector<std::string> resp;
        for (auto& r : app.Serve(reqs, now)) for (auto& b : bodies_of(r.bytes)) resp.push_back(b);
        emit("serve", resp);
        resp.clear();
        for (auto& r : app.ServeConnections(bufs, 11, now)) for (auto& b : bodies_of(r.bytes)) resp.push_back(b);
        emit("conns", resp);
        const gofr::App::ReadResponse r = app.ServeRead(read);
        if (r.rc != GOFR_OK || r.consumed != read.size()) throw std::runtime_error("ServeRead: read not served whole");
        emit("read", bodies_of(r.bytes));
        group++;
    }
    return 0;
}
