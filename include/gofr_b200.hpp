// gofr_b200.hpp — C++ stand-in for the reference's app API over the C ABI (gofr_b200.h); header only, C++17.
//
// The reference is Go and no Go toolchain exists in this image, so the host side a GoFr user touches is mirrored here
// with the same names, argument meaning and error behaviour (SURVEY.md §8f rank 3):
//
//   gofr.New()                                   pkg/gofr/gofr.go:49-73        gofr::App app;
//   app.GET / PUT / POST / DELETE(pattern, h)    pkg/gofr/gofr.go:152-177      app.GET("/hello", handler);
//   type Handler func(*Context) (interface{}, error)   pkg/gofr/handler.go:12  gofr::Handler = Result(Context&)
//   c.Param(key) / c.PathParam(key)              pkg/gofr/http/request.go:28-38    c.Param("name"), c.PathParam("id")
//   app.Run()                                    pkg/gofr/gofr.go:90-126       app.Run(device): default routes, seal, engine
//   router.ServeHTTP(w, r)                       pkg/gofr/httpServer.go:29-33  app.ServeHTTP(req) / app.Serve(batch)
//
// Handlers are arbitrary closures, so they run on the host, between the two GPU stages of the split API:
//   gofr_batch_route      → mux match + middleware decisions (301 / 404 / 405 / OPTIONS) + mux.Vars spans
//   (closures run here, only for requests whose handler the reference would have called)
//   gofr_batch_submit     → Responder.Respond on every (data, err) + net/http framing: the response bytes
// A handler that throws is answered like a Go handler that panics (middleware.panicRecovery, middleware/logger.go:91-114).
//   c.Bind(&v)                                   pkg/gofr/context.go:52-54     c.Bind(&v) for a struct type the route declared
//                                                                               with Binds(): json.Unmarshal with Go's rules runs
//                                                                               on the GPU (gofr_batch_bind) before the closures
// Not mirrored: datasources, logging, CLI.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <ctime>
#include <functional>
#include <memory>
#include <optional>
#include <random>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <variant>
#include <vector>

#include "gofr_b200.h"

namespace gofr {

// Go's `error` as far as Responder.Respond looks at it: the message, and whether errors.Is(err, http.ErrMissingFile).
struct Error {
    std::string message;
    bool missing_file = false;
};
inline Error ErrMissingFile() { return Error{"http: no such file", true}; }

// A value of a struct type registered with App::Struct (fields in declaration order).  A field holds what its type says:
// int64_t / bool / std::string / double for the scalar kinds (uint64_t for a Uint64 member, a double for a Float32 one, a
// std::string or Nil for a []byte), a StructValue for a nested struct, Nil for a nil pointer, slice or map, a List for
// []T and a Map for map[string]T (a *T that is not nil is just the T).
struct Value;
struct Nil {};
// time.Time as Time.MarshalJSON sees it: Unix seconds, nanoseconds, zone offset in seconds east of UTC (Time{} = the zero Time)
struct Time {
    int64_t unix_seconds = -62135596800ll;
    uint32_t nanoseconds = 0;
    int32_t zone_offset_seconds = 0;
};
using List = std::vector<Value>;
struct StructValue {
    uint32_t type_id = 0;
    std::vector<Value> fields;
};
struct Map {
    std::vector<std::pair<std::string, Value>> entries;  // any order: the encoder sorts like encoding/json does
};
struct Value {
    std::variant<int64_t, bool, std::string, double, Nil, StructValue, List, Map, uint64_t, Time> v;
    Value() : v(int64_t(0)) {}
    Value(int64_t x) : v(x) {}
    Value(uint64_t x) : v(x) {}
    Value(Time x) : v(x) {}
    Value(int x) : v(int64_t(x)) {}
    Value(bool x) : v(x) {}
    Value(double x) : v(x) {}
    Value(std::string x) : v(std::move(x)) {}
    Value(const char* x) : v(std::string(x)) {}
    Value(Nil x) : v(x) {}
    Value(StructValue x) : v(std::move(x)) {}
    Value(List x) : v(std::move(x)) {}
    Value(Map x) : v(std::move(x)) {}
};
// interface{} as handlers of this path return it: nil, a string, or a registered struct.
using Data = std::variant<std::monostate, std::string, StructValue>;
// response.Raw{Data: ...} (pkg/gofr/http/response/raw.go:3-5): Respond writes the data bare, without the envelope
struct Raw {
    Data data;
    Raw() = default;
    Raw(Data d) : data(std::move(d)) {}
    Raw(const char* s) : data(std::string(s)) {}
};
// (interface{}, error)
struct Result {
    Data data;
    std::optional<Error> err;
    bool raw = false;  // data was returned wrapped in response.Raw
    Result() = default;
    Result(Raw r) : data(std::move(r.data)), raw(true) {}                     // return response.Raw{...}, nil
    Result(Raw r, Error e) : data(std::move(r.data)), err(std::move(e)), raw(true) {}
    Result(Data d) : data(std::move(d)) {}                                    // return data, nil
    Result(const char* s) : data(std::string(s)) {}
    Result(std::string s) : data(std::move(s)) {}
    Result(Error e) : err(std::move(e)) {}                                    // return nil, err
    Result(Data d, Error e) : data(std::move(d)), err(std::move(e)) {}        // return data, err
};

namespace detail {
inline int hexval(unsigned char c) {
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return -1;
}
// url.QueryUnescape: '+' is a space, %XX is a byte, anything else stands for itself; a bad escape is an error.
inline bool query_unescape(const std::string& s, size_t lo, size_t hi, std::string* out) {
    out->clear();
    for (size_t i = lo; i < hi; i++) {
        const unsigned char c = (unsigned char)s[i];
        if (c == '+') out->push_back(' ');
        else if (c == '%') {
            if (i + 2 >= hi) return false;
            const int a = hexval((unsigned char)s[i + 1]), b = hexval((unsigned char)s[i + 2]);
            if (a < 0 || b < 0) return false;
            out->push_back((char)(a * 16 + b));
            i += 2;
        } else out->push_back((char)c);
    }
    return true;
}
// r.URL.Query().Get(key): url.ParseQuery keeps going after a bad pair (and drops pairs containing ';'), Get returns
// the first value of the key.
inline std::string query_get(const std::string& raw, const std::string& key) {
    size_t pos = 0;
    std::string k, v;
    while (pos <= raw.size()) {
        size_t amp = raw.find('&', pos);
        if (amp == std::string::npos) amp = raw.size();
        const size_t lo = pos, hi = amp;
        pos = amp + 1;
        if (hi == lo) { if (amp == raw.size()) break; continue; }
        if (raw.find(';', lo) < hi) { if (amp == raw.size()) break; continue; }
        size_t eq = raw.find('=', lo);
        if (eq == std::string::npos || eq > hi) eq = hi;
        const bool ok = query_unescape(raw, lo, eq, &k) && (eq == hi ? (v.clear(), true) : query_unescape(raw, eq + 1, hi, &v));
        if (ok && k == key) return v;
        if (amp == raw.size()) break;
    }
    return std::string();
}
// Variable names of a mux template in order of appearance: "{name}" or "{name:pattern}", braces may nest inside the
// pattern (mux's braceIndices).
inline std::vector<std::string> template_vars(const std::string& pattern) {
    std::vector<std::string> names;
    int level = 0;
    size_t start = 0;
    for (size_t i = 0; i < pattern.size(); i++) {
        if (pattern[i] == '{') { if (level++ == 0) start = i + 1; }
        else if (pattern[i] == '}' && level > 0 && --level == 0) {
            std::string inner = pattern.substr(start, i - start);
            const size_t colon = inner.find(':');
            names.push_back(colon == std::string::npos ? inner : inner.substr(0, colon));
        }
    }
    return names;
}
inline void put_u32(std::string* s, uint32_t v) { s->append(reinterpret_cast<const char*>(&v), 4); }
}  // namespace detail

class App;

// What a handler sees of the request (gofr.Context embeds http.Request, pkg/gofr/context.go:12-27).
class Context {
public:
    std::string Param(const std::string& key) const { return detail::query_get(query_, key); }   // request.go:28-30
    std::string PathParam(const std::string& key) const {                                         // request.go:36-38
        std::string v;
        for (auto& kv : path_params_) if (kv.first == key) v = kv.second;  // a map: the last variable of that name wins
        return v;
    }
    const std::string& Method() const { return method_; }
    const std::string& Path() const { return path_; }
    const std::string& Body() const { return body_; }
    // Context.Bind (pkg/gofr/context.go:52-54 -> http/request.go:40-47): json.Unmarshal(body, &v) with v of the struct type
    // the route was registered to bind.  The decoding already happened on the GPU (gofr_batch_bind, Go's rules: exact then
    // case-insensitive keys, unknown keys skipped, null a no-op, the first UnmarshalTypeError reported); this copies the
    // fields out of the request's row, or returns json.Unmarshal's error.  A route without Binds() gets an error saying so.
    std::optional<Error> Bind(StructValue* v) const {
        if (bind_status_ == 0xFFFFFFFFu) return Error{"gofr::Context::Bind: the route was registered without a struct type to bind", false};
        if (bind_status_ != GOFR_BIND_OK) return Error{bind_row_, false};
        v->type_id = bind_type_;
        v->fields.clear();
        size_t w = 0, sp = 0;
        for (uint32_t kind : bind_kinds_) sp += (kind == GOFR_F_INT64 || kind == GOFR_F_INT || kind == GOFR_F_FLOAT64) ? 8 : 4;
        auto word = [&](size_t at) { uint32_t x; memcpy(&x, bind_row_.data() + at, 4); return x; };
        for (uint32_t kind : bind_kinds_) {
            if (kind == GOFR_F_INT64 || kind == GOFR_F_INT) { v->fields.emplace_back((int64_t)((uint64_t)word(w) | (uint64_t)word(w + 4) << 32)); w += 8; }
            else if (kind == GOFR_F_FLOAT64) { const uint64_t b = (uint64_t)word(w) | (uint64_t)word(w + 4) << 32; double x; memcpy(&x, &b, 8); v->fields.emplace_back(x); w += 8; }
            else if (kind == GOFR_F_INT32) { v->fields.emplace_back((int64_t)(int32_t)word(w)); w += 4; }
            else if (kind == GOFR_F_BOOL) { v->fields.emplace_back(word(w) != 0); w += 4; }
            else { const uint32_t n = word(w); v->fields.emplace_back(bind_row_.substr(sp, n)); sp += n; w += 4; }
        }
        return std::nullopt;
    }

private:
    friend class App;
    std::string method_, path_, query_, body_;
    std::vector<std::pair<std::string, std::string>> path_params_;
    uint32_t bind_status_ = 0xFFFFFFFFu, bind_type_ = 0;  // GOFR_BIND_* of this request's body, 0xFFFFFFFF: nothing was bound
    std::string bind_row_;                                // the row (GOFR_BIND_OK) or err.Error() (GOFR_BIND_ERROR)
    std::vector<uint32_t> bind_kinds_;
};

using Handler = std::function<Result(Context&)>;

class App {
public:
    struct Request {
        std::string method = "GET";
        std::string target = "/";            // origin form, as httptest.NewRequest takes it: path[?query]
        std::string body;
        std::optional<std::array<uint8_t, 16>> trace_id;  // the tracer middleware's span id; random when absent
    };
    struct Response {
        int status = 0;
        std::string bytes;                   // wire bytes (GOFR_FRAME_WIRE), or what the frame mode says
    };
    // Field list of a struct type handlers return: same as reflect sees it (Go name, kind, json tag, omitempty).
    class StructType {
    public:
        StructType& Int64(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_INT64, json, omitempty); }
        StructType& Int(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_INT, json, omitempty); }
        StructType& Int32(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_INT32, json, omitempty); }
        StructType& Bool(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_BOOL, json, omitempty); }
        StructType& String(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_STRING, json, omitempty); }
        StructType& Float64(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_FLOAT64, json, omitempty); }
        StructType& Float32(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_FLOAT32, json, omitempty); }
        StructType& Uint64(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_UINT64, json, omitempty); }
        StructType& TimeField(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_TIME, json, omitempty); }
        // []byte: encoding/json writes it as base64; the value is a std::string of the bytes, or Nil for the nil slice
        StructType& Bytes(const char* go, const char* json = "", bool omitempty = false) { return add(go, GOFR_F_BYTES, json, omitempty); }
        // a field of a struct type registered BEFORE this one
        StructType& Struct(const char* go, const StructType& of, const char* json = "", bool omitempty = false) {
            add(go, GOFR_F_STRUCT, json, omitempty);
            fields_.back().elem = of.id_;
            return *this;
        }
        // the field added last is a *T / []T / map[string]T of the kind it was added with
        StructType& Ptr() { fields_.back().container = GOFR_C_PTR; return *this; }
        StructType& Slice() { fields_.back().container = GOFR_C_SLICE; return *this; }
        StructType& SliceOfPtr() { fields_.back().container = GOFR_C_SLICE_PTR; return *this; }  // []*T: Nil elements are nil pointers
        StructType& MapOf() { fields_.back().container = GOFR_C_MAP; return *this; }
        uint32_t id() const { return id_; }
        StructValue operator()(std::vector<Value> fields) const { return StructValue{id_, std::move(fields)}; }

    private:
        friend class App;
        struct F { std::string go, json; uint32_t kind; bool omitempty; uint32_t container = GOFR_C_VALUE, elem = 0; };
        StructType& add(const char* go, uint32_t kind, const char* json, bool omitempty) {
            fields_.push_back(F{go, json, kind, omitempty});
            return *this;
        }
        bool bare_ = false;  // App::Bare: the one field stands for the type itself
        uint32_t id_ = 0;
        std::string go_type_;
        std::vector<F> fields_;
    };

    explicit App(uint32_t frame_mode = GOFR_FRAME_WIRE) { check(gofr_table_create(&table_, frame_mode), "gofr_table_create"); }
    ~App() {
        gofr_conn_app_frontend_destroy(reads_);
        if (engine_) gofr_engine_destroy(engine_);
        if (table_) gofr_table_destroy(table_);
    }
    App(const App&) = delete;
    App& operator=(const App&) = delete;

    // a struct type some handler returns, e.g. app.Struct("main.Person").Int("ID", "id").String("Name", "name")
    StructType& Struct(const std::string& go_type) {
        types_.emplace_back(new StructType());
        types_.back()->id_ = (uint32_t)types_.size();  // ids start at 1: 0 means "no struct type"
        types_.back()->go_type_ = go_type;
        return *types_.back();
    }

    // a non-struct type some handler returns: app.Bare("[]main.Addr").Struct("", addr).Slice(), app.Bare("map[string]string")
    // .String("").MapOf(), app.Bare("[]float64").Float64("").Slice().  Its values are StructValues with that one field.
    StructType& Bare(const std::string& go_type) {
        StructType& t = Struct(go_type);
        t.bare_ = true;
        return t;
    }

    void GET(const std::string& pattern, Handler h, const StructType* returns = nullptr) { add("GET", pattern, std::move(h), returns); }
    void PUT(const std::string& pattern, Handler h, const StructType* returns = nullptr) { add("PUT", pattern, std::move(h), returns); }
    void POST(const std::string& pattern, Handler h, const StructType* returns = nullptr) { add("POST", pattern, std::move(h), returns); }
    void DELETE(const std::string& pattern, Handler h, const StructType* returns = nullptr) { add("DELETE", pattern, std::move(h), returns); }
    void PATCH(const std::string& pattern, Handler h, const StructType* returns = nullptr) { add("PATCH", pattern, std::move(h), returns); }
    // App.add (gofr.go:171-177): registration order is match priority, as in mux
    void add(const std::string& method, const std::string& pattern, Handler h, const StructType* returns = nullptr) {
        if (engine_) throw std::logic_error("gofr::App: routes are frozen once Run has been called");
        routes_.push_back(RouteInfo{method, pattern, std::move(h), returns ? returns->id_ : 0u, detail::template_vars(pattern), 0u});
    }
    // the struct type the handler of the route registered LAST passes to c.Bind: app.POST(...); app.Binds(person);
    void Binds(const StructType& t) {
        if (routes_.empty() || engine_) throw std::logic_error("gofr::App::Binds: register the route first, before Run");
        routes_.back().bind_type = t.id_;
    }

    // App.Run (gofr.go:90-126) minus the listener: registers the struct types and routes, appends the default routes
    // (health, favicon, catch-all — gofr.go:102-107), seals the table and brings the engine up on `device`.
    void Run(int device = 0, const std::string& favicon = std::string()) {
        if (engine_) return;
        for (auto& t : types_) {
            std::vector<gofr_field_desc> fd(t->fields_.size());
            for (size_t i = 0; i < fd.size(); i++) {
                memset(&fd[i], 0, sizeof fd[i]);
                fd[i].go_name = t->fields_[i].go.c_str();
                fd[i].json_name = t->fields_[i].json.c_str();
                fd[i].kind = t->fields_[i].kind;
                fd[i].omitempty = t->fields_[i].omitempty ? 1 : 0;
                fd[i].container = (uint8_t)t->fields_[i].container;
                fd[i].elem_schema = (uint16_t)t->fields_[i].elem;
                fd[i].flags = t->bare_ ? GOFR_FIELD_BARE : 0;
            }
            check(gofr_table_add_schema(table_, t->id_, t->go_type_.c_str(), fd.data(), (uint32_t)fd.size()), "gofr_table_add_schema");
        }
        for (auto& r : routes_) {
            gofr_handler_desc h;
            memset(&h, 0, sizeof h);
            h.kind = GOFR_H_RESULT;
            h.schema_id = r.type_id;
            uint32_t id = 0;
            check(gofr_table_add_route(table_, method_code(r.method), r.pattern.c_str(), (uint32_t)r.pattern.size(), &h, &id),
                  "gofr_table_add_route");
        }
        check(gofr_table_add_default_routes(table_, (const uint8_t*)favicon.data(), (uint32_t)favicon.size()),
              "gofr_table_add_default_routes");
        check(gofr_table_seal(table_), "gofr_table_seal");
        check(gofr_engine_create(&engine_, table_, device), "gofr_engine_create");
    }

    // router.ServeHTTP for one request (a batch of one).
    Response ServeHTTP(const Request& r, int64_t unix_now = 0) { return Serve(std::vector<Request>{r}, unix_now)[0]; }

    // router.ServeHTTP for a batch: every response is what the reference's server would have written for that request.
    std::vector<Response> Serve(const std::vector<Request>& reqs, int64_t unix_now = 0) {
        if (!engine_) throw std::logic_error("gofr::App: call Run before Serve");
        const uint32_t n = (uint32_t)reqs.size();
        std::vector<Response> out(n);
        if (!n) return out;
        // ---- stage 0: what net/http hands to the router, as a request batch: method, URL.Path (decoded) | URL.RawQuery,
        // then the body ----
        std::vector<gofr_req_desc> desc(n);
        std::vector<uint8_t> ids((size_t)n * 16);
        std::string arena;
        for (uint32_t i = 0; i < n; i++) {
            const Parsed p = parse_target(reqs[i].target);
            memset(&desc[i], 0, sizeof desc[i]);
            desc[i].arena_off = (uint32_t)arena.size();
            desc[i].path_len = (uint16_t)p.path.size();
            desc[i].query_len = (uint16_t)p.query.size();
            desc[i].data_len = (uint32_t)reqs[i].body.size();
            desc[i].method = method_code(reqs[i].method);
            desc[i].flags = p.force_query ? GOFR_REQ_FORCE_QUERY : 0;
            arena += p.path;
            arena += p.query;
            arena.append((4 - arena.size() % 4) % 4, '\0');
            arena += reqs[i].body;
            arena.append((4 - arena.size() % 4) % 4, '\0');
            if (arena.size() > 0xFFFFFFF0u) throw std::invalid_argument("gofr::App::Serve: more than 4 GiB of requests");
            if (reqs[i].trace_id) memcpy(&ids[(size_t)i * 16], reqs[i].trace_id->data(), 16);
            else for (int k = 0; k < 16; k += 8) { const uint64_t v = rng_(); memcpy(&ids[(size_t)i * 16 + k], &v, 8); }
        }
        arena.append(64, '\0');
        gofr_req_batch in;
        memset(&in, 0, sizeof in);
        in.desc = desc.data(); in.trace_ids = ids.data(); in.arena = (const uint8_t*)arena.data(); in.arena_bytes = arena.size(); in.n = n;
        gofr_format_http_date(unix_now ? unix_now : (int64_t)time(nullptr), in.date);
        // ---- stage 1 (GPU): mux match, middleware decisions, path variables ----
        std::vector<uint32_t> meta(n), vars((size_t)n * GOFR_MAX_PATH_VARS);
        check(gofr_batch_route(engine_, &in, meta.data(), vars.data()), "gofr_batch_route");
        // ---- stage 1b (GPU): Context.Bind — json.Unmarshal of the bodies of the routes that declared a struct type ----
        const std::vector<Bound> bound = bind_batch(desc.data(), (const uint8_t*)arena.data(), arena.size(), meta.data(), n);
        // ---- the closures (host), only where the reference would have called one ----
        std::string rec;
        std::vector<uint32_t> rec_off;
        run_closures(desc.data(), (const uint8_t*)arena.data(), meta.data(), vars.data(), n, bound, &rec, &rec_off, "gofr::App::Serve");
        std::string arena2;
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t at = desc[i].arena_off;
            desc[i].arena_off = (uint32_t)arena2.size();
            desc[i].data_len = rec_off[i + 1] - rec_off[i];
            arena2.append(arena, at, (size_t)desc[i].path_len + desc[i].query_len);
            arena2.append((4 - arena2.size() % 4) % 4, '\0');
            arena2.append(rec, rec_off[i], desc[i].data_len);
            arena2.append((4 - arena2.size() % 4) % 4, '\0');
        }
        arena2.append(64, '\0');
        in.arena = (const uint8_t*)arena2.data();
        in.arena_bytes = arena2.size();
        // ---- stage 2 (GPU): Responder.Respond + framing ----
        uint64_t cap = 4096;
        for (uint32_t i = 0; i < n; i++) cap += gofr_table_response_bound(table_, desc[i].path_len, desc[i].query_len, desc[i].data_len);
        std::vector<uint8_t> bytes(cap);
        std::vector<uint32_t> off(n + 1), meta2(n);
        gofr_resp_batch rb;
        memset(&rb, 0, sizeof rb);
        rb.out = bytes.data(); rb.out_cap = cap; rb.out_off = off.data(); rb.meta = meta2.data();
        gofr_ticket t = 0;
        check(gofr_batch_submit(engine_, &in, &rb, &t), "gofr_batch_submit");
        check(gofr_batch_wait(engine_, t), "gofr_batch_wait");
        for (uint32_t i = 0; i < n; i++) {
            out[i].status = (int)GOFR_META_STATUS(meta2[i]);
            out[i].bytes.assign((const char*)bytes.data() + off[i], off[i + 1] - off[i]);
        }
        return out;
    }

    // What ServeConnections hands back for one connection: the bytes to write, how many of its received bytes they answer,
    // and GOFR_HTTP_CONN_DONE / MORE (keep the bytes from `consumed` on and append the next read) / DEFER (hand the bytes
    // from `consumed` on to net/http).
    struct ConnResponse {
        std::string bytes;
        uint32_t consumed = 0;
        uint32_t conn_status = GOFR_HTTP_CONN_DONE;
    };

    // net/http's conn.serve → router.ServeHTTP for a batch of connections: buffers[c] is what connection c received (pipelined
    // requests, maybe the first part of the next one).  Frames, parses and routes them on the GPU (gofr_conn_batch_route),
    // binds the bodies of the routes that declared a struct type (gofr_batch_bind on the exported requests), runs the closures
    // with a Context built from the parsed request, then splices their results in and answers every request on the GPU
    // (gofr_conn_batch_respond).  Request j of connection c gets the trace id include/gofr_b200.h states for (trace_seed, c, j).
    std::vector<ConnResponse> ServeConnections(const std::vector<std::string>& buffers, uint64_t trace_seed, int64_t unix_now = 0) {
        if (!engine_) throw std::logic_error("gofr::App: call Run before ServeConnections");
        const uint32_t nc = (uint32_t)buffers.size();
        std::vector<ConnResponse> out(nc);
        if (!nc) return out;
        std::string buf;
        std::vector<uint32_t> boff(nc + 1);
        for (uint32_t c = 0; c < nc; c++) {
            boff[c] = (uint32_t)buf.size();
            buf += buffers[c];
            if (buf.size() > 0xFFFFFFF0u) throw std::invalid_argument("gofr::App::ServeConnections: more than 4 GiB of buffers");
        }
        boff[nc] = (uint32_t)buf.size();
        buf.append(16, '\0');
        gofr_conn_batch in;
        memset(&in, 0, sizeof in);
        in.buf = (const uint8_t*)buf.data(); in.buf_off = boff.data(); in.buf_bytes = boff[nc]; in.n_conns = nc;
        in.trace_seed = trace_seed;
        gofr_format_http_date(unix_now ? unix_now : (int64_t)time(nullptr), in.date);
        uint32_t req_cap = 0;
        uint64_t cap0 = 0;
        check(gofr_conn_batch_bound(table_, boff.data(), nc, &req_cap, &cap0), "gofr_conn_batch_bound");
        const size_t rc1 = std::max<uint32_t>(req_cap, 1);
        // ---- stage 1 (GPU): frame, parse, route; the parsed requests come back ----
        std::vector<gofr_req_desc> desc(rc1);
        std::vector<uint8_t> arena((size_t)boff[nc] + 64), ids(rc1 * 16);
        std::vector<uint32_t> meta(rc1), vars(rc1 * GOFR_MAX_PATH_VARS), req_at(rc1), req_first(nc + 1), consumed(nc), cstat(nc);
        gofr_conn_route rt;
        memset(&rt, 0, sizeof rt);
        rt.req_cap = req_cap; rt.desc = desc.data(); rt.arena = arena.data(); rt.meta = meta.data(); rt.vars = vars.data();
        rt.req_at = req_at.data(); rt.trace_ids = ids.data(); rt.req_first = req_first.data(); rt.consumed = consumed.data();
        rt.conn_status = cstat.data();
        check(gofr_conn_batch_route(engine_, &in, &rt), "gofr_conn_batch_route");
        const uint32_t n = req_first[nc];
        // ---- stage 1b (GPU): Context.Bind on the exported requests ----
        const std::vector<Bound> bound = bind_batch(desc.data(), arena.data(), arena.size(), meta.data(), n);
        // ---- the closures (host), only where the reference would have called one ----
        std::string rec;
        std::vector<uint32_t> rec_off;
        run_closures(desc.data(), arena.data(), meta.data(), vars.data(), n, bound, &rec, &rec_off, "gofr::App::ServeConnections");
        // ---- stage 2 (GPU): the results spliced in, Responder.Respond + framing for every request ----
        uint64_t cap = 0;
        check(gofr_conn_respond_bound(table_, desc.data(), n, rec_off.data(), &cap), "gofr_conn_respond_bound");
        cap += 4096;
        gofr_conn_results res;
        memset(&res, 0, sizeof res);
        res.rec = (const uint8_t*)rec.data(); res.rec_off = rec_off.data(); res.rec_bytes = rec.size(); res.n_req = n;
        std::vector<uint8_t> bytes(cap);
        std::vector<uint32_t> off(rc1 + 1);
        gofr_conn_resp o;
        memset(&o, 0, sizeof o);
        o.out = bytes.data(); o.out_cap = cap; o.req_cap = req_cap; o.out_off = off.data(); o.meta = meta.data();
        o.req_at = req_at.data(); o.req_first = req_first.data(); o.consumed = consumed.data(); o.conn_status = cstat.data();
        gofr_ticket tk = 0;
        check(gofr_conn_batch_respond(engine_, &in, &res, &o, nullptr, &tk), "gofr_conn_batch_respond");
        check(gofr_batch_wait(engine_, tk), "gofr_batch_wait");
        for (uint32_t c = 0; c < nc; c++) {
            const uint32_t a = off[req_first[c]], b = off[req_first[c + 1]];
            out[c].bytes.assign((const char*)bytes.data() + a, b - a);
            out[c].consumed = consumed[c];
            out[c].conn_status = cstat[c];
        }
        return out;
    }

    // Starts the per-read entry ServeRead (after Run, before any ServeRead): a gofr_conn_app_frontend on this App's engine
    // whose route batches bind the bodies of the routes registered with Binds, with max_batch / max_wait_us as
    // gofr_frontend_create's, reads of at most max_conn_bytes, and middleware.Logging's lines when log is set.
    void ServeReads(uint32_t max_batch = 1024, uint32_t max_wait_us = 200, uint32_t max_conn_bytes = 16384, uint64_t seed = 0,
                    bool log = false, int32_t tz_offset_s = 0) {
        if (!engine_) throw std::logic_error("gofr::App: call Run before ServeReads");
        if (reads_) throw std::logic_error("gofr::App::ServeReads: already started");
        std::vector<uint32_t> schema(routes_.size()), fields(routes_.size());
        for (size_t r = 0; r < routes_.size(); r++) {
            schema[r] = routes_[r].bind_type;
            fields[r] = schema[r] ? (uint32_t)types_[schema[r] - 1]->fields_.size() : 0u;
            max_fields_ = std::max(max_fields_, fields[r]);
            if (!schema[r]) continue;
            const StructType& t = *types_[schema[r] - 1];
            size_t name = 0;
            for (auto& f : t.fields_) name = std::max(name, (f.json.empty() ? f.go : f.json).size());
            max_names_ = std::max<uint64_t>(max_names_, t.go_type_.size() + name);
        }
        check(gofr_conn_app_frontend_create(&reads_, engine_, max_batch, max_wait_us, max_conn_bytes, log ? 1 : 0, tz_offset_s, seed,
                                            schema.data(), (uint32_t)schema.size(), fields.data()),
              "gofr_conn_app_frontend_create");
        reads_max_ = max_conn_bytes;
        reads_log_ = log;
    }
    // pin the Date header and the log time of ServeRead's respond batches (tests); 0 = wall clock
    void SetReadClock(int64_t unix_ns) { check(gofr_conn_app_frontend_set_clock(reads_, unix_ns), "gofr_conn_app_frontend_set_clock"); }
    gofr_conn_app_stats ReadStats() const {
        gofr_conn_app_stats st{};
        check(gofr_conn_app_frontend_stats(reads_, &st), "gofr_conn_app_frontend_stats");
        return st;
    }

    // What ServeRead hands back for one read: ServeConnections' ConnResponse for it, request k's response at bytes[out_off[k]
    // .. out_off[k+1]), each request's trace id (the bytes of its X-Correlation-Id) and, with log, middleware.Logging's lines
    // of the requests answered on the GPU.
    struct ReadResponse : ConnResponse {
        int rc = GOFR_OK;  // GOFR_ERR_CAPACITY: the read exceeds max_conn_bytes, nothing was queued (hand it to net/http)
        std::vector<uint32_t> out_off{0};
        std::vector<std::array<uint8_t, 16>> trace_ids;
        std::string log;
    };

    // net/http's conn.serve for one read of one connection (the kept tail plus the new bytes), on the connection's own
    // thread: the read is framed, parsed, routed and bound on the GPU with the other threads' reads (one route batch), the
    // closures of its requests run here, on the calling thread, with the Context ServeConnections builds, and their results
    // are spliced in and every request answered on the GPU (one respond batch, gofr_conn_batch_respond_ex under the trace
    // key the route call returned).  Thread-safe: any number of threads, one call per connection at a time.  remote and
    // start_unix_ns are Logging's req.RemoteAddr and start clock for this read.
    ReadResponse ServeRead(const std::string& buf, const std::string& remote = std::string(), int64_t start_unix_ns = 0) const {
        if (!reads_) throw std::logic_error("gofr::App: call ServeReads before ServeRead");
        ReadResponse r;
        if (buf.size() > reads_max_) { r.rc = GOFR_ERR_CAPACITY; return r; }
        const uint32_t len = (uint32_t)buf.size(), off[2] = {0, len}, roff[2] = {0, (uint32_t)remote.size()};
        uint32_t req_cap = 0;
        uint64_t cap0 = 0;
        check(gofr_conn_batch_bound(table_, off, 1, &req_cap, &cap0), "gofr_conn_batch_bound");
        const size_t rc1 = std::max<uint32_t>(req_cap, 1);
        // ---- route round: frame, parse, route and bind on the GPU ----
        std::vector<gofr_req_desc> desc(rc1);
        std::vector<uint8_t> arena((size_t)len + 80), ids(rc1 * 16);
        std::vector<uint32_t> meta(rc1), vars(rc1 * GOFR_MAX_PATH_VARS), req_at(rc1), bstat(rc1), row_off(rc1 + 1);
        std::vector<uint8_t> rows((size_t)req_cap * (8 * max_fields_ + 70 + max_names_) + 3 * (size_t)len + 1);  // GOFR_BIND_ROW_BOUND over the read
        uint32_t first[2] = {0, 0};
        gofr_conn_route rt{};
        rt.req_cap = req_cap; rt.desc = desc.data(); rt.arena = arena.data(); rt.meta = meta.data(); rt.vars = vars.data();
        rt.req_at = req_at.data(); rt.trace_ids = ids.data(); rt.req_first = first; rt.consumed = &r.consumed; rt.conn_status = &r.conn_status;
        gofr_conn_app_bind bd{bstat.data(), row_off.data(), rows.data(), rows.size(), 0};
        uint64_t key = 0;
        check(gofr_conn_app_frontend_route(reads_, (const uint8_t*)buf.data(), len, &rt, &bd, &key), "gofr_conn_app_frontend_route");
        const uint32_t n = first[1];
        std::vector<Bound> bound(n);
        for (uint32_t i = 0; i < n; i++) {
            bound[i].status = bstat[i];
            bound[i].row.assign((const char*)rows.data() + row_off[i], row_off[i + 1] - row_off[i]);
        }
        // ---- the closures, on this thread ----
        std::string rec;
        std::vector<uint32_t> rec_off;
        run_closures(desc.data(), arena.data(), meta.data(), vars.data(), n, bound, &rec, &rec_off, "gofr::App::ServeRead");
        // ---- respond round: the results spliced in, every request answered on the GPU ----
        uint64_t cap = 0;
        check(gofr_conn_respond_bound(table_, desc.data(), n, rec_off.data(), &cap), "gofr_conn_respond_bound");
        cap += 4096;
        uint32_t line_cap = 0;
        uint64_t log_cap = 0;
        if (reads_log_) check(gofr_conn_log_bound(off, roff, 1, &line_cap, &log_cap), "gofr_conn_log_bound");
        r.bytes.resize(cap);
        r.trace_ids.resize(rc1);
        r.log.resize(log_cap + 1);
        r.out_off.resize(rc1 + 1);
        std::vector<uint32_t> log_off(line_cap + 1), log_req(std::max<uint32_t>(line_cap, 1));
        gofr_conn_results res{(const uint8_t*)rec.data(), rec_off.data(), rec.size(), n, 0};
        gofr_conn_resp o{};
        o.out = (uint8_t*)&r.bytes[0]; o.out_cap = cap; o.req_cap = req_cap; o.out_off = r.out_off.data(); o.meta = meta.data();
        o.req_at = req_at.data(); o.trace_ids = r.trace_ids[0].data(); o.req_first = first; o.consumed = &r.consumed;
        o.conn_status = &r.conn_status;
        gofr_conn_log l{};
        l.line_cap = line_cap; l.out = (uint8_t*)&r.log[0]; l.out_cap = log_cap; l.log_off = log_off.data(); l.log_req = log_req.data();
        r.rc = gofr_conn_app_frontend_respond(reads_, (const uint8_t*)buf.data(), len, key, &res, (const uint8_t*)remote.data(),
                                              (uint32_t)remote.size(), start_unix_ns, &o, reads_log_ ? &l : nullptr);
        check(r.rc, "gofr_conn_app_frontend_respond");
        r.bytes.resize(o.out_bytes);
        r.trace_ids.resize(first[1]);
        r.out_off.resize(first[1] + 1);
        r.log.resize(reads_log_ ? l.out_bytes : 0);
        return r;
    }

    // url.ParseRequestURI as Serve applies it to Request::target (tests): false for what httptest.NewRequest would refuse
    static bool ParseTarget(const std::string& target, std::string* path, std::string* raw_query, bool* force_query) {
        try {
            Parsed p = parse_target(target);
            *path = p.path; *raw_query = p.query; *force_query = p.force_query;
            return true;
        } catch (const std::invalid_argument&) {
            return false;
        }
    }

    // the record Serve hands to stage 2 for this (data, err) when the route returns struct type `returns` (tests)
    std::string ResultRecord(const Result& res, const StructType* returns = nullptr) const { return encode_result(returns ? returns->id_ : 0u, res); }

    gofr_engine* engine() const { return engine_; }
    gofr_table* table() const { return table_; }

private:
    struct RouteInfo {
        std::string method, pattern;
        Handler fn;
        uint32_t type_id;
        std::vector<std::string> var_names;
        uint32_t bind_type;  // struct type of c.Bind, 0: the handler does not bind
    };
    struct Bound { uint32_t status = 0xFFFFFFFFu; std::string row; };
    struct Parsed { std::string path, query; bool force_query = false; };

    static void check(int rc, const char* where) {
        if (rc != GOFR_OK) throw std::runtime_error(std::string(where) + ": " + gofr_last_error());
    }
    static const char* const* method_names() {
        static const char* names[] = {"GET", "HEAD", "POST", "PUT", "PATCH", "DELETE", "CONNECT", "OPTIONS", "TRACE"};
        return names;
    }
    static uint8_t method_code(const std::string& m) {
        for (uint8_t k = 0; k < 9; k++) if (m == method_names()[k]) return k;
        return GOFR_M_OTHER;
    }
    // the request-head parser only accepts the methods with a code below 9
    static std::string method_name(uint8_t code) { return code < 9 ? method_names()[code] : ""; }
    // url.ParseRequestURI for an origin-form target: Path is the unescaped part before the first '?', RawQuery the rest
    static Parsed parse_target(const std::string& target) {
        if (target.empty() || target[0] != '/') throw std::invalid_argument("gofr::App: request target must be in origin form: " + target);
        Parsed p;
        const size_t q = target.find('?');
        const size_t pe = q == std::string::npos ? target.size() : q;
        for (size_t i = 0; i < pe; i++) {
            if (target[i] == '%') {
                const int a = i + 2 < pe ? detail::hexval((unsigned char)target[i + 1]) : -1;
                const int b = i + 2 < pe ? detail::hexval((unsigned char)target[i + 2]) : -1;
                if (a < 0 || b < 0) throw std::invalid_argument("gofr::App: invalid URL escape in " + target);
                p.path.push_back((char)(a * 16 + b));
                i += 2;
            } else p.path.push_back(target[i]);
        }
        if (q != std::string::npos) {
            p.query = target.substr(q + 1);
            p.force_query = p.query.empty();
        }
        if (p.path.size() > 0xFFFF || p.query.size() > 0xFFFF) throw std::invalid_argument("gofr::App: request target too long");
        return p;
    }

    // Context.Bind for every request of a routed batch (desc into arena, meta as gofr_route_device gives it) whose route
    // declared a struct type: one gofr_batch_bind per type, rows in slots of GOFR_BIND_ROW_SLOT for the type's fields and
    // the longest of those bodies, and one more for the rows that outgrew it.  bound[i].status stays 0xFFFFFFFF for a
    // request that was not bound.
    std::vector<Bound> bind_batch(const gofr_req_desc* desc, const uint8_t* arena, uint64_t arena_bytes, const uint32_t* meta, uint32_t n) const {
        std::vector<Bound> bound(n);
        for (auto& t : types_) {
            std::vector<uint32_t> who;
            std::vector<gofr_req_desc> bd;
            uint32_t longest = 0;
            for (uint32_t i = 0; i < n; i++) {
                const uint32_t route = GOFR_META_ROUTE(meta[i]);
                if (GOFR_META_STATUS(meta[i]) || route >= routes_.size() || routes_[route].bind_type != t->id_) continue;
                who.push_back(i);
                bd.push_back(desc[i]);
                longest = std::max(longest, desc[i].data_len);
            }
            if (who.empty()) continue;
            gofr_req_batch bin;
            memset(&bin, 0, sizeof bin);
            bin.desc = bd.data(); bin.arena = arena; bin.arena_bytes = arena_bytes; bin.n = (uint32_t)who.size();
            const uint32_t slot = (uint32_t)GOFR_BIND_ROW_SLOT(t->fields_.size(), longest);
            std::vector<uint8_t> rows((size_t)who.size() * slot);
            std::vector<uint32_t> blen(who.size()), bstat(who.size());
            check(gofr_batch_bind(engine_, t->id_, &bin, rows.data(), slot, blen.data(), bstat.data()), "gofr_batch_bind");
            std::vector<uint32_t> over;  // rows the slot did not hold: the bind reported their exact length
            std::vector<gofr_req_desc> od;
            uint32_t wide = 0;
            for (size_t k = 0; k < who.size(); k++) {
                bound[who[k]].status = bstat[k];
                if (blen[k] <= slot) bound[who[k]].row.assign((const char*)rows.data() + k * slot, blen[k]);
                else if (bstat[k] != GOFR_BIND_HOST) { over.push_back(who[k]); od.push_back(bd[k]); wide = std::max(wide, blen[k]); }
            }
            if (over.empty()) continue;
            // invalid UTF-8 triples a string, a long literal or name lengthens an error text: bind those requests once more
            // in slots of the longest
            const uint32_t slot2 = (wide + 15u) & ~15u;
            bin.desc = od.data(); bin.n = (uint32_t)over.size();
            rows.assign((size_t)over.size() * slot2, 0);
            check(gofr_batch_bind(engine_, t->id_, &bin, rows.data(), slot2, blen.data(), bstat.data()), "gofr_batch_bind");
            for (size_t k = 0; k < over.size(); k++) {
                // gofr_batch_bind reports exact lengths, so every row fits here; one that does not is left to the host
                const bool host = blen[k] > slot2;
                bound[over[k]].status = host ? (uint32_t)GOFR_BIND_HOST : bstat[k];
                bound[over[k]].row.assign((const char*)rows.data() + k * slot2, host ? 0u : blen[k]);
            }
        }
        return bound;
    }

    // handler.ServeHTTP for every request of a routed batch (desc into arena, meta / vars as gofr_route_device gives them,
    // bound[i] its Context.Bind result), where the reference would call a closure: the request as net/http parsed it, the
    // closure, and its (data, err) as the GOFR_H_RESULT record stage 2 splices in.  Record i is rec[rec_off[i] .. rec_off[i+1])
    // (empty where no closure ran).
    void run_closures(const gofr_req_desc* desc, const uint8_t* arena, const uint32_t* meta, const uint32_t* vars, uint32_t n,
                      const std::vector<Bound>& bound, std::string* rec, std::vector<uint32_t>* rec_off, const char* who) const {
        rec_off->assign((size_t)n + 1, 0);
        for (uint32_t i = 0; i < n; i++) {
            (*rec_off)[i] = (uint32_t)rec->size();
            const uint32_t route = GOFR_META_ROUTE(meta[i]);
            if (GOFR_META_STATUS(meta[i]) == 0 && route < routes_.size())
                *rec += run_handler(routes_[route], desc[i], arena, &vars[(size_t)i * GOFR_MAX_PATH_VARS], bound[i]);
            if (rec->size() > 0xFFFFFFF0u) throw std::invalid_argument(std::string(who) + ": more than 4 GiB of handler results");
        }
        (*rec_off)[n] = (uint32_t)rec->size();
    }

    // handler.ServeHTTP (pkg/gofr/handler.go:32-36): build the Context from request d (path | query, then the body, in
    // arena), call the closure, describe (data, err) for Respond
    std::string run_handler(const RouteInfo& r, const gofr_req_desc& d, const uint8_t* arena, const uint32_t* vars, const Bound& bound) const {
        Context c;
        if (r.bind_type) {
            c.bind_status_ = bound.status;
            c.bind_type_ = r.bind_type;
            c.bind_row_ = bound.status == GOFR_BIND_HOST ? std::string("gofr::Context::Bind: body not decided on the device (nesting deeper than 64, or a float64 literal it does not round itself)") : bound.row;
            if (bound.status == GOFR_BIND_HOST) c.bind_status_ = GOFR_BIND_ERROR;
            for (auto& ty : types_) if (ty->id_ == r.bind_type) for (auto& f : ty->fields_) c.bind_kinds_.push_back(f.kind);
        }
        const char* at = (const char*)arena + d.arena_off;
        c.method_ = method_name(d.method);
        c.path_.assign(at, d.path_len);
        c.query_.assign(at + d.path_len, d.query_len);
        c.body_.assign(at + ((d.path_len + d.query_len + 3u) & ~3u), d.data_len);
        for (size_t k = 0; k < r.var_names.size() && k < GOFR_MAX_PATH_VARS; k++) {
            if (vars[k] == 0xFFFFFFFFu) continue;
            c.path_params_.emplace_back(r.var_names[k], c.path_.substr(vars[k] & 0xFFFFu, vars[k] >> 16));
        }
        Result res;
        try {
            res = r.fn(c);
        } catch (...) {
            std::string rec;
            detail::put_u32(&rec, 0xFFFFFFFFu);  // not an outcome: answered like a panicking handler
            return rec;
        }
        return encode_result(r.type_id, res);
    }

    // (data, err) as the GOFR_H_RESULT record stage 2 reads (include/gofr_b200.h): what Responder.Respond will see
    std::string encode_result(uint32_t route_type_id, const Result& res) const {
        std::string rec;
        const bool has_err = res.err.has_value();
        if (res.raw) {  // the error only picks the status code (responder.go:20-26)
            const uint32_t es = !has_err ? GOFR_RESULT_RAW_OK : res.err->missing_file ? GOFR_RESULT_RAW_MISSING : GOFR_RESULT_RAW_ERR;
            if (auto* sv = std::get_if<StructValue>(&res.data)) {
                std::string fixed, strings;
                if (sv->type_id != route_type_id || !encode_struct(*sv, &fixed, &strings)) { detail::put_u32(&rec, 0xFFFFFFFFu); return rec; }
                detail::put_u32(&rec, GOFR_RESULT_RAW_DATA | es << 8);
                rec += fixed;
                rec += strings;
            } else if (auto* s = std::get_if<std::string>(&res.data)) {
                detail::put_u32(&rec, GOFR_RESULT_RAW_STRING | es << 8);
                detail::put_u32(&rec, (uint32_t)s->size());
                rec += *s;
            } else detail::put_u32(&rec, GOFR_RESULT_RAW_NIL | es << 8);
            return rec;
        }
        if (auto* sv = std::get_if<StructValue>(&res.data)) {
            std::string fixed, strings;
            if (sv->type_id != route_type_id || !encode_struct(*sv, &fixed, &strings)) { detail::put_u32(&rec, 0xFFFFFFFFu); return rec; }
            if (has_err) {  // (data, err): message length word + fixed words, then message bytes + string bytes
                detail::put_u32(&rec, GOFR_RESULT_BOTH);
                detail::put_u32(&rec, (uint32_t)res.err->message.size());
                rec += fixed;
                rec += res.err->message;
                rec += strings;
            } else {
                detail::put_u32(&rec, GOFR_RESULT_DATA);
                rec += fixed;
                rec += strings;
            }
        } else if (has_err) {
            // a string next to an error is dropped here: response{Error, Data} with both members needs a struct type
            detail::put_u32(&rec, res.err->missing_file ? GOFR_RESULT_MISSING : GOFR_RESULT_ERROR);
            detail::put_u32(&rec, (uint32_t)res.err->message.size());
            rec += res.err->message;
        } else if (auto* s = std::get_if<std::string>(&res.data)) {
            detail::put_u32(&rec, GOFR_RESULT_STRING);
            detail::put_u32(&rec, (uint32_t)s->size());
            rec += *s;
        } else {
            detail::put_u32(&rec, GOFR_RESULT_NIL);
        }
        return rec;
    }

    const StructType* type_of(uint32_t id) const {
        for (auto& ty : types_) if (ty->id_ == id) return ty.get();
        return nullptr;
    }
    static bool scalar_words(uint32_t kind, const Value& v, std::string* out) {
        if (kind == GOFR_F_BOOL) {
            auto* b = std::get_if<bool>(&v.v);
            if (!b) return false;
            detail::put_u32(out, *b ? 1u : 0u);
        } else if (kind == GOFR_F_FLOAT64) {
            double d;
            if (auto* x = std::get_if<double>(&v.v)) d = *x;
            else if (auto* i = std::get_if<int64_t>(&v.v)) d = (double)*i;
            else return false;
            uint64_t bits;
            memcpy(&bits, &d, 8);
            detail::put_u32(out, (uint32_t)bits);
            detail::put_u32(out, (uint32_t)(bits >> 32));
        } else if (kind == GOFR_F_FLOAT32) {
            float d;
            if (auto* x = std::get_if<double>(&v.v)) d = (float)*x;
            else if (auto* i = std::get_if<int64_t>(&v.v)) d = (float)*i;
            else return false;
            uint32_t bits;
            memcpy(&bits, &d, 4);
            detail::put_u32(out, bits);
        } else if (kind == GOFR_F_TIME) {
            auto* t = std::get_if<Time>(&v.v);
            if (!t) return false;
            detail::put_u32(out, (uint32_t)(uint64_t)t->unix_seconds);
            detail::put_u32(out, (uint32_t)((uint64_t)t->unix_seconds >> 32));
            detail::put_u32(out, t->nanoseconds);
            detail::put_u32(out, (uint32_t)t->zone_offset_seconds);
        } else if (kind == GOFR_F_UINT64) {
            uint64_t u;
            if (auto* x = std::get_if<uint64_t>(&v.v)) u = *x;
            else if (auto* i = std::get_if<int64_t>(&v.v); i && *i >= 0) u = (uint64_t)*i;
            else return false;
            detail::put_u32(out, (uint32_t)u);
            detail::put_u32(out, (uint32_t)(u >> 32));
        } else {
            auto* x = std::get_if<int64_t>(&v.v);
            if (!x) return false;
            if (kind == GOFR_F_INT32) detail::put_u32(out, (uint32_t)(int32_t)*x);
            else { detail::put_u32(out, (uint32_t)(uint64_t)*x); detail::put_u32(out, (uint32_t)((uint64_t)*x >> 32)); }
        }
        return true;
    }
    // T by value: its fixed words to `fixed`, its variable part to `var` (include/gofr_b200.h "Row format")
    bool encode_plain(const StructType::F& f, const Value& v, std::string* fixed, std::string* var) const {
        if (f.kind == GOFR_F_STRING) {
            auto* s = std::get_if<std::string>(&v.v);
            if (!s) return false;
            detail::put_u32(fixed, (uint32_t)s->size());
            *var += *s;
            return true;
        }
        if (f.kind == GOFR_F_BYTES) {  // length word (GOFR_NIL_COUNT: the nil slice), bytes in the variable part
            if (std::holds_alternative<Nil>(v.v)) { detail::put_u32(fixed, GOFR_NIL_COUNT); return true; }
            auto* s = std::get_if<std::string>(&v.v);
            if (!s) return false;
            detail::put_u32(fixed, (uint32_t)s->size());
            *var += *s;
            return true;
        }
        if (f.kind == GOFR_F_STRUCT) {
            auto* sv = std::get_if<StructValue>(&v.v);
            return sv && sv->type_id == f.elem && encode_struct(*sv, fixed, var);
        }
        return scalar_words(f.kind, v, fixed);
    }
    // E(T): an element of a slice / map, entirely in the variable part
    bool encode_element(const StructType::F& f, const Value& v, std::string* var) const {
        if (f.kind == GOFR_F_STRING) {
            auto* s = std::get_if<std::string>(&v.v);
            if (!s) return false;
            detail::put_u32(var, (uint32_t)s->size());
            *var += *s;
            return true;
        }
        if (f.kind == GOFR_F_BYTES) {
            if (std::holds_alternative<Nil>(v.v)) { detail::put_u32(var, GOFR_NIL_COUNT); return true; }
            auto* s = std::get_if<std::string>(&v.v);
            if (!s) return false;
            detail::put_u32(var, (uint32_t)s->size());
            *var += *s;
            return true;
        }
        if (f.kind == GOFR_F_STRUCT) {
            auto* sv = std::get_if<StructValue>(&v.v);
            std::string fx, vr;
            if (!sv || sv->type_id != f.elem || !encode_struct(*sv, &fx, &vr)) return false;
            *var += fx;
            *var += vr;
            return true;
        }
        return scalar_words(f.kind, v, var);
    }
    size_t fixed_bytes(const StructType::F& f) const {
        if (f.container == GOFR_C_SLICE || f.container == GOFR_C_MAP || f.container == GOFR_C_SLICE_PTR) return 4;
        size_t n = f.kind == GOFR_F_TIME ? 16 : (f.kind == GOFR_F_INT64 || f.kind == GOFR_F_INT || f.kind == GOFR_F_FLOAT64 || f.kind == GOFR_F_UINT64) ? 8 : 4;
        if (f.kind == GOFR_F_STRUCT) {
            n = 0;
            if (const StructType* t = type_of(f.elem)) for (auto& g : t->fields_) n += fixed_bytes(g);
        }
        return n + (f.container == GOFR_C_PTR ? 4 : 0);
    }
    bool encode_struct(const StructValue& sv, std::string* fixed, std::string* var) const {
        const StructType* t = type_of(sv.type_id);
        if (!t || t->fields_.size() != sv.fields.size()) return false;
        for (size_t i = 0; i < sv.fields.size(); i++) {
            const StructType::F& f = t->fields_[i];
            const Value& v = sv.fields[i];
            const bool nil = std::holds_alternative<Nil>(v.v);
            if (f.container == GOFR_C_VALUE) {
                if (!encode_plain(f, v, fixed, var)) return false;
            } else if (f.container == GOFR_C_PTR) {
                if (nil) fixed->append(fixed_bytes(f), '\0');
                else { detail::put_u32(fixed, 1); if (!encode_plain(f, v, fixed, var)) return false; }
            } else if (f.container == GOFR_C_SLICE || f.container == GOFR_C_SLICE_PTR) {
                auto* l = std::get_if<List>(&v.v);
                if (!nil && !l) return false;
                detail::put_u32(fixed, nil ? GOFR_NIL_COUNT : (uint32_t)l->size());
                if (l) for (auto& e : *l) {
                    if (f.container == GOFR_C_SLICE_PTR) {  // presence word; a nil element owns nothing else
                        const bool enil = std::holds_alternative<Nil>(e.v);
                        detail::put_u32(var, enil ? 0u : 1u);
                        if (enil) continue;
                    }
                    if (!encode_element(f, e, var)) return false;
                }
            } else {
                auto* m = std::get_if<Map>(&v.v);
                if (!nil && !m) return false;
                detail::put_u32(fixed, nil ? GOFR_NIL_COUNT : (uint32_t)m->entries.size());
                if (m) for (auto& kv : m->entries) {
                    detail::put_u32(var, (uint32_t)kv.first.size());
                    *var += kv.first;
                    if (!encode_element(f, kv.second, var)) return false;
                }
            }
        }
        return true;
    }

    gofr_table* table_ = nullptr;
    gofr_engine* engine_ = nullptr;
    std::vector<std::unique_ptr<StructType>> types_;
    std::vector<RouteInfo> routes_;
    std::mt19937_64 rng_{0x9E3779B97F4A7C15ull};
    gofr_conn_app_frontend* reads_ = nullptr;  // ServeRead's front-end (ServeReads)
    uint32_t reads_max_ = 0, max_fields_ = 0;
    uint64_t max_names_ = 0;  // of the bound types: Go type name plus longest JSON name (GOFR_BIND_ROW_BOUND's names)
    bool reads_log_ = false;
    friend class ProtoCodec;
};

// grpc-go's proto codec for a batch of unary calls on the app's engine (gofr_proto_batch_decode / _encode, host buffers):
// Decode turns request frames (5-byte prefix + message) into rows in the layout of include/gofr_b200.h ("Row format"),
// the handlers run on the host, Encode turns their response rows into frames.  Built from message types: msgs[m] lists the
// fields of type m in ascending number order (a GOFR_PB_MESSAGE or GOFR_PB_MAP field names a type by its index in msgs),
// `root` is the type of the records.  The app must be running (App::Run).
class ProtoCodec {
public:
    struct Field {
        uint32_t number;
        uint32_t type;          // GOFR_PB_*, GOFR_PB_MESSAGE or GOFR_PB_MAP
        bool repeated = false;
        uint16_t msg = 0;       // GOFR_PB_MESSAGE / GOFR_PB_MAP: the message or entry type
        uint8_t presence = 0;   // 0, GOFR_PB_OPTIONAL or a oneof group 1..7
    };
    struct Batch {
        std::vector<std::string> records;  // rows (Decode) or frames (Encode); empty where status is not GOFR_GRPC_OK
        std::vector<uint32_t> status;      // GOFR_GRPC_*: a frame still GOFR_GRPC_DEFER is for the host's own decoder
    };

    // the description in the ABI's form, checked (gofr_proto_nested_bound) on construction
    struct Description {
        Description(const std::vector<std::vector<Field>>& msgs, uint32_t root_) : root(root_) {
            bool any_presence = false;
            for (auto& fs : msgs) {
                this->msgs.push_back(gofr_proto_nmsg{(uint16_t)fields.size(), (uint16_t)fs.size()});
                for (auto& f : fs) {
                    fields.push_back(gofr_proto_nfield{f.number, (uint8_t)f.type, (uint8_t)(f.repeated ? 1 : 0), f.msg});
                    presence_.push_back(f.presence);
                    any_presence |= f.presence != 0;
                }
            }
            if (!any_presence) presence_.clear();
            bound(true);
        }
        const uint8_t* presence() const { return presence_.empty() ? nullptr : presence_.data(); }
        // (per_byte, per_record) of gofr_proto_nested_bound for the direction
        std::pair<uint32_t, uint32_t> bound(bool decode) const {
            uint32_t pb = 0, pr = 0;
            check(gofr_proto_nested_bound(msgs.data(), (uint32_t)msgs.size(), fields.data(), (uint32_t)fields.size(), root,
                                          presence(), decode ? 1 : 0, &pb, &pr), "gofr_proto_nested_bound");
            return {pb, pr};
        }
        uint32_t root;
        std::vector<gofr_proto_nmsg> msgs;
        std::vector<gofr_proto_nfield> fields;
        std::vector<uint8_t> presence_;
    };
    static void check(int rc, const char* where) {
        if (rc != GOFR_OK) throw std::runtime_error(std::string(where) + ": " + gofr_last_error());
    }

    ProtoCodec(const App& app, const std::vector<std::vector<Field>>& msgs, uint32_t root) : engine_(app.engine_), d_(msgs, root) {
        if (!engine_) throw std::logic_error("gofr::ProtoCodec: call App::Run first");
    }
    Batch Decode(const std::vector<std::string>& frames) const { return run(frames, true); }
    // rows are padded with zero bytes to a multiple of 4
    Batch Encode(const std::vector<std::string>& rows) const { return run(rows, false); }

private:
    Batch run(const std::vector<std::string>& in, bool decode) const {
        std::string data;
        std::vector<uint32_t> off{0};
        for (auto& r : in) {
            data += r;
            if (!decode) data.append((4 - data.size() % 4) % 4, '\0');
            off.push_back((uint32_t)data.size());
        }
        const auto [pb, pr] = d_.bound(decode);
        const uint64_t cap = (uint64_t)pb * data.size() + (uint64_t)pr * in.size();
        std::vector<uint8_t> out(cap ? cap : 1);
        std::vector<uint32_t> out_off(in.size() + 1), meta(in.size() ? in.size() : 1);
        gofr_proto_batch b{reinterpret_cast<const uint8_t*>(data.data()), data.size(), off.data(), (uint32_t)in.size()};
        gofr_resp_batch rb{out.data(), cap, out_off.data(), meta.data(), 0};
        gofr_ticket t = 0;
        auto call = decode ? gofr_proto_batch_decode : gofr_proto_batch_encode;
        check(call(engine_, d_.msgs.data(), (uint32_t)d_.msgs.size(), d_.fields.data(), (uint32_t)d_.fields.size(), d_.root, d_.presence(),
                   &b, &rb, &t),
              decode ? "gofr_proto_batch_decode" : "gofr_proto_batch_encode");
        check(gofr_batch_wait(engine_, t), "gofr_batch_wait");
        Batch r;
        for (size_t i = 0; i < in.size(); i++) {
            r.records.emplace_back(reinterpret_cast<const char*>(out.data()) + out_off[i], out_off[i + 1] - out_off[i]);
            r.status.push_back(meta[i]);
        }
        return r;
    }

    gofr_engine* engine_;
    Description d_;
};

// grpc-go's codec one message at a time (gofr_proto_frontend_call): Call blocks until the batch the record joined has come
// back, so each RPC's thread calls it the way grpc-go calls encoding.Codec.Unmarshal / Marshal.  Decode: the message
// without its 5-byte prefix → the row; encode: a row (padded with zero bytes to a multiple of 4) → the marshalled message
// without the prefix.  One message type, one direction; any number of threads may call one ProtoFrontend.  Built from the
// same Field lists as ProtoCodec; the app must be running (App::Run).  An encode front-end made with log also writes the
// gRPC LoggingInterceptor's RPCLog line of each CallLog (gofr_proto_frontend_call_log), for methods of at most
// max_log_bytes bytes.
class ProtoFrontend {
public:
    using Field = ProtoCodec::Field;
    struct Result {
        int rc = GOFR_OK;      // GOFR_ERR_CAPACITY: the record exceeds max_record_bytes, nothing was queued (use the host codec)
        uint32_t status = 0;   // GOFR_GRPC_*: GOFR_GRPC_DEFER is for the host's own decoder
        std::string record;    // the row (decode) or the message (encode); empty where status is not GOFR_GRPC_OK
        std::string line;      // CallLog: the call's RPCLog line (empty for GOFR_LOG_NONE)
    };

    ProtoFrontend(const App& app, const std::vector<std::vector<Field>>& msgs, uint32_t root, bool decode, uint32_t max_batch = 1024,
                  uint32_t max_wait_us = 200, uint32_t max_record_bytes = 4096, bool log = false, uint32_t max_log_bytes = 256)
        : d_(msgs, root) {
        if (!app.engine()) throw std::logic_error("gofr::ProtoFrontend: call App::Run first");
        std::tie(per_byte_, per_record_) = d_.bound(decode);
        if (log)
            ProtoCodec::check(gofr_proto_frontend_create_log(&f_, app.engine(), d_.msgs.data(), (uint32_t)d_.msgs.size(), d_.fields.data(),
                                                             (uint32_t)d_.fields.size(), root, d_.presence(), decode ? 1 : 0,
                                                             max_batch, max_wait_us, max_record_bytes, max_log_bytes),
                              "gofr_proto_frontend_create_log");
        else
            ProtoCodec::check(gofr_proto_frontend_create(&f_, app.engine(), d_.msgs.data(), (uint32_t)d_.msgs.size(), d_.fields.data(),
                                                         (uint32_t)d_.fields.size(), root, d_.presence(), decode ? 1 : 0, max_batch,
                                                         max_wait_us, max_record_bytes),
                              "gofr_proto_frontend_create");
    }
    ~ProtoFrontend() { gofr_proto_frontend_destroy(f_); }
    ProtoFrontend(const ProtoFrontend&) = delete;
    ProtoFrontend& operator=(const ProtoFrontend&) = delete;

    Result Call(const std::string& in) const {
        Result r;
        // room for the bound of this record: the front-end never answers GOFR_ERR_CAPACITY for the output
        std::vector<uint8_t> out((size_t)per_byte_ * (in.size() + 5) + per_record_);
        uint32_t len = 0;
        r.rc = in.size() > UINT32_MAX ? GOFR_ERR_CAPACITY
                                      : gofr_proto_frontend_call(f_, reinterpret_cast<const uint8_t*>(in.data()), (uint32_t)in.size(),
                                                                 out.data(), (uint32_t)out.size(), &len, &r.status);
        if (r.rc == GOFR_ERR_CAPACITY) return r;
        ProtoCodec::check(r.rc, "gofr_proto_frontend_call");
        r.record.assign(reinterpret_cast<const char*>(out.data()), len);
        return r;
    }
    // Call plus the RPCLog line LoggingInterceptor writes once the handler has returned: `row` is the handler's response
    // (empty when it failed: the record is then to be ignored, the line is still written), `trace_id` the span's, `log` its
    // start_unix_ns, elapsed_ns, tz_offset_s and kind (GOFR_LOG_RPC, or GOFR_LOG_NONE for no line) and `method`
    // info.FullMethod.
    Result CallLog(const std::string& row, const std::array<uint8_t, 16>& trace_id, gofr_log_desc log, const std::string& method) const {
        Result r;
        std::vector<uint8_t> out((size_t)per_byte_ * (row.size() + 5) + per_record_);
        std::string line(320 + 7 * method.size(), '\0');  // gofr_batch_log_bound of the record: never too small
        uint32_t len = 0, line_len = 0;
        log.method_len = (uint16_t)method.size();
        r.rc = row.size() > UINT32_MAX || method.size() > UINT16_MAX
                   ? GOFR_ERR_CAPACITY
                   : gofr_proto_frontend_call_log(f_, reinterpret_cast<const uint8_t*>(row.data()), (uint32_t)row.size(), trace_id.data(),
                                                  &log, reinterpret_cast<const uint8_t*>(method.data()), out.data(), (uint32_t)out.size(),
                                                  &len, &r.status, reinterpret_cast<uint8_t*>(&line[0]), (uint32_t)line.size(), &line_len);
        if (r.rc == GOFR_ERR_CAPACITY) return r;
        ProtoCodec::check(r.rc, "gofr_proto_frontend_call_log");
        r.record.assign(reinterpret_cast<const char*>(out.data()), len);
        r.line.assign(line.data(), line_len);
        return r;
    }
    // pin the log time of every line (tests); 0 = wall clock
    void SetLogClock(int64_t unix_ns) const {
        ProtoCodec::check(gofr_proto_frontend_set_log_clock(f_, unix_ns), "gofr_proto_frontend_set_log_clock");
    }
    std::pair<uint64_t, uint64_t> Stats() const {
        uint64_t b = 0, n = 0;
        ProtoCodec::check(gofr_proto_frontend_stats(f_, &b, &n), "gofr_proto_frontend_stats");
        return {b, n};
    }

private:
    ProtoCodec::Description d_;
    uint32_t per_byte_ = 0, per_record_ = 0;
    gofr_proto_frontend* f_ = nullptr;
};

// net/http's conn.serve one read at a time (gofr_conn_frontend_serve): Serve takes the bytes a connection's thread holds (the
// kept tail plus its new read) and blocks until the batch it joined has been framed, parsed and answered on the GPU.  A
// request of a GOFR_H_HOST route (status 0 in meta) is a hole: the caller runs that route's closure and writes its response
// at the hole's place.  On GOFR_HTTP_CONN_MORE keep buf[consumed ..] and append the next read; on GOFR_HTTP_CONN_DEFER write
// the responses, then hand buf[consumed ..] to net/http.  Any number of threads may call one ConnFrontend, one call per
// connection at a time.  The engine serves `table`: fused routes and GOFR_H_HOST holes.  An App's routes are closures; serve
// them one read at a time with App::ServeRead.
class ConnFrontend {
public:
    struct Read {
        int rc = GOFR_OK;           // GOFR_ERR_CAPACITY: the read exceeds max_conn_bytes, nothing was queued (use net/http)
        std::string bytes;          // the responses back to back: request k's is bytes[out_off[k] .. out_off[k+1]), a hole's empty
        std::vector<uint32_t> out_off{0}, meta, req_at;  // meta as gofr_batch_submit's; req_at: the request's first byte in buf
        std::vector<std::array<uint8_t, 16>> trace_ids;  // each the bytes of its response's X-Correlation-Id
        uint32_t consumed = 0, conn_status = GOFR_HTTP_CONN_DONE;
        std::string log;            // with log: middleware.Logging's lines, line m = log[log_off[m] .. log_off[m+1]) for request log_req[m]
        std::vector<uint32_t> log_off{0}, log_req;
    };

    ConnFrontend(gofr_engine* engine, const gofr_table* table, uint32_t max_batch = 1024, uint32_t max_wait_us = 200,
                 uint32_t max_conn_bytes = 16384, bool log = false, int32_t tz_offset_s = 0, uint64_t seed = 0)
        : table_(table), max_conn_bytes_(max_conn_bytes), log_(log) {
        ProtoCodec::check(gofr_conn_frontend_create(&f_, engine, max_batch, max_wait_us, max_conn_bytes, log ? 1 : 0, tz_offset_s, seed),
                          "gofr_conn_frontend_create");
    }
    ~ConnFrontend() { gofr_conn_frontend_destroy(f_); }
    ConnFrontend(const ConnFrontend&) = delete;
    ConnFrontend& operator=(const ConnFrontend&) = delete;

    // remote: the connection's req.RemoteAddr (at most 255 bytes); start_unix_ns: Logging's start clock for this read
    Read Serve(const std::string& buf, const std::string& remote = std::string(), int64_t start_unix_ns = 0) const {
        Read r;
        if (buf.size() > max_conn_bytes_) { r.rc = GOFR_ERR_CAPACITY; return r; }
        // capacities that always suffice for this read: the front-end never answers GOFR_ERR_CAPACITY for them
        const uint32_t off[2] = {0, (uint32_t)buf.size()}, roff[2] = {0, (uint32_t)remote.size()};
        uint32_t req_cap = 0, line_cap = 0;
        uint64_t out_cap = 0, log_cap = 0;
        ProtoCodec::check(gofr_conn_batch_bound(table_, off, 1, &req_cap, &out_cap), "gofr_conn_batch_bound");
        if (log_) ProtoCodec::check(gofr_conn_log_bound(off, roff, 1, &line_cap, &log_cap), "gofr_conn_log_bound");
        r.bytes.resize(out_cap);
        r.out_off.resize(req_cap + 1);
        r.meta.resize(req_cap);
        r.req_at.resize(req_cap);
        r.trace_ids.resize(req_cap);
        r.log.resize(log_cap);
        r.log_off.resize(line_cap + 1);
        r.log_req.resize(line_cap);
        uint32_t first[2] = {0, 0};
        gofr_conn_resp o{};
        o.out = reinterpret_cast<uint8_t*>(&r.bytes[0]); o.out_cap = out_cap; o.req_cap = req_cap; o.out_off = r.out_off.data();
        o.meta = r.meta.data(); o.req_at = r.req_at.data(); o.trace_ids = r.trace_ids.empty() ? nullptr : r.trace_ids[0].data();
        o.req_first = first; o.consumed = &r.consumed; o.conn_status = &r.conn_status;
        gofr_conn_log l{};
        l.line_cap = line_cap; l.out = reinterpret_cast<uint8_t*>(&r.log[0]); l.out_cap = log_cap; l.log_off = r.log_off.data();
        l.log_req = r.log_req.data();
        r.rc = gofr_conn_frontend_serve(f_, reinterpret_cast<const uint8_t*>(buf.data()), (uint32_t)buf.size(),
                                        reinterpret_cast<const uint8_t*>(remote.data()), (uint32_t)remote.size(), start_unix_ns, &o,
                                        log_ ? &l : nullptr);
        ProtoCodec::check(r.rc, "gofr_conn_frontend_serve");
        const uint32_t n = first[1];
        r.bytes.resize(o.out_bytes);
        r.out_off.resize(n + 1);
        r.meta.resize(n);
        r.req_at.resize(n);
        r.trace_ids.resize(n);
        r.log.resize(log_ ? l.out_bytes : 0);
        r.log_off.resize((log_ ? l.lines : 0) + 1);
        r.log_req.resize(log_ ? l.lines : 0);
        return r;
    }
    // pin the Date header and the log time of every batch (tests); 0 = wall clock
    void SetClock(int64_t unix_ns) { ProtoCodec::check(gofr_conn_frontend_set_clock(f_, unix_ns), "gofr_conn_frontend_set_clock"); }
    // batches, connection reads served, batches served again after their outputs grew
    std::array<uint64_t, 3> Stats() const {
        std::array<uint64_t, 3> s{};
        ProtoCodec::check(gofr_conn_frontend_stats(f_, &s[0], &s[1], &s[2]), "gofr_conn_frontend_stats");
        return s;
    }

private:
    const gofr_table* table_;
    uint32_t max_conn_bytes_;
    bool log_;
    gofr_conn_frontend* f_ = nullptr;
};

}  // namespace gofr
