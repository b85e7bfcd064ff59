// The reference's gRPC example, Server.SayHello (examples/grpc-server/grpc/server.go), served one RPC at a time from many
// threads, the way grpc-go runs a unary handler on each RPC's goroutine: the request message → gofr::ProtoFrontend decode
// (encoding.Codec.Unmarshal, GPU) → the handler on the host → gofr::ProtoFrontend encode (Marshal, GPU) → the response
// message.  The front-ends batch whatever the threads hand in at the same time.  The calls are the three cases of the
// reference's TestServer_SayHello (examples/grpc-server/grpc/server_test.go) followed by generated names.  Prints one line
// per call — "<message>\t<marshalled HelloResponse in hex>" — which tests/test_proto_frontend.py compares with python
// protobuf; exits non-zero when a response is not what the handler returned.  With a log path, the server also logs as GoFr's
// LoggingInterceptor does (pkg/gofr/grpc/log.go:27-50): each call's span gets a trace id and the handler is timed on its
// thread, and the encode front-end writes the call's RPCLog line for method /Hello/SayHello beside its message
// (gofr::ProtoFrontend::CallLog).  The lines go to that file in call order.
//   g++ -std=c++17 -pthread -Iinclude examples/cpp/grpc_server.cpp gofr_b200/libgofr_b200.so -o grpc_server
//   grpc_server [threads] [calls per thread] [log path]
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "gofr_b200.hpp"

// HelloRequest { string name = 1; } and HelloResponse { string message = 1; } (hello.proto): one string field each, so a
// row is the string's length word followed by its bytes
static std::string row_of(const std::string& s) {
    std::string row;
    const uint32_t n = (uint32_t)s.size();
    row.append(reinterpret_cast<const char*>(&n), 4);
    return row + s;
}
static std::string string_of(const std::string& row) {
    uint32_t n = 0;
    memcpy(&n, row.data(), 4);
    return row.substr(4, n);
}
// proto.Marshal(&HelloRequest{Name: name}), for names shorter than 128 bytes: what grpc-go hands to Unmarshal
static std::string request_message(const std::string& name) {
    return name.empty() ? std::string() : std::string("\x0a", 1) + (char)name.size() + name;
}

// Server.SayHello
static std::string SayHello(std::string name) {
    if (name.empty()) name = "World";
    return "Hello " + name + "!";
}

static int64_t unix_ns() {
    return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::system_clock::now().time_since_epoch()).count();
}

int main(int argc, char** argv) {
    const int threads = argc > 1 ? atoi(argv[1]) : 8, per_thread = argc > 2 ? atoi(argv[2]) : 25;
    const char* log_path = argc > 3 ? argv[3] : nullptr;
    gofr::App app;
    app.Run();
    using F = gofr::ProtoFrontend::Field;
    const gofr::ProtoFrontend unmarshal(app, {{F{1, GOFR_PB_STRING}}}, 0, true, 64, 200, 256);
    const gofr::ProtoFrontend marshal(app, {{F{1, GOFR_PB_STRING}}}, 0, false, 64, 200, 256, log_path != nullptr);
    // time.Local's offset, as the logger's time.Time values carry it
    const time_t now = time(nullptr);
    struct tm local;
    localtime_r(&now, &local);
    const int32_t tz_offset_s = (int32_t)local.tm_gmtoff;

    struct Case { std::string input, resp; };
    std::vector<Case> tests = {{"world", "Hello world!"}, {"123", "Hello 123!"}, {"", "Hello World!"}};
    for (int k = (int)tests.size(); k < threads * per_thread; k++) {
        const std::string name = "caller-" + std::to_string(k) + std::string((size_t)(k % 40), (char)('a' + k % 26));
        tests.push_back({name, "Hello " + name + "!"});
    }
    std::vector<std::string> lines(tests.size()), log_lines(tests.size());
    std::mutex mu;
    int failed = 0;
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++)
        th.emplace_back([&, t] {
            for (size_t i = (size_t)t; i < tests.size(); i += (size_t)threads) {
                const gofr::ProtoFrontend::Result in = unmarshal.Call(request_message(tests[i].input));
                std::string msg, bytes, log_line;
                uint32_t status = in.status;
                if (in.rc == GOFR_OK && in.status == GOFR_GRPC_OK) {
                    // the interceptor's span and clock around the handler
                    std::array<uint8_t, 16> trace_id{};
                    for (int k = 0; k < 8; k++) trace_id[15 - k] = (uint8_t)((uint64_t)(i + 1) >> (8 * k));
                    const int64_t start = unix_ns();
                    msg = SayHello(string_of(in.record));
                    gofr_log_desc rec{};
                    rec.start_unix_ns = start; rec.elapsed_ns = unix_ns() - start; rec.tz_offset_s = tz_offset_s; rec.kind = GOFR_LOG_RPC;
                    const gofr::ProtoFrontend::Result out =
                        log_path ? marshal.CallLog(row_of(msg), trace_id, rec, "/Hello/SayHello") : marshal.Call(row_of(msg));
                    status = out.rc == GOFR_OK ? out.status : 0x100u | (uint32_t)out.rc;
                    bytes = out.record;
                    log_line = out.line;
                }
                // the message carries one string field: tag 0x0a, a one-byte length, the text
                const std::string got = bytes.size() > 2 ? bytes.substr(2) : std::string();
                std::string line = msg + "\t";
                for (unsigned char c : bytes) { char h[3]; snprintf(h, sizeof h, "%02x", c); line += h; }
                std::lock_guard<std::mutex> g(mu);
                if (status != GOFR_GRPC_OK || got != tests[i].resp) {
                    fprintf(stderr, "TEST[%zu], Failed: status %u, got \"%s\", want \"%s\"\n", i, status, got.c_str(), tests[i].resp.c_str());
                    failed = 1;
                }
                lines[i] = line;
                log_lines[i] = log_line;
            }
        });
    for (auto& x : th) x.join();
    for (auto& l : lines) printf("%s\n", l.c_str());
    if (log_path) {
        FILE* f = fopen(log_path, "wb");
        if (!f) { perror(log_path); return 1; }
        for (auto& l : log_lines) fwrite(l.data(), 1, l.size(), f);  // each line ends in '\n'
        fclose(f);
    }
    const auto [batches, calls] = unmarshal.Stats();
    fprintf(stderr, "%llu requests decoded in %llu batches\n", (unsigned long long)calls, (unsigned long long)batches);
    return failed;
}
