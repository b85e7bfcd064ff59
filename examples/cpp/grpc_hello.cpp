// The reference's gRPC example, Server.SayHello (examples/grpc-server/grpc/server.go), on a batch of unary calls through
// the C++ stand-in of the app API: request frames → gofr::ProtoCodec::Decode (GPU) → the handler on the host →
// gofr::ProtoCodec::Encode (GPU) → response frames.  The batch is the three cases of the reference's TestServer_SayHello
// (examples/grpc-server/grpc/server_test.go).  Prints one line per case — "<message>\t<response frame in hex>" — which
// tests/test_proto_batch.py compares with python protobuf; exits non-zero when a response is not what the test expects.
//   g++ -std=c++17 -Iinclude examples/cpp/grpc_hello.cpp gofr_b200/libgofr_b200.so -o grpc_hello
#include <cstdio>
#include <string>
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
// proto.Marshal(&HelloRequest{Name: name}) behind grpc-go's 5-byte prefix (the name is shorter than 128 bytes)
static std::string request_frame(const std::string& name) {
    std::string body = name.empty() ? std::string() : std::string("\x0a", 1) + (char)name.size() + name;
    const uint32_t n = (uint32_t)body.size();
    std::string f(1, '\0');
    for (int k = 3; k >= 0; k--) f += (char)((n >> (8 * k)) & 0xFF);
    return f + body;
}

// Server.SayHello
static std::string SayHello(std::string name) {
    if (name.empty()) name = "World";
    return "Hello " + name + "!";
}

int main() {
    gofr::App app;
    app.Run();
    using F = gofr::ProtoCodec::Field;
    const gofr::ProtoCodec request(app, {{F{1, GOFR_PB_STRING}}}, 0), response(app, {{F{1, GOFR_PB_STRING}}}, 0);

    struct Case { std::string input, resp; };
    const std::vector<Case> tests = {{"world", "Hello world!"}, {"123", "Hello 123!"}, {"", "Hello World!"}};
    std::vector<std::string> frames;
    for (auto& tc : tests) frames.push_back(request_frame(tc.input));

    const gofr::ProtoCodec::Batch in = request.Decode(frames);
    std::vector<std::string> rows;
    for (size_t i = 0; i < tests.size(); i++) {
        if (in.status[i] != GOFR_GRPC_OK) { fprintf(stderr, "TEST[%zu], Failed: request status %u\n", i, in.status[i]); return 1; }
        rows.push_back(row_of(SayHello(string_of(in.records[i]))));
    }
    const gofr::ProtoCodec::Batch out = response.Encode(rows);

    int failed = 0;
    for (size_t i = 0; i < tests.size(); i++) {
        const std::string& f = out.records[i];
        // the frame carries one string field: prefix, tag 0x0a, a one-byte length, the message
        const std::string msg = f.size() > 7 ? f.substr(7) : std::string();
        if (out.status[i] != GOFR_GRPC_OK || msg != tests[i].resp) {
            fprintf(stderr, "TEST[%zu], Failed: got \"%s\", want \"%s\"\n", i, msg.c_str(), tests[i].resp.c_str());
            failed = 1;
        }
        printf("%s\t", msg.c_str());
        for (unsigned char c : f) printf("%02x", c);
        printf("\n");
    }
    return failed;
}
