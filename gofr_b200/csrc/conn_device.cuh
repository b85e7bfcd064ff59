// conn_device.cuh — per-connection logic of gofr_conn_batch_submit's compact step (conn_kernel.cu), compiled for the device
// and, through tests/emu/emu_conn.cpp, for the host.
//
// After the framer and the request-head kernel, record r of a chunk is one request of a connection, or that connection's tail
// (the last record of a MORE / DEFER connection).  A tail's zero descriptor is a GET of an empty path (GOFR_M_GET == 0), which
// the serve kernel would answer: so the tails are dropped BEFORE serving, by copying every connection's whole requests to its
// place in a compacted column — descriptor, first byte in the buffer and trace id.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/gofr_b200.h"

#if defined(__CUDACC__)
#define GOFR_CONN_HD __host__ __device__ __forceinline__
#else
#define GOFR_CONN_HD inline
#endif

namespace gofr {

GOFR_CONN_HD uint64_t conn_splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// The trace id of request j of connection c (include/gofr_b200.h, gofr_conn_batch_submit): two splitmix64 draws keyed by
// (seed, c, j), stored little-endian.  `key` is conn_trace_key(seed, c), computed once per connection.
GOFR_CONN_HD uint64_t conn_trace_key(uint64_t seed, uint32_t c) { return conn_splitmix64(seed ^ conn_splitmix64((uint64_t)c)); }
// The key of the chunk's connection i, batch connection conn0 + i: keys[i] when the caller gave a key column
// (gofr_conn_batch_respond_ex), else conn_trace_key(seed, conn0 + i).
GOFR_CONN_HD uint64_t conn_key(const uint64_t* keys, uint64_t seed, uint32_t conn0, uint32_t i) {
    return keys ? keys[i] : conn_trace_key(seed, conn0 + i);
}
GOFR_CONN_HD void conn_trace_id(uint64_t key, uint32_t j, uint8_t* out16) {
    const uint64_t lo = conn_splitmix64(key + 2ull * j), hi = conn_splitmix64(key + 2ull * j + 1ull);
    memcpy(out16, &lo, 8);
    memcpy(out16 + 8, &hi, 8);
}

// Whole requests of connection c of a framed chunk: its records minus the tail
GOFR_CONN_HD uint32_t conn_requests(const uint32_t* first, const uint32_t* conn_status, uint32_t c) {
    return first[c + 1] - first[c] - (conn_status[c] != GOFR_HTTP_CONN_DONE ? 1u : 0u);
}

// Copies the `count` whole requests of a connection, records rec0 .. rec0 + count, to compacted places k0 .. k0 + count:
// descriptor (its arena offset stays valid: the arena is not moved), first byte (the record's start) and trace id.
GOFR_CONN_HD void conn_put(const gofr_req_desc* desc_in, const uint32_t* rec_off, uint32_t rec0, uint32_t count, uint64_t key,
                           gofr_req_desc* desc_out, uint32_t* req_at, uint8_t* ids, uint32_t k0) {
    for (uint32_t j = 0; j < count; j++) {
        desc_out[k0 + j] = desc_in[rec0 + j];
        req_at[k0 + j] = rec_off[rec0 + j];
        conn_trace_id(key, j, ids + (size_t)(k0 + j) * 16);
    }
}

}  // namespace gofr
