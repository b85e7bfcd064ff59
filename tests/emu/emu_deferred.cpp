// emu_deferred.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the second pass of the nested proto3 decoder (gofr_b200/csrc/proto_nested_deferred_device.cuh, the same
// __host__ __device__ functions proto_nested_deferred_kernel.cu calls) on the CPU: the walk with the sorted-list map step,
// executed as a CTA of one thread, so the lists are collected, bitonic-sorted and compacted on the CPU by the device code
// itself.  The tile loop, place_tile and the look-back only exist in the kernel and are covered by the `-m gpu` test.
// Nothing in the product links or loads this file.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../gofr_b200/csrc/proto_nested_deferred_device.cuh"

using namespace gofr;

// frames whose meta_in word is GOFR_GRPC_DEFER are decoded again; the others get an empty row and keep their status.
// desc: the PbnDesc the product's gofr_proto_nested_describe_ex built.  Returns -1 when rows_cap is too small.
extern "C" int emu_proto_decode_nested_deferred(const void* desc, const uint8_t* in, const uint32_t* in_off, uint32_t n,
                                                const uint32_t* meta_in, uint8_t* rows, uint64_t rows_cap, uint32_t* row_off,
                                                uint32_t* meta) {
    PbnDesc D;
    memcpy(&D, desc, sizeof D);
    std::vector<PdnSortMem> lists(1);
    pdn_host_sort_mem = lists.data();
    uint64_t pos = 0;
    int rc = 0;
    for (uint32_t i = 0; i < n && !rc; i++) {
        const uint8_t* f = in + in_off[i];
        const uint32_t fn = in_off[i + 1] - in_off[i];
        PdnRow r = {meta_in[i], 0};
        if (meta_in[i] == GOFR_GRPC_DEFER) r = pdn_deferred_size(D, f, fn);
        row_off[i] = (uint32_t)pos;
        meta[i] = r.status;
        if (pos + r.out_len > rows_cap) { rc = -1; break; }
        pdn_deferred_emit(D, f, fn, r, rows + pos);
        pos += r.out_len;
    }
    row_off[n] = (uint32_t)pos;
    pdn_host_sort_mem = nullptr;
    return rc;
}
extern "C" uint32_t emu_deferred_desc_bytes() { return (uint32_t)sizeof(PbnDesc); }
