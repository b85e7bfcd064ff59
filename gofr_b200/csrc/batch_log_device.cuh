// batch_log_device.cuh — which record of a host batch gets a log line from the calls that write one (gofr_batch_submit_log:
// middleware.Logging's line; gofr_proto_batch_encode_log: the gRPC LoggingInterceptor's), and the fields of its record the
// call fills.  Compiled for the device (batch_log_kernel.cu, proto_log_kernel.cu) and, through tests/emu/emu_batch_log.cpp
// and tests/emu/emu_proto_log.cpp, for the host.
#pragma once
#include <stdint.h>

#include "../../include/gofr_b200.h"
#include "engine_internal.h"

namespace gofr {

// Request i has a line exactly when a matched route answered it (gorilla/mux wraps middleware around matched routes only:
// its cleanPath 301 and own 404 / 405 carry GOFR_ROUTE_NONE), it has a status (a GOFR_H_HOST hole is logged by the call
// that serves its closure's result) and the caller asked for one.
GOFR_INTERNAL_HD bool batch_logged(uint32_t meta, uint32_t kind) {
    return (meta >> 16) != GOFR_ROUTE_NONE && (meta & 0xFFFFu) != 0 && kind == GOFR_LOG_REQUEST;
}

// The serve kernel's meta of the request and the batch's clock into its record: whether it has a line, and when it does,
// its status, log time and elapsed time as the connection path computes them.
GOFR_INTERNAL_HD bool batch_log_fill(gofr_log_desc& d, uint32_t meta, int64_t log_ns) {
    if (!batch_logged(meta, d.kind)) return false;
    d.status = (uint16_t)(meta & 0xFFFFu);
    d.log_unix_ns = log_ns;
    d.elapsed_ns = log_ns - d.start_unix_ns;
    return true;
}

// Call i of an encode batch has a line exactly when the caller asked for one: LoggingInterceptor logs in its deferred
// function (grpc/log.go:27-50), after the handler, whether or not the handler failed and before grpc-go marshals anything,
// so neither the response row nor its encoding decides.  Its log time is the batch's; elapsed_ns is the caller's, who
// measured time.Since(start) on the handler's own thread.
GOFR_INTERNAL_HD bool proto_log_fill(gofr_log_desc& d, int64_t log_ns) {
    if (d.kind != GOFR_LOG_RPC) return false;
    d.log_unix_ns = log_ns;
    return true;
}

}  // namespace gofr
