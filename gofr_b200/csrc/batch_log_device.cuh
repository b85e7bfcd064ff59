// batch_log_device.cuh — which request of a host batch gets middleware.Logging's line from gofr_batch_submit_log, and the
// fields of its record the call fills.  Compiled for the device (batch_log_kernel.cu) and, through
// tests/emu/emu_batch_log.cpp, for the host.
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

}  // namespace gofr
