// Package gofrb200 binds libgofr_b200.so (include/gofr_b200.h) over cgo.
//
// UNVERIFIED SOURCE: there is no Go toolchain in the build image or on the GPU box, so this file has never been
// compiled.  It shows the exact binding a GoFr maintainer would add; every C call is one declared in
// include/gofr_b200.h.  The C++/Python harnesses in this repository exercise the same ABI.
//
// How it plugs into GoFr (reference paths):
//   - App.add (pkg/gofr/gofr.go:171-177) additionally calls Table.AddRoute with the declarative handler kind (or
//     HHost for an arbitrary closure);
//   - App.Run (pkg/gofr/gofr.go:90-126) calls Table.AddDefaultRoutes, Table.Seal and NewEngine instead of
//     httpServer.Run, and starts a Batcher that collects parsed requests from the connection goroutines;
//   - the Batcher hands batches to Engine.Serve and fans the response bytes back to the connections.
package gofrb200

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../gofr_b200 -lgofr_b200 -Wl,-rpath,${SRCDIR}/../../gofr_b200
#include <stdlib.h>
#include "gofr_b200.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"time"
	"unsafe"
)

// Method codes: mux compares exact upper-case method strings, everything else is MOther.
const (
	MGet = iota
	MHead
	MPost
	MPut
	MPatch
	MDelete
	MConnect
	MOptions
	MTrace
	MOther = 15
)

var methodCodes = map[string]uint8{"GET": MGet, "HEAD": MHead, "POST": MPost, "PUT": MPut, "PATCH": MPatch,
	"DELETE": MDelete, "CONNECT": MConnect, "OPTIONS": MOptions, "TRACE": MTrace}

func MethodCode(m string) uint8 {
	if c, ok := methodCodes[m]; ok {
		return c
	}
	return MOther
}

func check(rc C.int, where string) error {
	if rc == 0 {
		return nil
	}
	return fmt.Errorf("%s: gofr error %d: %s", where, int(rc), C.GoString(C.gofr_last_error()))
}

// Table mirrors the route slice of mux.Router: routes in registration order, frozen by Seal.
type Table struct{ t *C.gofr_table }

func NewTable(frameMode uint32) (*Table, error) {
	var t *C.gofr_table
	if err := check(C.gofr_table_create(&t, C.uint32_t(frameMode)), "gofr_table_create"); err != nil {
		return nil, err
	}
	return &Table{t}, nil
}

// Handler is the declarative description of a gofr.Handler closure (GOFR_H_* in the header).
type Handler struct {
	Kind     uint32
	SchemaID uint32
	S0, S1   string
	S2, S3   string
	Blob     []byte
}

func (t *Table) AddRoute(method string, pattern string, h Handler) (uint32, error) {
	var d C.gofr_handler_desc
	d.kind = C.uint32_t(h.Kind)
	d.schema_id = C.uint32_t(h.SchemaID)
	cs := func(s string) (*C.char, C.uint32_t) { return C.CString(s), C.uint32_t(len(s)) }
	d.s0, d.s0_len = cs(h.S0)
	d.s1, d.s1_len = cs(h.S1)
	d.s2, d.s2_len = cs(h.S2)
	d.s3, d.s3_len = cs(h.S3)
	defer func() {
		C.free(unsafe.Pointer(d.s0)); C.free(unsafe.Pointer(d.s1)); C.free(unsafe.Pointer(d.s2)); C.free(unsafe.Pointer(d.s3))
	}()
	if len(h.Blob) > 0 {
		d.blob = (*C.uint8_t)(unsafe.Pointer(&h.Blob[0]))
		d.blob_len = C.uint32_t(len(h.Blob))
	}
	p := C.CString(pattern)
	defer C.free(unsafe.Pointer(p))
	var id C.uint32_t
	m := C.uint32_t(MethodCode(method))
	err := check(C.gofr_table_add_route(t.t, m, p, C.uint32_t(len(pattern)), &d, &id), "gofr_table_add_route")
	return uint32(id), err
}

func (t *Table) AddDefaultRoutes(favicon []byte) error {
	var p *C.uint8_t
	if len(favicon) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&favicon[0]))
	}
	return check(C.gofr_table_add_default_routes(t.t, p, C.uint32_t(len(favicon))), "gofr_table_add_default_routes")
}

func (t *Table) Seal() error { return check(C.gofr_table_seal(t.t), "gofr_table_seal") }

// Engine is one GPU.
type Engine struct{ e *C.gofr_engine }

func NewEngine(t *Table, device int) (*Engine, error) {
	var e *C.gofr_engine
	if err := check(C.gofr_engine_create(&e, t.t, C.int(device)), "gofr_engine_create"); err != nil {
		return nil, err
	}
	return &Engine{e}, nil
}

// Batch is the pinned SoA staging area one batch of parsed requests is appended to by the connection goroutines.
type Batch struct {
	Desc     []C.gofr_req_desc // n
	TraceIDs []byte            // n*16
	Arena    []byte
}

// Serve runs one batch through the GPU.  out/off/meta are caller-owned (ideally from gofr_alloc_pinned).
func (e *Engine) Serve(b *Batch, now time.Time, out []byte, off, meta []uint32) (int, error) {
	n := len(b.Desc)
	if n == 0 {
		return 0, nil
	}
	if len(off) < n+1 || len(meta) < n {
		return 0, errors.New("gofrb200: off/meta too small")
	}
	var in C.gofr_req_batch
	in.desc = &b.Desc[0]
	in.trace_ids = (*C.uint8_t)(unsafe.Pointer(&b.TraceIDs[0]))
	in.arena = (*C.uint8_t)(unsafe.Pointer(&b.Arena[0]))
	in.arena_bytes = C.uint64_t(len(b.Arena))
	in.n = C.uint32_t(n)
	C.gofr_format_http_date(C.int64_t(now.Unix()), &in.date[0])
	var o C.gofr_resp_batch
	o.out = (*C.uint8_t)(unsafe.Pointer(&out[0]))
	o.out_cap = C.uint64_t(len(out))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&off[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&meta[0]))
	var ticket C.gofr_ticket
	if err := check(C.gofr_batch_submit(e.e, &in, &o, &ticket), "gofr_batch_submit"); err != nil {
		return 0, err
	}
	if err := check(C.gofr_batch_wait(e.e, ticket), "gofr_batch_wait"); err != nil {
		return 0, err
	}
	return int(o.out_bytes), nil
}

// LogRecord is what middleware.Logging's deferred function reads from the clock and the request
// (pkg/gofr/http/middleware/logger.go:49-63); Append packs it as one gofr_log_desc plus its strings.
type LogBatch struct {
	Desc     []C.gofr_log_desc
	TraceIDs []byte // 16 bytes per record
	Arena    []byte // method | user_agent | x_forwarded_for | remote_addr | request_uri per record
}

func (b *LogBatch) Append(start time.Time, elapsed time.Duration, now time.Time, traceID [16]byte, method, userAgent, xff,
	remoteAddr, requestURI string, status int) {
	_, off := start.Zone()
	var d C.gofr_log_desc
	d.start_unix_ns = C.int64_t(start.UnixNano())
	d.elapsed_ns = C.int64_t(elapsed.Nanoseconds())
	d.log_unix_ns = C.int64_t(now.UnixNano())
	d.arena_off = C.uint32_t(len(b.Arena))
	d.method_len, d.ua_len, d.xff_len = C.uint16_t(len(method)), C.uint16_t(len(userAgent)), C.uint16_t(len(xff))
	d.remote_len, d.uri_len = C.uint16_t(len(remoteAddr)), C.uint16_t(len(requestURI))
	d.status = C.uint16_t(status)
	d.tz_offset_s = C.int32_t(off)
	d.kind = C.GOFR_LOG_REQUEST
	b.Desc = append(b.Desc, d)
	b.TraceIDs = append(b.TraceIDs, traceID[:]...)
	b.Arena = append(append(append(append(append(b.Arena, method...), userAgent...), xff...), remoteAddr...), requestURI...)
}

// AppendRPC packs what GoFr's gRPC LoggingInterceptor reads for one call (pkg/gofr/grpc/log.go:27-50): its start, the
// handler's time.Since(start), the span's trace id and info.FullMethod.  The record asks for an RPCLog line
// (GOFR_LOG_RPC); ProtoEncodeBatchLog fills its log time.
func (b *LogBatch) AppendRPC(start time.Time, elapsed time.Duration, traceID [16]byte, method string) {
	_, off := start.Zone()
	var d C.gofr_log_desc
	d.start_unix_ns = C.int64_t(start.UnixNano())
	d.elapsed_ns = C.int64_t(elapsed.Nanoseconds())
	d.arena_off = C.uint32_t(len(b.Arena))
	d.method_len = C.uint16_t(len(method))
	d.tz_offset_s = C.int32_t(off)
	d.kind = C.GOFR_LOG_RPC
	b.Desc = append(b.Desc, d)
	b.TraceIDs = append(b.TraceIDs, traceID[:]...)
	b.Arena = append(b.Arena, method...)
}

// SubmitLog serves one batch like Serve and writes middleware.Logging's line for each request in the same call
// (gofr_batch_submit_log): log holds one record per request of b, appended with Append, whose status and clocks the call
// fills from the response and from now; request i's line is lines[logOff[i]:logOff[i+1]], empty when mux answered it
// without middleware (301 / 404 / 405) or it is a GOFR_H_HOST hole.  logOff needs len(b.Desc)+1 entries; a short lines
// buffer is gofr_batch_wait's GOFR_ERR_CAPACITY (gofr_batch_log_bound sizes it).  Returns the response and line bytes.
func (e *Engine) SubmitLog(b *Batch, log *LogBatch, now time.Time, out []byte, off, meta []uint32, lines []byte,
	logOff []uint32) (int, int, error) {
	n := len(b.Desc)
	if n == 0 {
		return 0, 0, nil
	}
	if len(off) < n+1 || len(meta) < n || len(log.Desc) != n || len(logOff) < n+1 || len(lines) == 0 {
		return 0, 0, errors.New("gofrb200: SubmitLog columns too small")
	}
	var in C.gofr_req_batch
	in.desc = &b.Desc[0]
	in.trace_ids = (*C.uint8_t)(unsafe.Pointer(&b.TraceIDs[0]))
	in.arena = (*C.uint8_t)(unsafe.Pointer(&b.Arena[0]))
	in.arena_bytes = C.uint64_t(len(b.Arena))
	in.n = C.uint32_t(n)
	C.gofr_format_http_date(C.int64_t(now.Unix()), &in.date[0])
	var o C.gofr_resp_batch
	o.out = (*C.uint8_t)(unsafe.Pointer(&out[0]))
	o.out_cap = C.uint64_t(len(out))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&off[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&meta[0]))
	var l C.gofr_batch_log
	l.desc = &log.Desc[0]
	if len(log.Arena) > 0 {
		l.arena = (*C.uint8_t)(unsafe.Pointer(&log.Arena[0]))
	}
	l.arena_bytes = C.uint64_t(len(log.Arena))
	l.log_unix_ns = C.int64_t(now.UnixNano())
	l.out = (*C.uint8_t)(unsafe.Pointer(&lines[0]))
	l.out_cap = C.uint64_t(len(lines))
	l.log_off = (*C.uint32_t)(unsafe.Pointer(&logOff[0]))
	var ticket C.gofr_ticket
	if err := check(C.gofr_batch_submit_log(e.e, &in, &o, &l, &ticket), "gofr_batch_submit_log"); err != nil {
		return 0, 0, err
	}
	if err := check(C.gofr_batch_wait(e.e, ticket), "gofr_batch_wait"); err != nil {
		return 0, 0, err
	}
	return int(o.out_bytes), int(l.out_bytes), nil
}

// RequestLogDevice runs gofr_requestlog_device on buffers that already live in device memory (the batcher uploads the
// LogBatch next to the request batch); lines come back packed, line i = out[off[i]:off[i+1]].
func (e *Engine) RequestLogDevice(dDesc, dTraceIDs, dArena unsafe.Pointer, n int, dOut unsafe.Pointer, outCap uint64,
	dOff unsafe.Pointer, stream unsafe.Pointer) error {
	return check(C.gofr_requestlog_device(e.e, (*C.gofr_log_desc)(dDesc), (*C.uint8_t)(dTraceIDs), (*C.uint8_t)(dArena),
		C.uint32_t(n), (*C.uint8_t)(dOut), C.uint64_t(outCap), (*C.uint32_t)(dOff), stream), "gofr_requestlog_device")
}

// RouteDevice is stage 1 of the split API for closures that stay in Go: routing decisions and mux.Vars spans for a
// batch resident in device memory (gofr_route_device).  meta[i] = status | route << 16; status 0 = run handler `route`.
func (e *Engine) RouteDevice(dDesc, dArena unsafe.Pointer, n int, dMeta, dVars unsafe.Pointer, stream unsafe.Pointer) error {
	return check(C.gofr_route_device(e.e, (*C.gofr_req_desc)(dDesc), (*C.uint8_t)(dArena), C.uint32_t(n), (*C.uint32_t)(dMeta),
		(*C.uint32_t)(dVars), stream), "gofr_route_device")
}

// BindDevice is Context.Bind as a GPU stage for closures that stay in Go (gofr_bind_device): body i (the data section of
// request i) is decoded with encoding/json's rules into a row of schema schemaID (status 0), or into err.Error() (status 1),
// in slot i of dRows; status 2 = decide on the host.  pkg/gofr/context.go:52-54, pkg/gofr/http/request.go:40-47.
func (e *Engine) BindDevice(schemaID uint32, dDesc, dArena unsafe.Pointer, n int, dRows unsafe.Pointer, slotBytes uint32,
	dLen, dStatus unsafe.Pointer, stream unsafe.Pointer) error {
	return check(C.gofr_bind_device(e.e, C.uint32_t(schemaID), (*C.gofr_req_desc)(dDesc), (*C.uint8_t)(dArena), C.uint32_t(n),
		(*C.uint8_t)(dRows), C.uint32_t(slotBytes), (*C.uint32_t)(dLen), (*C.uint32_t)(dStatus), stream), "gofr_bind_device")
}

// BindHostThread pins the calling OS thread (runtime.LockOSThread first) to the CPUs and memory of the NUMA node the GPU
// hangs off; call it before AllocPinned and before the goroutines that fill batches are started (gofr_bind_host_thread).
func BindHostThread(device int) (numaNode int, err error) {
	var node C.int
	err = check(C.gofr_bind_host_thread(C.int(device), &node), "gofr_bind_host_thread")
	return int(node), err
}

// ServeDeviceSlots writes response i into its own slotBytes-sized, 16-byte aligned slot of dOut and its length into
// dOutLen[i] (gofr_serve_device_slots): the layout a ring of fixed-size response buffers maps onto directly.
func (e *Engine) ServeDeviceSlots(dDesc, dTraceIDs, dArena unsafe.Pointer, n int, now time.Time, dOut unsafe.Pointer,
	slotBytes uint32, dOutLen, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	var date [29]C.char
	C.gofr_format_http_date(C.int64_t(now.Unix()), &date[0])
	return check(C.gofr_serve_device_slots(e.e, (*C.gofr_req_desc)(dDesc), (*C.uint8_t)(dTraceIDs), (*C.uint8_t)(dArena),
		C.uint32_t(n), &date[0], (*C.uint8_t)(dOut), C.uint32_t(slotBytes), (*C.uint32_t)(dOutLen), (*C.uint32_t)(dMeta), stream),
		"gofr_serve_device_slots")
}

// HTTPParseDevice turns raw HTTP/1.1 request messages (back to back in dRaw, message i = dRaw[off[i]:off[i+1]]) into
// request descriptors + arena for the serve calls (gofr_http_parse_device).  status[i] != 0 (GOFR_HTTP_DEFER): hand
// that connection's bytes to net/http as before.
func (e *Engine) HTTPParseDevice(dRaw, dRawOff unsafe.Pointer, n int, dDesc, dArena, dStatus, dSpans unsafe.Pointer,
	stream unsafe.Pointer) error {
	return check(C.gofr_http_parse_device(e.e, (*C.uint8_t)(dRaw), (*C.uint32_t)(dRawOff), C.uint32_t(n), (*C.gofr_req_desc)(dDesc),
		(*C.uint8_t)(dArena), (*C.uint32_t)(dStatus), (*C.uint64_t)(dSpans), stream), "gofr_http_parse_device")
}

// Connection statuses of HTTPFrameDevice (GOFR_HTTP_CONN_*).
const (
	HTTPConnDone  = 0 // every byte belongs to a whole request
	HTTPConnMore  = 1 // the last record is the beginning of a request: keep it and append the next read
	HTTPConnDefer = 2 // the last record starts with a request outside the subset: hand the bytes from consumed on to net/http
)

// HTTPFrameDevice cuts connection receive buffers (connection c = dBuf[off[c]:off[c+1]]) into the record column
// HTTPParseDevice takes as dRawOff (gofr_http_frame_device): a connection's whole requests in order, then one tail record
// when bytes are left over.  Connection c owns records dFirst[c] .. dFirst[c+1]; dFirst[nConns] is the record count.
func (e *Engine) HTTPFrameDevice(dBuf, dBufOff unsafe.Pointer, nConns int, dRecOff unsafe.Pointer, recCap int, dFirst, dConsumed,
	dConnStatus unsafe.Pointer, stream unsafe.Pointer) error {
	return check(C.gofr_http_frame_device(e.e, (*C.uint8_t)(dBuf), (*C.uint32_t)(dBufOff), C.uint32_t(nConns), (*C.uint32_t)(dRecOff),
		C.uint32_t(recCap), (*C.uint32_t)(dFirst), (*C.uint32_t)(dConsumed), (*C.uint32_t)(dConnStatus), stream), "gofr_http_frame_device")
}

// ConnResponses receives what ServeConnections returns; the caller owns the slices (ideally from gofr_alloc_pinned) and
// sizes them with ConnBound.  Request k's response is Out[OutOff[k]:OutOff[k+1]]; connection c owns requests
// ReqFirst[c] .. ReqFirst[c+1].  TraceIDs may be nil.  With Log set, ServeConnections also writes middleware.Logging's
// lines for the requests answered on the device (gofr_conn_batch_submit_log).
type ConnResponses struct {
	Out                            []byte
	OutOff, Meta, ReqAt            []uint32 // req_cap + 1, req_cap, req_cap
	TraceIDs                       []byte   // req_cap * 16, or nil
	ReqFirst, Consumed, ConnStatus []uint32 // n + 1, n, n
	Log                            *ConnLog
}

// ConnLog is the request log of a connection batch.  Inputs: connection c's req.RemoteAddr is
// Remote[RemoteOff[c]:RemoteOff[c+1]] (at most 255 bytes) and its requests' start clock Start[c]; every line is logged at
// LogTime.  Outputs, sized with ConnLogBound: line m is Out[LogOff[m]:LogOff[m+1]] and belongs to request LogReq[m]; Lines
// and OutBytes are what the batch needed.  A request with status 0 (GOFR_H_HOST) has no line: log it once its closure ran.
type ConnLog struct {
	Remote         []byte
	RemoteOff      []uint32 // n + 1
	Start          []time.Time
	LogTime        time.Time
	Out            []byte
	LogOff, LogReq []uint32 // line_cap + 1, line_cap
	Lines          uint32
	OutBytes       uint64
}

// ConnLogBound gives the line and byte capacities that always suffice for the request log of connections with these
// offsets (gofr_conn_log_bound; no GPU needed).
func ConnLogBound(bufOff, remoteOff []uint32) (lineCap uint32, outCap uint64, err error) {
	if len(bufOff) == 0 || len(remoteOff) != len(bufOff) {
		return 0, 0, errors.New("gofrb200: bufOff and remoteOff need n + 1 entries")
	}
	var lc C.uint32_t
	var oc C.uint64_t
	err = check(C.gofr_conn_log_bound((*C.uint32_t)(unsafe.Pointer(&bufOff[0])), (*C.uint32_t)(unsafe.Pointer(&remoteOff[0])),
		C.uint32_t(len(bufOff)-1), &lc, &oc), "gofr_conn_log_bound")
	return uint32(lc), uint64(oc), err
}

// ConnBound gives the request and byte capacities that always suffice for connections with these offsets
// (gofr_conn_batch_bound; no GPU needed).
func (t *Table) ConnBound(bufOff []uint32) (reqCap uint32, outCap uint64, err error) {
	if len(bufOff) == 0 {
		return 0, 0, errors.New("gofrb200: bufOff needs n + 1 entries")
	}
	var rc C.uint32_t
	var oc C.uint64_t
	err = check(C.gofr_conn_batch_bound(t.t, (*C.uint32_t)(unsafe.Pointer(&bufOff[0])), C.uint32_t(len(bufOff)-1), &rc, &oc),
		"gofr_conn_batch_bound")
	return uint32(rc), uint64(oc), err
}

// ServeConnections serves every whole request in the connections' receive buffers (connection c = buf[bufOff[c]:bufOff[c+1]])
// with gofr_conn_batch_submit + wait and returns the response bytes written.  Write Out[OutOff[ReqFirst[c]]:OutOff[ReqFirst[c+1]]]
// to connection c, splicing in the host's responses for GOFR_H_HOST requests (status 0 in Meta); then keep its bytes from
// Consumed[c] on (HTTPConnMore) or hand them to net/http (HTTPConnDefer).  traceSeed must be fresh per batch.
func (e *Engine) ServeConnections(buf []byte, bufOff []uint32, now time.Time, traceSeed uint64, r *ConnResponses) (uint64, error) {
	return e.respondConnections(buf, bufOff, now, traceSeed, nil, r)
}

// ConnRoute receives what RouteConnections returns; the caller owns the slices and sizes them with ConnBound (reqCap) and
// len(buf) + 64 (Arena).  Request k: Meta[k] = status | route id << 16 (status 0: the closure of that route runs), its path
// variables Vars[8k:8k+8] (offset | length << 16 inside its path, 0xFFFFFFFF unused), ReqAt[k], TraceIDs[16k:16k+16] and
// its parsed request Desc[k], whose bytes are Arena[Desc[k].arena_off:] (decoded path | query | pad4 | body).
type ConnRoute struct {
	Desc                           []C.gofr_req_desc // req_cap
	Arena                          []byte            // len(buf) + 64
	Meta, ReqAt                    []uint32          // req_cap
	Vars                           []uint32          // req_cap * 8
	TraceIDs                       []byte            // req_cap * 16
	ReqFirst, Consumed, ConnStatus []uint32          // n + 1, n, n
}

// RouteConnections is stage 1 of serving connection buffers with handler closures (gofr_conn_batch_route, synchronous):
// frame, parse and route on the device.  Run the closures of the requests whose status is 0, encode each (data, err) as a
// GOFR_H_RESULT record, and pass the records to RespondConnections with the same buf, bufOff and traceSeed.
func (e *Engine) RouteConnections(buf []byte, bufOff []uint32, traceSeed uint64, r *ConnRoute) error {
	n := len(bufOff) - 1
	if n <= 0 {
		return nil
	}
	k := len(r.Meta)
	if len(buf) == 0 || k == 0 || len(r.Desc) < k || len(r.Arena) < len(buf)+64 || len(r.ReqAt) < k || len(r.Vars) < 8*k ||
		len(r.TraceIDs) < 16*k || len(r.ReqFirst) < n+1 || len(r.Consumed) < n || len(r.ConnStatus) < n {
		return errors.New("gofrb200: ConnRoute columns too small")
	}
	var in C.gofr_conn_batch
	in.buf = (*C.uint8_t)(unsafe.Pointer(&buf[0]))
	in.buf_off = (*C.uint32_t)(unsafe.Pointer(&bufOff[0]))
	in.buf_bytes = C.uint64_t(len(buf))
	in.n_conns = C.uint32_t(n)
	in.trace_seed = C.uint64_t(traceSeed)
	var o C.gofr_conn_route
	o.req_cap = C.uint32_t(k)
	o.desc = &r.Desc[0]
	o.arena = (*C.uint8_t)(unsafe.Pointer(&r.Arena[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&r.Meta[0]))
	o.vars = (*C.uint32_t)(unsafe.Pointer(&r.Vars[0]))
	o.req_at = (*C.uint32_t)(unsafe.Pointer(&r.ReqAt[0]))
	o.trace_ids = (*C.uint8_t)(unsafe.Pointer(&r.TraceIDs[0]))
	o.req_first = (*C.uint32_t)(unsafe.Pointer(&r.ReqFirst[0]))
	o.consumed = (*C.uint32_t)(unsafe.Pointer(&r.Consumed[0]))
	o.conn_status = (*C.uint32_t)(unsafe.Pointer(&r.ConnStatus[0]))
	return check(C.gofr_conn_batch_route(e.e, &in, &o), "gofr_conn_batch_route")
}

// RespondConnections is stage 2 (gofr_conn_batch_respond + wait): ServeConnections with request k's data section replaced by
// its closure's record rec[recOff[k]:recOff[k+1]] where that is not empty.  recOff has one entry per request of stage 1 plus
// one.  Size r.Out with RespondBound.
func (e *Engine) RespondConnections(buf []byte, bufOff []uint32, now time.Time, traceSeed uint64, rec []byte, recOff []uint32,
	r *ConnResponses) (uint64, error) {
	if len(recOff) == 0 {
		return 0, errors.New("gofrb200: recOff needs one entry per request plus one")
	}
	res := &C.gofr_conn_results{}
	if len(rec) > 0 {
		res.rec = (*C.uint8_t)(unsafe.Pointer(&rec[0]))
	}
	res.rec_off = (*C.uint32_t)(unsafe.Pointer(&recOff[0]))
	res.rec_bytes = C.uint64_t(len(rec))
	res.n_req = C.uint32_t(len(recOff) - 1)
	return e.respondConnections(buf, bufOff, now, traceSeed, res, r)
}

// RespondBound gives an output capacity that always suffices for RespondConnections on the requests stage 1 described
// (gofr_conn_respond_bound; no GPU needed).
func (t *Table) RespondBound(desc []C.gofr_req_desc, recOff []uint32) (uint64, error) {
	if len(recOff) != len(desc)+1 {
		return 0, errors.New("gofrb200: recOff needs len(desc) + 1 entries")
	}
	var oc C.uint64_t
	var d *C.gofr_req_desc
	if len(desc) > 0 {
		d = &desc[0]
	}
	err := check(C.gofr_conn_respond_bound(t.t, d, C.uint32_t(len(desc)), (*C.uint32_t)(unsafe.Pointer(&recOff[0])), &oc),
		"gofr_conn_respond_bound")
	return uint64(oc), err
}

func (e *Engine) respondConnections(buf []byte, bufOff []uint32, now time.Time, traceSeed uint64, res *C.gofr_conn_results,
	r *ConnResponses) (uint64, error) {
	n := len(bufOff) - 1
	if n <= 0 {
		return 0, nil
	}
	if len(buf) == 0 || len(r.Out) == 0 || len(r.Meta) == 0 || len(r.OutOff) < len(r.Meta)+1 || len(r.ReqAt) < len(r.Meta) ||
		(r.TraceIDs != nil && len(r.TraceIDs) < 16*len(r.Meta)) || len(r.ReqFirst) < n+1 || len(r.Consumed) < n || len(r.ConnStatus) < n {
		return 0, errors.New("gofrb200: ConnResponses columns too small")
	}
	var in C.gofr_conn_batch
	in.buf = (*C.uint8_t)(unsafe.Pointer(&buf[0]))
	in.buf_off = (*C.uint32_t)(unsafe.Pointer(&bufOff[0]))
	in.buf_bytes = C.uint64_t(len(buf))
	in.n_conns = C.uint32_t(n)
	in.trace_seed = C.uint64_t(traceSeed)
	C.gofr_format_http_date(C.int64_t(now.Unix()), &in.date[0])
	var o C.gofr_conn_resp
	o.out = (*C.uint8_t)(unsafe.Pointer(&r.Out[0]))
	o.out_cap = C.uint64_t(len(r.Out))
	o.req_cap = C.uint32_t(len(r.Meta))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&r.OutOff[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&r.Meta[0]))
	o.req_at = (*C.uint32_t)(unsafe.Pointer(&r.ReqAt[0]))
	if r.TraceIDs != nil {
		o.trace_ids = (*C.uint8_t)(unsafe.Pointer(&r.TraceIDs[0]))
	}
	o.req_first = (*C.uint32_t)(unsafe.Pointer(&r.ReqFirst[0]))
	o.consumed = (*C.uint32_t)(unsafe.Pointer(&r.Consumed[0]))
	o.conn_status = (*C.uint32_t)(unsafe.Pointer(&r.ConnStatus[0]))
	var lg *C.gofr_conn_log
	var start []int64
	if l := r.Log; l != nil {
		if len(l.RemoteOff) < n+1 || len(l.Start) < n || len(l.Out) == 0 || len(l.LogReq) == 0 || len(l.LogOff) < len(l.LogReq)+1 {
			return 0, errors.New("gofrb200: ConnLog columns too small")
		}
		start = make([]int64, n)
		for c := 0; c < n; c++ {
			start[c] = l.Start[c].UnixNano()
		}
		_, tz := l.LogTime.Zone()
		lg = &C.gofr_conn_log{}
		if len(l.Remote) > 0 {
			lg.remote = (*C.uint8_t)(unsafe.Pointer(&l.Remote[0]))
		}
		lg.remote_off = (*C.uint32_t)(unsafe.Pointer(&l.RemoteOff[0]))
		lg.start_unix_ns = (*C.int64_t)(unsafe.Pointer(&start[0]))
		lg.log_unix_ns = C.int64_t(l.LogTime.UnixNano())
		lg.tz_offset_s = C.int32_t(tz)
		lg.line_cap = C.uint32_t(len(l.LogReq))
		lg.out = (*C.uint8_t)(unsafe.Pointer(&l.Out[0]))
		lg.out_cap = C.uint64_t(len(l.Out))
		lg.log_off = (*C.uint32_t)(unsafe.Pointer(&l.LogOff[0]))
		lg.log_req = (*C.uint32_t)(unsafe.Pointer(&l.LogReq[0]))
	}
	var ticket C.gofr_ticket
	if err := check(C.gofr_conn_batch_respond(e.e, &in, res, &o, lg, &ticket), "gofr_conn_batch_respond"); err != nil {
		return 0, err
	}
	err := check(C.gofr_batch_wait(e.e, ticket), "gofr_batch_wait")
	if lg != nil {
		r.Log.Lines, r.Log.OutBytes = uint32(lg.lines), uint64(lg.out_bytes)
	}
	return uint64(o.out_bytes), err
}

// Frontend gathers single requests from many goroutines into batches (gofr_frontend_*): the per-request call that stands
// where router.ServeHTTP stands in the reference (pkg/gofr/httpServer.go:29-33).
type Frontend struct{ f *C.gofr_frontend }

func NewFrontend(e *Engine, maxBatch, maxWaitMicros, slotBytes, maxRequestBytes int) (*Frontend, error) {
	var f *C.gofr_frontend
	if err := check(C.gofr_frontend_create(&f, e.e, C.uint32_t(maxBatch), C.uint32_t(maxWaitMicros), C.uint32_t(slotBytes),
		C.uint32_t(maxRequestBytes)), "gofr_frontend_create"); err != nil {
		return nil, err
	}
	return &Frontend{f}, nil
}

// Close must not run while a Serve call is in progress.
func (f *Frontend) Close() { C.gofr_frontend_destroy(f.f); f.f = nil }

// Serve blocks until the batch this request joined has been served; resp[:n] is the response (wire bytes in FRAME_WIRE
// mode), meta = status | route id << 16.  A response that does not fit resp or the slot returns an error with n set.
func (f *Frontend) Serve(method uint8, path, query []byte, flags uint8, body []byte, traceID *[16]byte, resp []byte) (n int, meta uint32, err error) {
	var cn, cm C.uint32_t
	rc := C.gofr_frontend_serve(f.f, C.uint8_t(method), bytesPtr(path), C.uint16_t(len(path)), bytesPtr(query), C.uint16_t(len(query)),
		C.uint8_t(flags), bytesPtr(body), C.uint32_t(len(body)), (*C.uint8_t)(unsafe.Pointer(&traceID[0])), bytesPtr(resp),
		C.uint32_t(len(resp)), &cn, &cm)
	return int(cn), uint32(cm), check(rc, "gofr_frontend_serve")
}

func bytesPtr(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&b[0]))
}

// ProtoField is one field of a flat proto3 message type: (number, FieldDescriptorProto.Type).
type ProtoField struct{ Number, Type uint32 }

// ProtoEncodeDevice marshals n rows (GOFR_H_ROW layout, resident in HBM) as messages of the given type and frames them
// for gRPC (gofr_proto_encode_device): what proto.Marshal + grpc-go's msgHeader do for a unary handler's response.
func (e *Engine) ProtoEncodeDevice(fields []ProtoField, dRows, dRowOff unsafe.Pointer, n int, dOut unsafe.Pointer, outCap uint64,
	dOutOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	var fp *C.gofr_proto_field
	if len(fields) > 0 {
		fp = (*C.gofr_proto_field)(unsafe.Pointer(&fields[0]))
	}
	return check(C.gofr_proto_encode_device(e.e, fp, C.uint32_t(len(fields)), (*C.uint8_t)(dRows), (*C.uint32_t)(dRowOff), C.uint32_t(n),
		(*C.uint8_t)(dOut), C.uint64_t(outCap), (*C.uint32_t)(dOutOff), (*C.uint32_t)(dMeta), stream), "gofr_proto_encode_device")
}

// ProtoDecodeDevice is the other direction (gofr_proto_decode_device): length-prefixed request frames → rows.
func (e *Engine) ProtoDecodeDevice(fields []ProtoField, dIn, dInOff unsafe.Pointer, n int, dRows unsafe.Pointer, rowsCap uint64,
	dRowOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	var fp *C.gofr_proto_field
	if len(fields) > 0 {
		fp = (*C.gofr_proto_field)(unsafe.Pointer(&fields[0]))
	}
	return check(C.gofr_proto_decode_device(e.e, fp, C.uint32_t(len(fields)), (*C.uint8_t)(dIn), (*C.uint32_t)(dInOff), C.uint32_t(n),
		(*C.uint8_t)(dRows), C.uint64_t(rowsCap), (*C.uint32_t)(dRowOff), (*C.uint32_t)(dMeta), stream), "gofr_proto_decode_device")
}

// ProtoNField / ProtoNMsg describe message types with nested and repeated fields (gofr_proto_nfield / gofr_proto_nmsg):
// Msgs[m] owns Fields[FirstField : FirstField+NFields] in ascending field-number order; a field of Type 11
// (TYPE_MESSAGE) names its message type in Msg.  protoreflect gives all of it: for a generated message,
// walk md.Fields() (fd.Number(), fd.Kind(), fd.IsList(), fd.Message()).  A map field (fd.IsMap()) has Type ProtoMap,
// Repeated 0 and its entry type (fd.Message(): fields 1 key, 2 value) in Msg; rows carry its entries in ascending key
// order, which makes the output protobuf-go's Deterministic bytes.  (This file is not compiled in the repository's tests.)
type ProtoNField struct {
	Number   uint32
	Type     uint8
	Repeated uint8
	Msg      uint16
}
type ProtoNMsg struct{ FirstField, NFields uint16 }

// ProtoMap is the ProtoNField.Type of a map field (GOFR_PB_MAP).
const ProtoMap = C.GOFR_PB_MAP

// ProtoEncodeNestedDevice marshals n rows as messages of type msgs[root] and frames them for gRPC
// (gofr_proto_encode_nested_device): proto.Marshal for responses that are not flat — nested messages (a presence word
// and the message's fixed part inline in the row), repeated fields (a count, the elements in the row's variable part).
func (e *Engine) ProtoEncodeNestedDevice(msgs []ProtoNMsg, fields []ProtoNField, root uint32, dRows, dRowOff unsafe.Pointer, n int,
	dOut unsafe.Pointer, outCap uint64, dOutOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	if len(msgs) == 0 || len(fields) == 0 {
		return errors.New("gofrb200: empty message description")
	}
	return check(C.gofr_proto_encode_nested_device(e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), (*C.uint8_t)(dRows),
		(*C.uint32_t)(dRowOff), C.uint32_t(n), (*C.uint8_t)(dOut), C.uint64_t(outCap), (*C.uint32_t)(dOutOff), (*C.uint32_t)(dMeta), stream),
		"gofr_proto_encode_nested_device")
}

// SlotCTAs queries (ctas == 0) or forces (4 / 5) the instance of the slot-layout serve kernel (gofr_engine_slot_ctas).
func (e *Engine) SlotCTAs(ctas int) (int, error) {
	var v C.int
	err := check(C.gofr_engine_slot_ctas(e.e, C.int(ctas), &v), "gofr_engine_slot_ctas")
	return int(v), err
}

// ProtoDecodeNestedDevice is the other direction (gofr_proto_decode_nested_device): length-prefixed request frames → rows of
// msgs[root].  dMeta[i] == 6 (GOFR_GRPC_DEFER): a valid frame this decoder leaves to proto.Unmarshal on the host.
func (e *Engine) ProtoDecodeNestedDevice(msgs []ProtoNMsg, fields []ProtoNField, root uint32, dIn, dInOff unsafe.Pointer, n int,
	dRows unsafe.Pointer, rowsCap uint64, dRowOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	if len(msgs) == 0 || len(fields) == 0 {
		return errors.New("gofrb200: empty message description")
	}
	return check(C.gofr_proto_decode_nested_device(e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), (*C.uint8_t)(dIn),
		(*C.uint32_t)(dInOff), C.uint32_t(n), (*C.uint8_t)(dRows), C.uint64_t(rowsCap), (*C.uint32_t)(dRowOff), (*C.uint32_t)(dMeta), stream),
		"gofr_proto_decode_nested_device")
}

// ProtoOptional is the presence byte of a proto3 optional field (GOFR_PB_OPTIONAL).
const ProtoOptional = C.GOFR_PB_OPTIONAL

// presenceArg checks that presence has one byte per field and returns the C pointer (nil: no presence).
func presenceArg(presence []uint8, fields []ProtoNField) (*C.uint8_t, error) {
	if presence == nil {
		return nil, nil
	}
	if len(presence) != len(fields) {
		return nil, errors.New("gofrb200: one presence byte per field")
	}
	return (*C.uint8_t)(unsafe.Pointer(&presence[0])), nil
}

// ProtoEncodeNestedExDevice is ProtoEncodeNestedDevice for message types with field presence
// (gofr_proto_encode_nested_ex_device): presence[i] describes fields[i].  From protoreflect:
//   - fd.ContainingOneof() that is not synthetic (oneof.IsSynthetic() == false): the field is a member of that oneof; give
//     the message type's oneofs the numbers 1..7 (md.Oneofs() in order, synthetic ones skipped) — at most 7 per type;
//   - fd.HasOptionalKeyword(): ProtoOptional (its synthetic oneof is not a group);
//   - anything else: 0.
// A set explicit-presence field is written even at its zero value.  In the row, an optional or oneof scalar, string or
// bytes field has a presence word 0 / 1 before its usual words; a oneof message member is laid out as any singular message
// field.  A nil presence is ProtoEncodeNestedDevice.
func (e *Engine) ProtoEncodeNestedExDevice(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, dRows, dRowOff unsafe.Pointer,
	n int, dOut unsafe.Pointer, outCap uint64, dOutOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	if len(msgs) == 0 || len(fields) == 0 {
		return errors.New("gofrb200: empty message description")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return err
	}
	return check(C.gofr_proto_encode_nested_ex_device(e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, (*C.uint8_t)(dRows),
		(*C.uint32_t)(dRowOff), C.uint32_t(n), (*C.uint8_t)(dOut), C.uint64_t(outCap), (*C.uint32_t)(dOutOff), (*C.uint32_t)(dMeta), stream),
		"gofr_proto_encode_nested_ex_device")
}

// ProtoDecodeNestedExDevice is ProtoDecodeNestedDevice with the presence bytes of ProtoEncodeNestedExDevice
// (gofr_proto_decode_nested_ex_device): an optional field is set iff it occurs; of a oneof, the member occurring last on
// the wire is the set one; a oneof message member sent twice gives dMeta[i] == 6 (GOFR_GRPC_DEFER).
func (e *Engine) ProtoDecodeNestedExDevice(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, dIn, dInOff unsafe.Pointer,
	n int, dRows unsafe.Pointer, rowsCap uint64, dRowOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	if len(msgs) == 0 || len(fields) == 0 {
		return errors.New("gofrb200: empty message description")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return err
	}
	return check(C.gofr_proto_decode_nested_ex_device(e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, (*C.uint8_t)(dIn),
		(*C.uint32_t)(dInOff), C.uint32_t(n), (*C.uint8_t)(dRows), C.uint64_t(rowsCap), (*C.uint32_t)(dRowOff), (*C.uint32_t)(dMeta), stream),
		"gofr_proto_decode_nested_ex_device")
}

// ProtoDecodeNestedDeferredDevice is the second pass after ProtoDecodeNestedExDevice
// (gofr_proto_decode_nested_deferred_device): the frames whose status in dMetaIn is 6 (GOFR_GRPC_DEFER) are decoded
// again with map fields of up to 4096 entries; every other frame gets an empty row and keeps its status.  Same
// description, frames and offsets as the first call; dMeta may be dMetaIn.  Row i comes from this call's dRows when
// dMetaIn[i] was 6 and dMeta[i] is 0 (GOFR_GRPC_OK), else from the first call's.
func (e *Engine) ProtoDecodeNestedDeferredDevice(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, dIn, dInOff unsafe.Pointer,
	n int, dMetaIn, dRows unsafe.Pointer, rowsCap uint64, dRowOff, dMeta unsafe.Pointer, stream unsafe.Pointer) error {
	if len(msgs) == 0 || len(fields) == 0 {
		return errors.New("gofrb200: empty message description")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return err
	}
	return check(C.gofr_proto_decode_nested_deferred_device(e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, (*C.uint8_t)(dIn),
		(*C.uint32_t)(dInOff), C.uint32_t(n), (*C.uint32_t)(dMetaIn), (*C.uint8_t)(dRows), C.uint64_t(rowsCap), (*C.uint32_t)(dRowOff),
		(*C.uint32_t)(dMeta), stream),
		"gofr_proto_decode_nested_deferred_device")
}

// ProtoNestedDescribeEx validates a description with presence bytes without a GPU (gofr_proto_nested_describe_ex): nil
// when the encode and decode calls would accept it.
func ProtoNestedDescribeEx(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8) error {
	if len(msgs) == 0 || len(fields) == 0 {
		return errors.New("gofrb200: empty message description")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return err
	}
	rc := C.gofr_proto_nested_describe_ex((*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, nil, 0)
	if rc == C.GOFR_ERR_CAPACITY { // valid: no room asked for the descriptor
		return nil
	}
	return check(rc, "gofr_proto_nested_describe_ex")
}

// ProtoNestedBound returns (perByte, perRecord) such that no record of b bytes yields more than perByte*b + perRecord
// output bytes (gofr_proto_nested_bound; no GPU): a row when decode is true, a whole frame when encoding.  Sum it over a
// batch to size the out buffer of ProtoDecodeBatch / ProtoEncodeBatch.
func ProtoNestedBound(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, decode bool) (perByte, perRecord uint32, err error) {
	if len(msgs) == 0 || len(fields) == 0 {
		return 0, 0, errors.New("gofrb200: empty message description")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return 0, 0, err
	}
	d := C.int(0)
	if decode {
		d = 1
	}
	var pb, pr C.uint32_t
	err = check(C.gofr_proto_nested_bound((*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, d, &pb, &pr),
		"gofr_proto_nested_bound")
	return uint32(pb), uint32(pr), err
}

// protoBatch runs gofr_proto_batch_decode / _encode on host buffers and waits for it: record i = data[off[i]:off[i+1]],
// results into out (ideally from gofr_alloc_pinned), outOff (n+1) and meta (n).  Returns the bytes written.
func (e *Engine) protoBatch(decode bool, msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, data []byte, off []uint32,
	out []byte, outOff, meta []uint32) (int, error) {
	if len(msgs) == 0 || len(fields) == 0 || len(off) == 0 {
		return 0, errors.New("gofrb200: empty message description or offsets")
	}
	n := len(off) - 1
	if n == 0 {
		return 0, nil
	}
	if len(outOff) < n+1 || len(meta) < n || len(out) == 0 {
		return 0, errors.New("gofrb200: out/outOff/meta too small")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return 0, err
	}
	var in C.gofr_proto_batch
	if len(data) > 0 {
		in.data = (*C.uint8_t)(unsafe.Pointer(&data[0]))
	}
	in.data_bytes = C.uint64_t(len(data))
	in.off = (*C.uint32_t)(unsafe.Pointer(&off[0]))
	in.n = C.uint32_t(n)
	var o C.gofr_resp_batch
	o.out = (*C.uint8_t)(unsafe.Pointer(&out[0]))
	o.out_cap = C.uint64_t(len(out))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&meta[0]))
	var ticket C.gofr_ticket
	cm, cf := (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), (*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0]))
	if decode {
		err = check(C.gofr_proto_batch_decode(e.e, cm, C.uint32_t(len(msgs)), cf, C.uint32_t(len(fields)), C.uint32_t(root), pp, &in, &o, &ticket),
			"gofr_proto_batch_decode")
	} else {
		err = check(C.gofr_proto_batch_encode(e.e, cm, C.uint32_t(len(msgs)), cf, C.uint32_t(len(fields)), C.uint32_t(root), pp, &in, &o, &ticket),
			"gofr_proto_batch_encode")
	}
	if err != nil {
		return 0, err
	}
	if err := check(C.gofr_batch_wait(e.e, ticket), "gofr_batch_wait"); err != nil {
		return 0, err
	}
	return int(o.out_bytes), nil
}

// ProtoDecodeBatch decodes a batch of request frames held in host memory (gofr_proto_batch_decode): both decode passes,
// merged, so row i = out[outOff[i]:outOff[i+1]] and meta[i] are final.  meta[i] == 6 (GOFR_GRPC_DEFER): hand frame i
// to proto.Unmarshal on the host; its row is empty, as is a failed frame's.
func (e *Engine) ProtoDecodeBatch(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, frames []byte, off []uint32,
	out []byte, outOff, meta []uint32) (int, error) {
	return e.protoBatch(true, msgs, fields, root, presence, frames, off, out, outOff, meta)
}

// ProtoEncodeBatch marshals a batch of response rows held in host memory into gRPC frames (gofr_proto_batch_encode): what
// ProtoEncodeNestedExDevice gives, status for status.  Row offsets are multiples of 4.
func (e *Engine) ProtoEncodeBatch(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, rows []byte, off []uint32,
	out []byte, outOff, meta []uint32) (int, error) {
	return e.protoBatch(false, msgs, fields, root, presence, rows, off, out, outOff, meta)
}

// ProtoEncodeBatchLog marshals a batch of response rows like ProtoEncodeBatch and writes the gRPC LoggingInterceptor's
// RPCLog line for each call in the same call (gofr_proto_batch_encode_log): log holds one record per row, appended with
// AppendRPC; its log time is now.  A call whose handler failed passes an empty row: its frame is to be ignored, its line is
// still written.  Call i's line is lines[logOff[i]:logOff[i+1]]; logOff needs len(off) entries; a short lines buffer is
// gofr_batch_wait's GOFR_ERR_CAPACITY (gofr_batch_log_bound sizes it).  Returns the frame and line bytes the batch needed.
func (e *Engine) ProtoEncodeBatchLog(msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, rows []byte, off []uint32,
	log *LogBatch, now time.Time, out []byte, outOff, meta []uint32, lines []byte, logOff []uint32) (int, int, error) {
	n := len(off) - 1
	if n <= 0 {
		return 0, 0, nil
	}
	if len(out) == 0 || len(outOff) < n+1 || len(meta) < n || len(log.Desc) != n || len(log.TraceIDs) < 16*n ||
		len(logOff) < n+1 || len(lines) == 0 {
		return 0, 0, errors.New("gofrb200: ProtoEncodeBatchLog columns too small")
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return 0, 0, err
	}
	var in C.gofr_proto_batch
	if len(rows) > 0 {
		in.data = (*C.uint8_t)(unsafe.Pointer(&rows[0]))
	}
	in.data_bytes = C.uint64_t(len(rows))
	in.off = (*C.uint32_t)(unsafe.Pointer(&off[0]))
	in.n = C.uint32_t(n)
	var o C.gofr_resp_batch
	o.out = (*C.uint8_t)(unsafe.Pointer(&out[0]))
	o.out_cap = C.uint64_t(len(out))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&outOff[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&meta[0]))
	var l C.gofr_batch_log
	l.desc = &log.Desc[0]
	if len(log.Arena) > 0 {
		l.arena = (*C.uint8_t)(unsafe.Pointer(&log.Arena[0]))
	}
	l.arena_bytes = C.uint64_t(len(log.Arena))
	l.log_unix_ns = C.int64_t(now.UnixNano())
	l.out = (*C.uint8_t)(unsafe.Pointer(&lines[0]))
	l.out_cap = C.uint64_t(len(lines))
	l.log_off = (*C.uint32_t)(unsafe.Pointer(&logOff[0]))
	var ticket C.gofr_ticket
	cm, cf := (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), (*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0]))
	if err := check(C.gofr_proto_batch_encode_log(e.e, cm, C.uint32_t(len(msgs)), cf, C.uint32_t(len(fields)), C.uint32_t(root), pp, &in,
		(*C.uint8_t)(unsafe.Pointer(&log.TraceIDs[0])), &o, &l, &ticket), "gofr_proto_batch_encode_log"); err != nil {
		return 0, 0, err
	}
	if err := check(C.gofr_batch_wait(e.e, ticket), "gofr_batch_wait"); err != nil {
		return 0, 0, err
	}
	return int(o.out_bytes), int(l.out_bytes), nil
}

// ProtoFrontend batches single messages from many goroutines through the nested codec (gofr_proto_frontend_*): the
// per-message call grpc-go makes on its codec (encoding.Codec.Unmarshal for a request, Marshal for a response, on the
// RPC's goroutine).  One message type, one direction.  Several ProtoFrontends and a Frontend may share one Engine.
type ProtoFrontend struct {
	f         *C.gofr_proto_frontend
	perByte   uint32
	perRecord uint32
	log       bool
}

// ErrProtoRecordTooLarge is what ProtoFrontend.Call returns, before anything is queued, for a record longer than the
// front-end's maxRecordBytes: marshal or unmarshal that one with protobuf-go.
var ErrProtoRecordTooLarge = errors.New("gofrb200: record exceeds the front-end's maxRecordBytes")

// NewProtoFrontend creates the decode (decode == true) or encode front-end of message type msgs[root].  maxBatch and
// maxWaitMicros mean what they mean for NewFrontend; a record longer than maxRecordBytes is refused
// (ErrProtoRecordTooLarge) before it is queued.
func NewProtoFrontend(e *Engine, msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8, decode bool,
	maxBatch, maxWaitMicros, maxRecordBytes int) (*ProtoFrontend, error) {
	perByte, perRecord, err := ProtoNestedBound(msgs, fields, root, presence, decode)
	if err != nil {
		return nil, err
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return nil, err
	}
	d := C.int(0)
	if decode {
		d = 1
	}
	var f *C.gofr_proto_frontend
	if err := check(C.gofr_proto_frontend_create(&f, e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, d, C.uint32_t(maxBatch),
		C.uint32_t(maxWaitMicros), C.uint32_t(maxRecordBytes)), "gofr_proto_frontend_create"); err != nil {
		return nil, err
	}
	return &ProtoFrontend{f, perByte, perRecord, false}, nil
}

// NewProtoFrontendLog creates the encode front-end of message type msgs[root] whose callers may also ask for their call's
// RPCLog line (CallLog), for methods of at most maxLogBytes bytes (gofr_proto_frontend_create_log).
func NewProtoFrontendLog(e *Engine, msgs []ProtoNMsg, fields []ProtoNField, root uint32, presence []uint8,
	maxBatch, maxWaitMicros, maxRecordBytes, maxLogBytes int) (*ProtoFrontend, error) {
	perByte, perRecord, err := ProtoNestedBound(msgs, fields, root, presence, false)
	if err != nil {
		return nil, err
	}
	pp, err := presenceArg(presence, fields)
	if err != nil {
		return nil, err
	}
	var f *C.gofr_proto_frontend
	if err := check(C.gofr_proto_frontend_create_log(&f, e.e, (*C.gofr_proto_nmsg)(unsafe.Pointer(&msgs[0])), C.uint32_t(len(msgs)),
		(*C.gofr_proto_nfield)(unsafe.Pointer(&fields[0])), C.uint32_t(len(fields)), C.uint32_t(root), pp, 0, C.uint32_t(maxBatch),
		C.uint32_t(maxWaitMicros), C.uint32_t(maxRecordBytes), C.uint32_t(maxLogBytes)), "gofr_proto_frontend_create_log"); err != nil {
		return nil, err
	}
	return &ProtoFrontend{f, perByte, perRecord, true}, nil
}

// Close must not run while a Call is in progress.
func (p *ProtoFrontend) Close() { C.gofr_proto_frontend_destroy(p.f); p.f = nil }

// Stats returns the batches run and the records they held.
func (p *ProtoFrontend) Stats() (batches, records uint64, err error) {
	var b, r C.uint64_t
	err = check(C.gofr_proto_frontend_stats(p.f, &b, &r), "gofr_proto_frontend_stats")
	return uint64(b), uint64(r), err
}

// Call blocks until the batch this record joined has come back.  Decode: in is the message as Unmarshal receives it (no
// 5-byte prefix), the result is its row.  Encode: in is a row, the result is the marshalled message without the prefix, as
// Marshal returns it.  status is a GOFR_GRPC_* code: 6 (GOFR_GRPC_DEFER) means "decode this one with proto.Unmarshal", as
// does ErrProtoRecordTooLarge.  out has room for the record's bound, so the result always fits.
func (p *ProtoFrontend) Call(in []byte) (out []byte, status uint32, err error) {
	buf := make([]byte, uint64(p.perByte)*uint64(len(in)+5)+uint64(p.perRecord))
	var n, st C.uint32_t
	rc := C.gofr_proto_frontend_call(p.f, bytesPtr(in), C.uint32_t(len(in)), bytesPtr(buf), C.uint32_t(len(buf)), &n, &st)
	if rc == C.GOFR_ERR_CAPACITY {
		return nil, 0, ErrProtoRecordTooLarge
	}
	if err = check(rc, "gofr_proto_frontend_call"); err != nil {
		return nil, 0, err
	}
	return buf[:n], uint32(st), nil
}

// CallLog is Call for an encode front-end made by NewProtoFrontendLog, plus the RPCLog line LoggingInterceptor writes once
// the handler has returned: row is the handler's response (empty when it failed: the message is then to be ignored, the
// line is still written), traceID the span's, start and elapsed the interceptor's clock around the handler, method
// info.FullMethod.  The line is the batch's (gofr_proto_frontend_call_log); its buffer has room for the line's bound.  A row
// longer than maxRecordBytes or a method longer than maxLogBytes is ErrProtoRecordTooLarge, before anything is queued.
func (p *ProtoFrontend) CallLog(row []byte, traceID [16]byte, start time.Time, elapsed time.Duration, method string) (out []byte,
	status uint32, line []byte, err error) {
	if !p.log || len(method) > 0xFFFF {
		return nil, 0, nil, errors.New("gofrb200: CallLog needs a front-end made by NewProtoFrontendLog and a method of at most 65535 bytes")
	}
	var lb LogBatch
	lb.AppendRPC(start, elapsed, traceID, method)
	buf := make([]byte, uint64(p.perByte)*uint64(len(row)+5)+uint64(p.perRecord))
	lbuf := make([]byte, 320+7*len(method))
	var n, st, ln C.uint32_t
	rc := C.gofr_proto_frontend_call_log(p.f, bytesPtr(row), C.uint32_t(len(row)), (*C.uint8_t)(unsafe.Pointer(&traceID[0])), &lb.Desc[0],
		bytesPtr(lb.Arena), bytesPtr(buf), C.uint32_t(len(buf)), &n, &st, bytesPtr(lbuf), C.uint32_t(len(lbuf)), &ln)
	if rc == C.GOFR_ERR_CAPACITY {
		return nil, 0, nil, ErrProtoRecordTooLarge
	}
	if err = check(rc, "gofr_proto_frontend_call_log"); err != nil {
		return nil, 0, nil, err
	}
	return buf[:n], uint32(st), lbuf[:ln], nil
}

// ConnFrontend batches single reads from many connection goroutines through the connection pipeline
// (gofr_conn_frontend_*): the per-connection loop of net/http's conn.serve (pkg/gofr/httpServer.go:29-33) hands in what it
// holds for its connection and gets that connection's answers back, framed, parsed and served on the GPU together with
// the other goroutines' reads.  Several front-ends of any kind may share one Engine.
type ConnFrontend struct {
	f            *C.gofr_conn_frontend
	maxConnBytes int
	log          bool
}

// ErrConnReadTooLarge is what ConnFrontend.Serve returns, before anything is queued, for a read longer than the
// front-end's maxConnBytes: serve that connection with net/http.
var ErrConnReadTooLarge = errors.New("gofrb200: read exceeds the front-end's maxConnBytes")

// NewConnFrontend: maxBatch and maxWaitMicros mean what they mean for NewFrontend; a read longer than maxConnBytes is
// refused (ErrConnReadTooLarge).  With log, Serve also returns middleware.Logging's lines, logged in a zone
// tzOffsetSeconds east of UTC.  Batch b draws its trace ids from splitmix64(splitmix64(seed) + b).
func NewConnFrontend(e *Engine, maxBatch, maxWaitMicros, maxConnBytes int, log bool, tzOffsetSeconds int32, seed uint64) (*ConnFrontend, error) {
	l := C.int(0)
	if log {
		l = 1
	}
	var f *C.gofr_conn_frontend
	if err := check(C.gofr_conn_frontend_create(&f, e.e, C.uint32_t(maxBatch), C.uint32_t(maxWaitMicros), C.uint32_t(maxConnBytes), l,
		C.int32_t(tzOffsetSeconds), C.uint64_t(seed)), "gofr_conn_frontend_create"); err != nil {
		return nil, err
	}
	return &ConnFrontend{f, maxConnBytes, log}, nil
}

// Close must not run while a Serve is in progress.
func (f *ConnFrontend) Close() { C.gofr_conn_frontend_destroy(f.f); f.f = nil }

// SetClock pins the Date header and the log time of every batch (tests); the zero Time restores the wall clock.
func (f *ConnFrontend) SetClock(t time.Time) error {
	ns := int64(0)
	if !t.IsZero() {
		ns = t.UnixNano()
	}
	return check(C.gofr_conn_frontend_set_clock(f.f, C.int64_t(ns)), "gofr_conn_frontend_set_clock")
}

// Stats returns the batches run, the reads they held, and the batches served again after their outputs grew.
func (f *ConnFrontend) Stats() (batches, conns, reruns uint64, err error) {
	var b, c, r C.uint64_t
	err = check(C.gofr_conn_frontend_stats(f.f, &b, &c, &r), "gofr_conn_frontend_stats")
	return uint64(b), uint64(c), uint64(r), err
}

// Serve blocks until the batch this read joined has been served and fills r as ServeConnections fills it for a batch of
// one connection: size its slices with Table.ConnBound([]uint32{0, len(buf)}) (ReqFirst 2, Consumed and ConnStatus 1).
// With r.Log set on a front-end created with log, its output fields (Out, LogOff, LogReq, sized with ConnLogBound) receive
// the connection's lines; its input fields are not used: remote and start are this read's req.RemoteAddr and Logging's
// start clock.  Returns the response bytes written.  Then write Out[:n], running the closures of the holes (status 0 in
// Meta) from buf[ReqAt[k]:]; keep buf[Consumed[0]:] on HTTPConnMore, hand it to net/http on HTTPConnDefer.
func (f *ConnFrontend) Serve(buf, remote []byte, start time.Time, r *ConnResponses) (uint64, error) {
	if len(buf) > f.maxConnBytes {
		return 0, ErrConnReadTooLarge
	}
	if len(r.Out) == 0 || len(r.Meta) == 0 || len(r.OutOff) < len(r.Meta)+1 || len(r.ReqAt) < len(r.Meta) ||
		(r.TraceIDs != nil && len(r.TraceIDs) < 16*len(r.Meta)) || len(r.ReqFirst) < 2 || len(r.Consumed) < 1 || len(r.ConnStatus) < 1 {
		return 0, errors.New("gofrb200: ConnResponses columns too small")
	}
	var o C.gofr_conn_resp
	o.out = (*C.uint8_t)(unsafe.Pointer(&r.Out[0]))
	o.out_cap = C.uint64_t(len(r.Out))
	o.req_cap = C.uint32_t(len(r.Meta))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&r.OutOff[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&r.Meta[0]))
	o.req_at = (*C.uint32_t)(unsafe.Pointer(&r.ReqAt[0]))
	if r.TraceIDs != nil {
		o.trace_ids = (*C.uint8_t)(unsafe.Pointer(&r.TraceIDs[0]))
	}
	o.req_first = (*C.uint32_t)(unsafe.Pointer(&r.ReqFirst[0]))
	o.consumed = (*C.uint32_t)(unsafe.Pointer(&r.Consumed[0]))
	o.conn_status = (*C.uint32_t)(unsafe.Pointer(&r.ConnStatus[0]))
	var lg *C.gofr_conn_log
	if l := r.Log; l != nil && f.log {
		if len(l.Out) == 0 || len(l.LogReq) == 0 || len(l.LogOff) < len(l.LogReq)+1 {
			return 0, errors.New("gofrb200: ConnLog columns too small")
		}
		lg = &C.gofr_conn_log{}
		lg.line_cap = C.uint32_t(len(l.LogReq))
		lg.out = (*C.uint8_t)(unsafe.Pointer(&l.Out[0]))
		lg.out_cap = C.uint64_t(len(l.Out))
		lg.log_off = (*C.uint32_t)(unsafe.Pointer(&l.LogOff[0]))
		lg.log_req = (*C.uint32_t)(unsafe.Pointer(&l.LogReq[0]))
	}
	ns := int64(0)
	if !start.IsZero() {
		ns = start.UnixNano()
	}
	rc := C.gofr_conn_frontend_serve(f.f, bytesPtr(buf), C.uint32_t(len(buf)), bytesPtr(remote), C.uint32_t(len(remote)), C.int64_t(ns),
		&o, lg)
	if lg != nil {
		r.Log.Lines, r.Log.OutBytes = uint32(lg.lines), uint64(lg.out_bytes)
	}
	return uint64(o.out_bytes), check(rc, "gofr_conn_frontend_serve")
}

// ConnAppFrontend serves handler-closure apps one connection read per call (gofr_conn_app_frontend_*): Route hands in a
// read and returns its requests routed, parsed and bound on the GPU together with the other goroutines' reads; the
// goroutine runs the closures itself, as long as they take; Respond hands in the same read with the closures' records and
// returns its responses.  Route batches and respond batches are independent, so no response waits for another
// connection's closure.  Several front-ends of any kind may share one Engine.
type ConnAppFrontend struct {
	f            *C.gofr_conn_app_frontend
	maxConnBytes int
	log          bool
	maxFields    int
}

// ConnAppRoute is what Route returns for one read: its requests as ServeConnections' stage 1 returns them for a batch of
// one (Desc into Arena, ReqAt into the read), each request's bind status (GOFR_BIND_*, 0xFFFFFFFF when not bound) and row
// Rows[RowOff[k]:RowOff[k+1]], and the read's trace key, which Respond takes.
type ConnAppRoute struct {
	Desc                 []C.gofr_req_desc
	Arena                []byte
	Meta, Vars, ReqAt    []uint32
	TraceIDs             []byte
	Consumed, ConnStatus uint32
	BindStatus, RowOff   []uint32
	Rows                 []byte
	TraceKey             uint64
}

// NewConnAppFrontend: maxBatch and maxWaitMicros mean what they mean for NewFrontend; a read longer than maxConnBytes is
// refused (ErrConnReadTooLarge).  routeSchema[r] is the schema route r binds (0: none) and schemaFields[r] that schema's
// field count.  With log, Respond also returns middleware.Logging's lines.
func NewConnAppFrontend(e *Engine, maxBatch, maxWaitMicros, maxConnBytes int, log bool, tzOffsetSeconds int32, seed uint64,
	routeSchema, schemaFields []uint32) (*ConnAppFrontend, error) {
	if len(routeSchema) != len(schemaFields) {
		return nil, errors.New("gofrb200: routeSchema and schemaFields differ in length")
	}
	l := C.int(0)
	if log {
		l = 1
	}
	var rs, sf *C.uint32_t
	maxFields := 0
	if len(routeSchema) > 0 {
		rs = (*C.uint32_t)(unsafe.Pointer(&routeSchema[0]))
		sf = (*C.uint32_t)(unsafe.Pointer(&schemaFields[0]))
		for _, n := range schemaFields {
			if int(n) > maxFields {
				maxFields = int(n)
			}
		}
	}
	var f *C.gofr_conn_app_frontend
	if err := check(C.gofr_conn_app_frontend_create(&f, e.e, C.uint32_t(maxBatch), C.uint32_t(maxWaitMicros), C.uint32_t(maxConnBytes), l,
		C.int32_t(tzOffsetSeconds), C.uint64_t(seed), rs, C.uint32_t(len(routeSchema)), sf), "gofr_conn_app_frontend_create"); err != nil {
		return nil, err
	}
	return &ConnAppFrontend{f, maxConnBytes, log, maxFields}, nil
}

// Close must not run while a Route or Respond is in progress.
func (f *ConnAppFrontend) Close() { C.gofr_conn_app_frontend_destroy(f.f); f.f = nil }

// SetClock pins the Date header and the log time of every respond batch (tests); the zero Time restores the wall clock.
func (f *ConnAppFrontend) SetClock(t time.Time) error {
	ns := int64(0)
	if !t.IsZero() {
		ns = t.UnixNano()
	}
	return check(C.gofr_conn_app_frontend_set_clock(f.f, C.int64_t(ns)), "gofr_conn_app_frontend_set_clock")
}

// Stats returns gofr_conn_app_stats: route and respond batches and reads, reruns, isolated batches, record-gather time.
func (f *ConnAppFrontend) Stats() (C.gofr_conn_app_stats, error) {
	var st C.gofr_conn_app_stats
	return st, check(C.gofr_conn_app_frontend_stats(f.f, &st), "gofr_conn_app_frontend_stats")
}

// Route blocks until the route batch this read joined has been routed and bound.
func (f *ConnAppFrontend) Route(buf []byte) (*ConnAppRoute, error) {
	if len(buf) > f.maxConnBytes {
		return nil, ErrConnReadTooLarge
	}
	reqCap := len(buf)/16 + 1 // the framer's most for one connection
	r := &ConnAppRoute{Desc: make([]C.gofr_req_desc, reqCap), Arena: make([]byte, len(buf)+80), Meta: make([]uint32, reqCap),
		Vars: make([]uint32, reqCap*C.GOFR_MAX_PATH_VARS), ReqAt: make([]uint32, reqCap), TraceIDs: make([]byte, 16*reqCap),
		BindStatus: make([]uint32, reqCap), RowOff: make([]uint32, reqCap+1)}
	var first [2]C.uint32_t
	var rt C.gofr_conn_route
	rt.req_cap = C.uint32_t(reqCap)
	rt.desc = &r.Desc[0]
	rt.arena = (*C.uint8_t)(unsafe.Pointer(&r.Arena[0]))
	rt.meta = (*C.uint32_t)(unsafe.Pointer(&r.Meta[0]))
	rt.vars = (*C.uint32_t)(unsafe.Pointer(&r.Vars[0]))
	rt.req_at = (*C.uint32_t)(unsafe.Pointer(&r.ReqAt[0]))
	rt.trace_ids = (*C.uint8_t)(unsafe.Pointer(&r.TraceIDs[0]))
	rt.req_first = &first[0]
	rt.consumed = (*C.uint32_t)(unsafe.Pointer(&r.Consumed))
	rt.conn_status = (*C.uint32_t)(unsafe.Pointer(&r.ConnStatus))
	var bd C.gofr_conn_app_bind
	bd.status = (*C.uint32_t)(unsafe.Pointer(&r.BindStatus[0]))
	bd.row_off = (*C.uint32_t)(unsafe.Pointer(&r.RowOff[0]))
	var key C.uint64_t
	// GOFR_BIND_ROW_BOUND without the schemas' names, which are not known here: a read whose error texts need more is
	// routed again with the rows it reported
	rowsCap := reqCap*(8*f.maxFields+70) + 3*len(buf)
	for {
		r.Rows = make([]byte, rowsCap)
		bd.rows = (*C.uint8_t)(unsafe.Pointer(&r.Rows[0]))
		bd.rows_cap = C.uint64_t(len(r.Rows))
		rc := C.gofr_conn_app_frontend_route(f.f, bytesPtr(buf), C.uint32_t(len(buf)), &rt, &bd, &key)
		if rc != C.GOFR_ERR_CAPACITY || int(bd.rows_bytes) <= rowsCap {
			if err := check(rc, "gofr_conn_app_frontend_route"); err != nil {
				return nil, err
			}
			break
		}
		rowsCap = int(bd.rows_bytes)
	}
	n := int(first[1])
	r.Desc, r.Meta, r.Vars, r.ReqAt = r.Desc[:n], r.Meta[:n], r.Vars[:n*C.GOFR_MAX_PATH_VARS], r.ReqAt[:n]
	r.TraceIDs, r.BindStatus, r.RowOff, r.Rows = r.TraceIDs[:16*n], r.BindStatus[:n], r.RowOff[:n+1], r.Rows[:bd.rows_bytes]
	r.TraceKey = uint64(key)
	return r, nil
}

// Respond blocks until the respond batch this read joined has been served: buf is the read Route took, key its TraceKey,
// request k's record recs[recOff[k]:recOff[k+1]] (GOFR_H_RESULT; empty: the request is answered as ServeConnections
// answers it).  r and the return value are ConnFrontend.Serve's.
func (f *ConnAppFrontend) Respond(buf []byte, key uint64, recs []byte, recOff []uint32, remote []byte, start time.Time, r *ConnResponses) (uint64, error) {
	if len(buf) > f.maxConnBytes {
		return 0, ErrConnReadTooLarge
	}
	if len(recOff) == 0 || len(r.Out) == 0 || len(r.Meta) == 0 || len(r.OutOff) < len(r.Meta)+1 || len(r.ReqAt) < len(r.Meta) ||
		(r.TraceIDs != nil && len(r.TraceIDs) < 16*len(r.Meta)) || len(r.ReqFirst) < 2 || len(r.Consumed) < 1 || len(r.ConnStatus) < 1 {
		return 0, errors.New("gofrb200: record offsets or ConnResponses columns too small")
	}
	var res C.gofr_conn_results
	res.rec = bytesPtr(recs)
	res.rec_off = (*C.uint32_t)(unsafe.Pointer(&recOff[0]))
	res.rec_bytes = C.uint64_t(len(recs))
	res.n_req = C.uint32_t(len(recOff) - 1)
	var o C.gofr_conn_resp
	o.out = (*C.uint8_t)(unsafe.Pointer(&r.Out[0]))
	o.out_cap = C.uint64_t(len(r.Out))
	o.req_cap = C.uint32_t(len(r.Meta))
	o.out_off = (*C.uint32_t)(unsafe.Pointer(&r.OutOff[0]))
	o.meta = (*C.uint32_t)(unsafe.Pointer(&r.Meta[0]))
	o.req_at = (*C.uint32_t)(unsafe.Pointer(&r.ReqAt[0]))
	if r.TraceIDs != nil {
		o.trace_ids = (*C.uint8_t)(unsafe.Pointer(&r.TraceIDs[0]))
	}
	o.req_first = (*C.uint32_t)(unsafe.Pointer(&r.ReqFirst[0]))
	o.consumed = (*C.uint32_t)(unsafe.Pointer(&r.Consumed[0]))
	o.conn_status = (*C.uint32_t)(unsafe.Pointer(&r.ConnStatus[0]))
	var lg *C.gofr_conn_log
	if l := r.Log; l != nil && f.log {
		if len(l.Out) == 0 || len(l.LogReq) == 0 || len(l.LogOff) < len(l.LogReq)+1 {
			return 0, errors.New("gofrb200: ConnLog columns too small")
		}
		lg = &C.gofr_conn_log{}
		lg.line_cap = C.uint32_t(len(l.LogReq))
		lg.out = (*C.uint8_t)(unsafe.Pointer(&l.Out[0]))
		lg.out_cap = C.uint64_t(len(l.Out))
		lg.log_off = (*C.uint32_t)(unsafe.Pointer(&l.LogOff[0]))
		lg.log_req = (*C.uint32_t)(unsafe.Pointer(&l.LogReq[0]))
	}
	ns := int64(0)
	if !start.IsZero() {
		ns = start.UnixNano()
	}
	rc := C.gofr_conn_app_frontend_respond(f.f, bytesPtr(buf), C.uint32_t(len(buf)), C.uint64_t(key), &res, bytesPtr(remote),
		C.uint32_t(len(remote)), C.int64_t(ns), &o, lg)
	if lg != nil {
		r.Log.Lines, r.Log.OutBytes = uint32(lg.lines), uint64(lg.out_bytes)
	}
	return uint64(o.out_bytes), check(rc, "gofr_conn_app_frontend_respond")
}
