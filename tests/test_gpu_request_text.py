"""The request-text corpus of tests/test_request_text.py through the kernels: query values, path variables, redirect
Locations and RequestLog fields, on every entry point that copies request bytes into its output.

What the CPU emulation cannot reach is exercised here: staged against unstaged tiles (a tile's span within or over the
staging budget, and spans of exactly in_cap and in_cap + 16), the warp-cooperative Writer's slow calls, the wide 4-CTA slot
instance against the 5-CTA one, the _values instances, the slot-overflow contract, the host chunk loop with pinned and
pageable buffers, the connection path from raw HTTP/1.1 messages with its log lines, and gofr_batch_submit_log.  Each
request passes two checks: the GPU equals the oracle byte for byte (output, offsets, meta), and the GPU equals the model
(tests/go_net_url.py) — status, Location, Content-Length against the body, the body, and each log line's method,
user_agent, ip and uri as encoding/json bytes.  Every response also fits gofr_table_response_bound.

Each campaign runs in a child process of its own: a fault in a kernel stays inside its test.
"""
import os
import random
import subprocess
import sys
import time

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from tests import oracle as O
from tests import test_batch_log as BL
from tests import test_conn_log as CL
from tests import test_gpu_geometry as TG
from tests import test_request_text as RT

ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATE = TG.DATE
assert DATE == RT.DATE


def _model_check(resps, meta, expects, labels, what):
    bad = RT.model_problems(resps, meta, expects)
    assert not bad, "%s: %r" % (what, [(labels[i], p) for i, p in bad[:6]])


def _bounds_hold(table, batch, off, what):
    L, h = _abi.lib(), table.handle
    d = batch.desc
    ln = np.diff(off.astype(np.int64))
    for i in range(batch.n):
        b = int(L.gofr_table_response_bound(h, int(d["path_len"][i]), int(d["query_len"][i]), int(d["data_len"][i])))
        assert ln[i] <= b, "%s: request %d is %d bytes, its bound %d" % (what, i, int(ln[i]), b)


def _host():
    corpus = RT.host_corpus()
    batch, labels = RT.host_batch(corpus)
    return batch, labels, [RT.host_expect(r) for _, r in corpus]


def _small(batch, limit):
    """the requests whose path and query take at most `limit` bytes (for tiles that fit a staging budget exactly)"""
    d = batch.desc
    keep = np.flatnonzero(d["path_len"].astype(np.int64) + d["query_len"] <= limit)
    ar = batch.arena.tobytes()
    reqs = []
    for i in keep.tolist():
        o, pl, ql = int(d["arena_off"][i]), int(d["path_len"][i]), int(d["query_len"][i])
        reqs.append(S.Req(S.M_GET, ar[o:o + pl], ar[o + pl:o + pl + ql], flags=int(d["flags"][i])))
    return S.RequestBatch.pack(reqs, seed=5), keep


# ---------------------------------------------------------------------------------------------------------------
# campaigns
# ---------------------------------------------------------------------------------------------------------------
def _gpu_packed():
    """gofr_serve_device on the text and values tables at three tile budgets, and tiles of exactly in_cap and in_cap + 16"""
    batch, labels, expects = _host()
    runs = []
    for spec_fn in (RT.text_spec, RT.values_spec):
        spec, table, ot = TG._table(spec_fn)
        want = TG.oracle(ot, table, batch)
        _bounds_hold(table, batch, want[1], spec_fn.__name__)
        for tile in (None, 16, 64):
            eng = TG._engine(spec_fn, tile)
            got = TG.gpu_packed(eng, table, batch)
            TG._same(got, want, "%s tile=%s" % (spec_fn.__name__, tile))
            if tile is None:
                _model_check(O.responses(got[0], got[1]), got[2], expects, labels, spec_fn.__name__)
            eng.close()
            runs.append(batch.n)
        small, keep = _small(batch, 52)
        w_small = TG.oracle(ot, table, small)
        done = 0
        for tile in (64, 256):
            eng = TG._engine(spec_fn, tile)
            for span in (TG.T * tile, TG.T * tile + 16):
                b = TG.tile_span_layout(small, span)
                if b is None:
                    continue
                got = TG.gpu_packed(eng, table, b)
                TG._same(got, w_small, "%s tile=%d span=%d" % (spec_fn.__name__, tile, span))
                _model_check(O.responses(got[0], got[1]), got[2], [expects[k] for k in keep], [labels[k] for k in keep],
                             "span %d" % span)
                done += 1
                runs.append(b.n)
            eng.close()
        assert done >= 3, done
    return "serve_device (packed, default and _values instances, tiles 16 / 64 / own, spans in_cap and in_cap + 16): " \
           "%d requests checked" % sum(runs)


def _gpu_slots():
    """gofr_serve_device_slots: the 4-CTA and 5-CTA instances on the text table, the wide instance on a one-shape table
    (checked to be the one in effect), the _values instance; a slot one byte short of a response"""
    batch, labels, expects = _host()
    counts = {}
    for spec_fn, forces in ((RT.text_spec, (4, 5)), (RT.values_spec, (0,))):
        spec, table, ot = TG._table(spec_fn)
        want = TG.oracle(ot, table, batch)
        eng = TG._engine(spec_fn)
        for force in forces:
            for slot in (512, 4096):
                TG.gpu_slots(eng, batch, slot, want, force=force)
                key = "%s ctas=%d" % (spec_fn.__name__, eng.slot_ctas())
                counts[key] = counts.get(key, 0) + batch.n
        # a slot exactly one byte shorter than some responses: those report their length and leave the slot untouched
        ln = np.diff(want[1].astype(np.int64))
        slot = int(next(L for L in sorted(set(ln.tolist())) if L % 16 == 1 and L > 100)) - 1
        assert (ln == slot + 1).any()
        TG.gpu_slots(eng, batch, slot, want)
        eng.close()
    # the wide instance: only H_PARAM_FORMAT routes of one shape
    wide = [(lab, r) for lab, r in RT.host_corpus() if r.path in (b"/hello", b"//hello")]
    wb, wl = RT.host_batch(wide)
    spec, table, ot = TG._table(RT.wide_spec)
    want = TG.oracle(ot, table, wb)
    eng = TG._engine(RT.wide_spec)
    assert eng.slot_ctas() == 4, "the one-shape table does not run the wide slot instance"
    for force in (4, 5):
        for slot in (512, 4096):
            TG.gpu_slots(eng, wb, slot, want, force=force)
            counts["wide_spec ctas=%d" % force] = counts.get("wide_spec ctas=%d" % force, 0) + wb.n
    eng.slot_ctas(0)
    out = TG.gpu_packed(eng, table, wb)
    TG._same(out, want, "wide table packed")
    wexp = [RT.expect(r.path, r.query, bool(r.flags & S.REQ_FORCE_QUERY),
                      routes=lambda p: ("param",) if p == b"/hello" else None) for _, r in wide]
    _model_check(O.responses(out[0], out[1]), out[2], wexp, wl, "wide table")
    eng.close()
    return "serve_device_slots: " + ", ".join("%s %d" % kv for kv in sorted(counts.items()))


def _gpu_host():
    """gofr_batch_submit: chunks of 1 and 129 requests, pinned and pageable"""
    batch, labels, expects = _host()
    spec, table, ot = TG._table(RT.text_spec)
    want = TG.oracle(ot, table, batch)
    eng = TG._engine(RT.text_spec)
    n = 0
    for pinned in (True, False):
        for chunk in (1, 129):
            got = TG.gpu_host(eng, table, batch, pinned, chunk)
            TG._same(got, want, "host pinned=%s chunk=%d" % (pinned, chunk))
            n += batch.n
    _model_check(O.responses(got[0], got[1]), got[2], expects, labels, "host")
    eng.close()
    return "serve_host (chunks 1 / 129, pinned and pageable): %d requests checked" % n


def _textproto_trim(v):
    """textproto.ReadMIMEHeader keeps a header value without its leading and trailing spaces and tabs"""
    return b"" if v is None else v.strip(b" \t")


def _gpu_conn():
    """gofr_conn_batch_submit_log on raw HTTP/1.1 messages, one per connection: columns and lines equal the oracle's, the
    responses and the lines' fields equal the model's"""
    from gofr_b200.engine import ConnLog
    msgs = RT.raw_corpus()
    buf, off = RT.raw_buffers(msgs)
    n = len(msgs)
    remotes = [b"192.0.2.1:1234", b" 10.0.0.9 ", b"\xc2\xa0r\xc2\xa0", b"", b"\xe3\x80\x80x"]
    rem = [remotes[k % len(remotes)] for k in range(n)]
    remote = np.frombuffer(b"".join(rem), dtype=np.uint8).copy()
    roff = np.concatenate([[0], np.cumsum([len(r) for r in rem])]).astype(np.uint32)
    start = np.full(n, CL.LOG_NS - 5000, dtype=np.int64)
    spec, table, _ = TG._table(RT.text_spec)
    want, _ = CL.model(spec, buf, off, CL.SEED, remote, roff, start)
    eng = TG._engine(RT.text_spec)
    checked = 0
    for pinned in (True, False):
        got = eng.serve_connections(buf, off, DATE, CL.SEED, pinned=pinned, log=ConnLog(remote, roff, start, CL.LOG_NS, CL.TZ))
        CL._check(got, want, "pinned=%s" % pinned)
        checked += n
    assert len(got.out_off) == n + 1
    _model_check(O.responses(got.out, got.out_off), got.meta, [RT.raw_expect(t) for _, t, _, _ in msgs], [m[0] for m in msgs],
                 "connections")
    lines = O.responses(got.log.out, got.log.log_off)
    assert len(lines) > n // 2
    for m, k in enumerate(got.log.log_req.tolist()):
        _, target, ua, xff = msgs[k]
        rec = S.LogRec(0, 0, 0, b"GET", _textproto_trim(ua), _textproto_trim(xff), rem[k], target)
        assert RT.log_segment(rec) in lines[m], (msgs[k][0], lines[m][:300], RT.log_segment(rec)[:200])
    eng.close()
    return "serve_connections with ConnLog: %d requests, %d lines checked" % (checked, 2 * len(lines))


def _gpu_log():
    """gofr_batch_submit_log and _slots_log: one RequestLog record per request of the host corpus"""
    recs = RT.log_corpus()
    corpus = RT.host_corpus()
    rnd = random.Random(7)
    picked = [corpus[rnd.randrange(len(corpus))] for _ in recs]
    batch, labels = RT.host_batch(picked)
    log = S.LogBatch.pack(recs)
    spec, table, _ = TG._table(RT.text_spec)
    want_resp, want_meta, want_lines = BL.expectation(spec, batch, log, date=DATE)
    eng = TG._engine(RT.text_spec)
    checked = 0
    for pinned in (True, False):
        r = eng.serve_host_log(batch, DATE, log, BL.LOG_NS, pinned=pinned)
        assert r.rc == 0 and r.responses() == want_resp and (r.meta == want_meta).all()
        assert r.line_list() == want_lines
        s = eng.serve_host_log(batch, DATE, log, BL.LOG_NS, slot_bytes=512, pinned=pinned)
        assert s.rc == 0 and s.line_list() == want_lines and (s.meta == want_meta).all()
        assert [x for x, L in zip(s.responses(512), s.out_len) if L <= 512] == [x for x in want_resp if len(x) <= 512]
        checked += 2 * batch.n
    lines = r.line_list()
    assert sum(1 for x in lines if x) > len(recs) // 2
    for i, rec in enumerate(recs):
        if lines[i]:
            assert RT.log_segment(rec) in lines[i], (i, lines[i][:300])
    _model_check(r.responses(), r.meta, [RT.host_expect(q) for _, q in picked], labels, "serve_host_log")
    eng.close()
    return "serve_host_log (packed and slots, pinned and pageable): %d requests and lines checked" % checked


CAMPAIGNS = {"packed": _gpu_packed, "slots": _gpu_slots, "host": _gpu_host, "connections": _gpu_conn, "log": _gpu_log}


def _gpu_main(name):
    import torch
    assert torch.cuda.is_available()
    t0 = time.perf_counter()
    msg = CAMPAIGNS[name]()
    print("%s (%.1f s)" % (msg, time.perf_counter() - t0))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CAMPAIGNS))
def test_gpu_campaign(name):
    r = subprocess.run([sys.executable, "-c", "import tests.test_gpu_request_text as t; t._gpu_main(%r)" % name], cwd=ROOT_DIR,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip())


def test_campaign_inputs_on_the_cpu():
    """what the campaigns need besides the GPU: the small-request tiles fit both budgets, a response one byte longer than
    a 16-byte multiple exists, the one-shape table is one the wide instance takes, the connection model accepts the corpus"""
    batch, _, _ = _host()
    small, _ = _small(batch, 52)
    for tile in (64, 256):
        assert TG.tile_span_layout(small, TG.T * tile) is not None and TG.tile_span_layout(small, TG.T * tile + 16) is not None
    spec, table, ot = TG._table(RT.text_spec)
    ln = np.diff(TG.oracle(ot, table, batch)[1].astype(np.int64))
    assert any(L % 16 == 1 and L > 100 for L in ln.tolist())
    import ctypes as C
    v = C.c_int(0)
    _abi.check(_abi.lib().gofr_table_slot_ctas(TG._table(RT.wide_spec)[1].handle, C.byref(v)), "gofr_table_slot_ctas")
    assert v.value == 4
    msgs = RT.raw_corpus()
    buf, off = RT.raw_buffers(msgs)
    n = len(msgs)
    want, lb = CL.model(spec, buf, off, CL.SEED, np.zeros(1, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.int64))
    assert len(want["meta"]) == n and lb.n > n // 2
