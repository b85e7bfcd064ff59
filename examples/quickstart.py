"""Quickstart: the examples/http-server routes of the reference (examples/http-server/main.go:21-25) served by the GPU.

    python examples/quickstart.py            # needs an H100 (there is no CPU path)

Prints the wire bytes of three responses, then the RequestLog lines middleware.Logging would have written for them."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from gofr_b200 import spec as S  # noqa: E402
from gofr_b200.engine import Engine  # noqa: E402
from gofr_b200.table import Table  # noqa: E402

# app := gofr.New(); app.GET("/hello", ...); app.GET("/error", ...); app.Run()
spec = S.TableSpec(routes=[
    S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=b"name", s1=b"World", s2=b"Hello ", s3=b"!"),
    S.Route(S.M_GET, "/error", S.H_STATIC_ERROR, s0=b"some error occurred"),
])
eng = Engine(Table(spec), device=0)

batch = S.RequestBatch.pack([S.Req(S.M_GET, b"/hello"), S.Req(S.M_GET, b"/hello", b"name=gofr"), S.Req(S.M_GET, b"/error")])
date = S.http_date(1_700_000_000)
resp = eng.alloc_responses(batch.n, 4096)
eng.serve_device(eng.upload(batch), date, resp)
out, off, meta = resp.to_host()
for i in range(batch.n):
    print(f"--- request {i}: status {int(meta[i]) & 0xFFFF}, route {int(meta[i]) >> 16}")
    print(out[int(off[i]):int(off[i + 1])].tobytes().decode())

logs = S.LogBatch.pack([S.LogRec(1_700_000_000_000_000_000 + 1000 * i, 250_000 + i, 1_700_000_000_000_300_000, b"GET", b"curl/8.4.0",
                                 b"", b"127.0.0.1:5%04d" % i, [b"/hello", b"/hello?name=gofr", b"/error"][i], int(meta[i]) & 0xFFFF,
                                 trace_id=batch.trace_ids[i].tobytes()) for i in range(batch.n)])
d_out, d_off = eng.request_log_device(logs)
o = d_off.cpu().numpy().view(np.uint32)
print(d_out[:int(o[-1])].cpu().numpy().tobytes().decode(), end="")
eng.close()
