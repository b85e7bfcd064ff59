#!/bin/bash
# emu_asan.sh — the kernels' per-request code (the __host__ __device__ functions tests/emu runs on the CPU) under
# AddressSanitizer + UBSan over the emulation tests: out-of-bounds reads past a row / message / path show up here.
set -e
cd "$(dirname "$0")/.."
g++ -O1 -g -std=c++17 -fPIC -shared -Wall -Wno-unknown-pragmas -fsanitize=address,undefined -fno-sanitize-recover=undefined \
    -o /tmp/libgofr_emu_asan.so tests/emu/emu_serve.cpp
g++ -O1 -g -std=c++17 -fPIC -shared -Wall -Wno-unknown-pragmas -fsanitize=address,undefined -fno-sanitize-recover=undefined \
    -o /tmp/libgofr_emu_http_frame_asan.so tests/emu/emu_http_frame.cpp
g++ -O1 -g -std=c++17 -fPIC -shared -Wall -Wno-unknown-pragmas -fsanitize=address,undefined -fno-sanitize-recover=undefined \
    -o /tmp/libgofr_emu_conn_log_asan.so tests/emu/emu_conn_log.cpp
g++ -O1 -g -std=c++17 -fPIC -shared -Wall -Wno-unknown-pragmas -fsanitize=address,undefined -fno-sanitize-recover=undefined \
    -o /tmp/libgofr_emu_conn_result_asan.so tests/emu/emu_conn_result.cpp
export GOFR_EMU_CONN_RESULT_LIB=/tmp/libgofr_emu_conn_result_asan.so
export GOFR_EMU_HTTP_FRAME_LIB=/tmp/libgofr_emu_http_frame_asan.so
export GOFR_EMU_CONN_LOG_LIB=/tmp/libgofr_emu_conn_log_asan.so
cp tests/emu/libgofr_emu.so /tmp/libgofr_emu_plain.so
cp /tmp/libgofr_emu_asan.so tests/emu/libgofr_emu.so
trap 'cp /tmp/libgofr_emu_plain.so tests/emu/libgofr_emu.so; touch tests/emu/libgofr_emu.so' EXIT
touch tests/emu/libgofr_emu.so
LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_values.py tests/test_proto_nested.py \
    tests/test_proto.py tests/test_http_parse.py tests/test_http_frame.py tests/test_route.py tests/test_slots.py tests/test_emu_parity.py tests/test_bind.py tests/test_bind_unmarshal.py \
    tests/test_result.py tests/test_reqlog.py tests/test_grpc.py tests/test_proto_presence.py tests/test_conn_log.py tests/test_conn_closures.py -x -q -m "not gpu" -p no:cacheprovider -W ignore
