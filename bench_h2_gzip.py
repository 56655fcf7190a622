"""Times the gunzip passes of b2_h2_conn_set_gunzip on h2 / gRPC client connections.

A grpcio server with compression=Gzip (gRPC C-core) answers one small call and then K echo calls of --reply-bytes on one connection,
half of them compressible text and half random bytes; the test oracle's client drives that conversation and records the server's bytes.
Then --conns device client connections each pack the same requests and parse the whole recorded reply stream in ONE batch
(b2_h2_client_process_batch, one run per connection), once on connections with gunzip on and once with it off: the difference is the
cost of inflating.  Prints one JSON line: calls/s both ways, compressed and inflated GB/s of the difference, the same messages inflated
by the host's zlib on one core (a labelled comparison, not the device path), and the GPU's name, power limit and SM clock read in the
same run.  Writes nothing; needs a GPU.
    python bench_h2_gzip.py --conns 256 --replies 64 --reply-bytes 4096 --steps 20 --warmup 3"""
import argparse
import json
import os
import random
import socket
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def capture(k, nbytes):
    from _h2client_loop import ECHO, GRPC_EXTRA, OracleClients, run_socket
    rng = random.Random(1)
    text = b"".join(b"key_%d: value %d;\n" % (i, i % 7) for i in range(nbytes // 10 + 1))[:nbytes]
    bodies = [text if i % 2 == 0 else bytes(rng.randrange(256) for _ in range(nbytes)) for i in range(k)]
    from _h2gzip import gzip_grpcio_server
    srv, port = gzip_grpcio_server()
    rec = []
    batches = [[(ECHO, b"first", GRPC_EXTRA)], [(ECHO, b, GRPC_EXTRA) for b in bodies]]
    try:
        with socket.create_connection(("127.0.0.1", port)) as s:
            s.settimeout(60)
            done = run_socket(OracleClients(1, pending=k + 8, stream_bytes=nbytes + 8192), s, 0, batches, record=rec)
    finally:
        srv.stop(0)
    assert len(done) == k + 1 and all(c["error_code"] == 0 for c in done.values())
    compressed = [c["msg"] for c in done.values() if c["flags"] & 4]
    assert compressed, "the server compressed nothing"
    return batches, b"".join(e[1] for e in rec if e[0] == "recv"), compressed


def gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                                       # (reported, not fatal: the number is then unlabelled)
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, default=256)
    ap.add_argument("--replies", type=int, default=64)
    ap.add_argument("--reply-bytes", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import brpc_b200
    from brpc_b200.abi import H2_FLAG_GUNZIPPED, RUN_DT
    from _h2client_loop import DeviceClients

    batches, stream, compressed = capture(a.replies, a.reply_bytes)
    n = a.conns
    ctx = brpc_b200.Context(device=0, max_batch_bytes=max(32 << 20, len(stream) * n + 4096), max_msgs=max(1 << 14, n * (a.replies + 8)),
                            max_runs=max(512, n), max_resp_bytes=max(64 << 20, n * (a.replies + 1) * (a.reply_bytes + 2048) * 2))
    ctx.h2_configure(max_conns=n, max_pending=a.replies + 8, stream_bytes=((a.reply_bytes + 4096 + 15) // 16) * 16 + 4096)
    data = np.frombuffer(stream * n + b"\0", np.uint8)
    runs = np.zeros(n, RUN_DT)
    for k in range(n):
        runs[k]["offset"] = k * len(stream); runs[k]["length"] = len(stream); runs[k]["socket_id"] = k
    region = ((a.replies + 1) * (a.reply_bytes + 1024) * 3 + 65536 + 63) // 64 * 64
    out = np.empty(region * n, np.uint8)
    times = {True: [], False: []}
    n_gz = 0
    for step in range(a.warmup + a.steps):
        for on in (False, True):                                                 # alternating, so that both see the same conditions
            dev = DeviceClients(ctx, range(n))
            if on:
                for k in range(n):
                    ctx.h2_conn_set_gunzip(k)
            for b in batches:
                res = dev.pack([(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", body, e) for k in range(n) for p, body, e in b])
                assert all(st == 0 for st, _, _ in res)
            t0 = time.perf_counter()
            rs, calls, _ = ctx.h2_client_process_batch(data, runs, call_cap=n * (a.replies + 2), out=out)
            dt = time.perf_counter() - t0
            assert len(calls) == n * (a.replies + 1) and int((calls["error_code"] != 0).sum()) == 0
            if on:
                n_gz = int(((calls["flags"] & H2_FLAG_GUNZIPPED) != 0).sum())
                assert n_gz == n * len(compressed)
            if step >= a.warmup:
                times[on].append(dt)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    cbytes = sum(len(m) for m in compressed) * n
    ibytes = sum(len(zlib.decompress(m, 31)) for m in compressed) * n
    t0 = time.perf_counter()                                                     # host zlib, one core, the same messages once per connection
    for _ in range(n):
        for m in compressed:
            zlib.decompress(m, 31)
    host_s = time.perf_counter() - t0
    extra = med[True] - med[False]
    calls_per_batch = n * (a.replies + 1)
    print(json.dumps({"bench": "h2_client_process_batch + gunzip", "conns": n, "calls_per_batch": calls_per_batch, "reply_bytes": a.reply_bytes,
                      "compressed_msgs_per_batch": n_gz, "compressed_bytes": cbytes, "inflated_bytes": ibytes,
                      "median_s_gunzip_on": med[True], "median_s_gunzip_off": med[False],
                      "calls_per_s_gunzip_on": calls_per_batch / med[True], "calls_per_s_gunzip_off": calls_per_batch / med[False],
                      "inflate_s": extra, "inflate_compressed_gbytes_per_s": cbytes / extra / 1e9 if extra > 0 else None,
                      "inflate_inflated_gbytes_per_s": ibytes / extra / 1e9 if extra > 0 else None,
                      "host_zlib_one_core": {"s": host_s, "inflated_gbytes_per_s": ibytes / host_s / 1e9, "note": "zlib.decompress on the host, not the device path"},
                      "steps": a.steps, "gpu": gpu_facts()}))


if __name__ == "__main__":
    main()
