"""Times b2_h2_client_process_batch: the receiving half of h2 / gRPC client connections on the device.

A grpcio server (gRPC C-core) answers one small call and then K echo calls of --reply-bytes on one connection; the test oracle's client
drives that conversation and records the server's bytes.  Then --conns device client connections each pack the same requests
(b2_h2_pack_requests) and parse the whole recorded reply stream in ONE batch (one run per connection): --conns x (K + 1) calls per batch.
Prints one JSON line: calls/s over the host-visible call (the input copy, the kernel and the copies back; it ends in a device
synchronise), with the GPU's name, power limit and max SM clock read in the same run.  Writes nothing; needs a GPU.
    python bench_h2_client_rx.py --conns 256 --replies 64 --reply-bytes 4096 --steps 20 --warmup 3"""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def capture(k, nbytes):
    from _h2client_loop import ECHO, GRPC_EXTRA, OracleClients, grpcio_server, run_socket
    srv, port = grpcio_server()
    rec = []
    batches = [[(ECHO, b"first", GRPC_EXTRA)], [(ECHO, bytes((i + j) & 0xff for j in range(nbytes)), GRPC_EXTRA) for i in range(k)]]
    try:
        with socket.create_connection(("127.0.0.1", port)) as s:
            s.settimeout(60)
            done = run_socket(OracleClients(1, pending=k + 8, stream_bytes=nbytes + 8192), s, 0, batches, record=rec)
    finally:
        srv.stop(0)
    assert len(done) == k + 1 and all(c["error_code"] == 0 for c in done.values())
    return batches, b"".join(e[1] for e in rec if e[0] == "recv")


def gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
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
    from brpc_b200.abi import RUN_DT
    from _h2client_loop import DeviceClients

    batches, stream = capture(a.replies, a.reply_bytes)
    n = a.conns
    ctx = brpc_b200.Context(device=0, max_batch_bytes=max(32 << 20, len(stream) * n + 4096), max_msgs=max(1 << 14, n * (a.replies + 8)),
                            max_runs=max(512, n), max_resp_bytes=max(64 << 20, n * (a.replies + 1) * (a.reply_bytes + 2048)))
    ctx.h2_configure(max_conns=n, max_pending=a.replies + 8, stream_bytes=((a.reply_bytes + 4096 + 15) // 16) * 16 + 4096)
    data = np.frombuffer(stream * n + b"\0", np.uint8)
    runs = np.zeros(n, RUN_DT)
    for k in range(n):
        runs[k]["offset"] = k * len(stream); runs[k]["length"] = len(stream); runs[k]["socket_id"] = k
    region = ((a.replies + 1) * (a.reply_bytes + 1024) * 2 + 65536 + 63) // 64 * 64
    out = np.empty(region * n, np.uint8)
    times = []
    for step in range(a.warmup + a.steps):
        dev = DeviceClients(ctx, range(n))                                       # fresh connections, the same requests on each
        for b in batches:
            res = dev.pack([(k, 1 | 8 | 16, p, b"127.0.0.1:1", b"application/grpc", body, e) for k in range(n) for p, body, e in b])
            assert all(st == 0 for st, _, _ in res)
        t0 = time.perf_counter()
        rs, calls, _ = ctx.h2_client_process_batch(data, runs, call_cap=n * (a.replies + 2), out=out)
        dt = time.perf_counter() - t0
        assert len(calls) == n * (a.replies + 1) and int((calls["error_code"] != 0).sum()) == 0
        assert all(int(r["consumed"]) == len(stream) for r in rs)
        if step >= a.warmup:
            times.append(dt)
    times.sort()
    med = times[len(times) // 2]
    print(json.dumps({"bench": "h2_client_process_batch", "conns": n, "calls_per_batch": n * (a.replies + 1), "reply_bytes": a.reply_bytes,
                      "batch_bytes": len(stream) * n, "median_s": med, "min_s": times[0], "calls_per_s": n * (a.replies + 1) / med,
                      "gbytes_per_s": len(stream) * n / med / 1e9, "steps": a.steps, "gpu": gpu_facts()}))


if __name__ == "__main__":
    main()
