"""Times b2_h2_serve_batch against the two-call path it replaces for device echo methods (b2_h2_process_batch, then b2_h2_pack_responses
of the records GpuH2Messenger builds), on the traffic of `bench.py --workload grpc_h2`: 256 connections x K unary calls of 4 KB per
batch, HPACK dynamic-table hits, the same bytes replayed every step with fresh stream ids.  Two contexts see the same batches; the paths
alternate step by step, and every step checks that both produced the same reply bytes.  Prints one JSON line with calls/s both ways and
the GPU's name and power limit read in the same run.  Writes nothing; needs a GPU.
    python bench_h2_serve.py --calls 8 --steps 30 --warmup 3"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


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
    ap.add_argument("--calls", type=int, default=8, help="calls per connection and batch (bench.py --workload grpc_h2 runs 8)")
    ap.add_argument("--msg-bytes", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import brpc_b200
    import _h2traffic as T
    from brpc_b200.abi import H2_FLAG_ANSWERED, H2_RESPONSE_DT, PinnedBuffer
    n, K, L = a.conns, a.calls, a.msg_bytes
    rng = random.Random(20260921)
    ctxs = {p: brpc_b200.Context(device=0, max_batch_bytes=64 << 20, max_msgs=1 << 16, max_runs=1024, max_resp_bytes=128 << 20) for p in ("serve", "two_calls")}
    message = bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz0123456789") for _ in range(L))
    first, batch = [], []
    for c in range(n):
        enc = T.HpackEncoder(rng); enc.fixed_mode = "auto"
        first.append(T.PREFACE + T.settings() + b"".join(T.request_frames(rng, enc, 1, message=message, chunk=16384)))
        calls = [T.request_frames(rng, enc, 3 + 2 * k, message=message, chunk=16384) for k in range(K)]
        batch.append(T.frame(8, 0, 0, (K * (L + 16)).to_bytes(4, "big")) + b"".join(b"".join(x) for x in calls))
    for ctx in ctxs.values():
        for c in range(n):
            ctx.h2_conn_reset(c)
    data_, runs = brpc_b200.make_runs(batch)
    pin_in = PinnedBuffer(len(data_)); data = pin_in.array; data[:] = data_
    out_bytes = n * (K * 1024 + 8192); rep_bytes = n * (K * (L + 512) + 4096)
    pin = {p: (PinnedBuffer(out_bytes), PinnedBuffer(rep_bytes)) for p in ctxs}
    pos = []
    for r_ in runs:
        p_ = int(r_["offset"]); end = p_ + int(r_["length"])
        while p_ < end:
            ln = (int(data[p_]) << 16) | (int(data[p_ + 1]) << 8) | int(data[p_ + 2]); pos.append(p_ + 5); p_ += 9 + ln
    pos = np.array(pos, dtype=np.int64)
    pos = pos[(data[pos] | data[pos + 1] | data[pos + 2] | data[pos + 3]) != 0]
    base_sid = ((data[pos].astype(np.int64) << 24) | (data[pos + 1].astype(np.int64) << 16) | (data[pos + 2].astype(np.int64) << 8) | data[pos + 3])

    def set_round(t):
        sid = base_sid + 2 * K * t
        data[pos] = (sid >> 24) & 255; data[pos + 1] = (sid >> 16) & 255; data[pos + 2] = (sid >> 8) & 255; data[pos + 3] = sid & 255

    ct = b"application/grpc"
    def serve(data, runs, k):
        rs, msgs, out, rep, spans = ctxs["serve"].h2_serve_batch(data, runs, msg_cap=n * (k + 2), out=pin["serve"][0].array, replies=pin["serve"][1].array)
        assert len(msgs) == n * k and np.all(msgs["flags"] & H2_FLAG_ANSWERED)
        return lambda: [bytes(rep[int(s["off"]):int(s["off"]) + int(s["len"])]) for s in spans]     # (read back after the timed window)

    def two_calls(data, runs, k):
        """what GpuH2Messenger does: the parse, then b2_h2_pack_responses of an echo record per call (the raw message, still on the device,
        and the request's own content-type value)"""
        ctx = ctxs["two_calls"]
        rs, msgs, out = ctx.h2_process_batch(data, runs, msg_cap=n * (k + 2), out=pin["two_calls"][0].array)
        assert len(msgs) == n * k
        hb = bytes(out[msgs[-1]["headers_off"]:msgs[-1]["headers_off"] + msgs[-1]["headers_len"]])   # (every call's records end the same way)
        r = np.zeros(len(msgs), dtype=H2_RESPONSE_DT)
        r["conn"] = runs["socket_id"][msgs["run_idx"]]; r["stream_id"] = msgs["stream_id"]; r["status_code"] = 200
        r["flags"] = 1 | 8 | np.where(msgs["flags"] & 16, 2, 4)
        r["content_type_off"] = msgs["headers_off"] + msgs["headers_len"] - (len(hb) - hb.rindex(ct)); r["content_type_len"] = len(ct)
        r["body_off"] = msgs["msg_off"]; r["body_len"] = msgs["msg_len"]
        pout, poffs, plens = ctx.h2_pack_responses(None, r, raw=True, out=pin["two_calls"][1].array)
        return lambda: [b"".join(bytes(pout[int(poffs[q * k + j]):int(poffs[q * k + j]) + int(plens[q * k + j])]) for j in range(k)) for q in range(n)]

    d0, r0 = brpc_b200.make_runs(first)
    assert serve(d0, r0, 1)() == two_calls(d0, r0, 1)()              # the first calls fill both connections' HPACK tables
    times = {"serve": [], "two_calls": []}
    for t in range(a.warmup + a.steps):
        set_round(t)
        t0 = time.perf_counter(); got = serve(data, runs, K); ts = time.perf_counter() - t0
        t0 = time.perf_counter(); want = two_calls(data, runs, K); tt = time.perf_counter() - t0
        assert got() == want(), t
        if t >= a.warmup:
            times["serve"].append(ts); times["two_calls"].append(tt)
    med = {p: sorted(v)[len(v) // 2] for p, v in times.items()}
    calls = n * K
    print(json.dumps({"bench": "b2_h2_serve_batch vs b2_h2_process_batch + b2_h2_pack_responses", "conns": n, "calls_per_batch": calls, "msg_bytes": L,
                      "median_s_serve": med["serve"], "median_s_two_calls": med["two_calls"],
                      "calls_per_s_serve": calls / med["serve"], "calls_per_s_two_calls": calls / med["two_calls"],
                      "speedup": med["two_calls"] / med["serve"], "steps": a.steps, "replies_equal": True, "gpu": gpu_facts()}))


if __name__ == "__main__":
    main()
