"""Latency of the stream pass on the ring (b2_stream_ring_enable) against the batch call with the same table, and against the ring without a
table on the echo part alone.  64 sockets x 16 connected streams with need_feedback; every batch carries one small DATA frame per socket
(each step a different stream of the socket) mixed with baidu_std echo requests.  Three contexts, alternated step by step in one process:
  (a) b2_ring_submit + b2_ring_wait on a context with the table and the opt-in;
  (b) b2_process_batch on a context with the same table (the only way before the opt-in);
  (c) b2_ring_submit + b2_ring_wait on a context without a table, on the same batch minus its stream frames.
Every step checks that (a) and (b) give the same descriptors, replies, stream messages, events and FEEDBACK bytes, and that (c) gives the
same echo replies.  Prints one JSON line: p50 / p99 wall-clock microseconds per batch and launches per batch for each, with the GPU's name
and power limit read in the same run.  Writes nothing; needs a GPU.
    python bench_stream_ring.py --steps 2000 --warmup 200"""
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
    ap.add_argument("--socks", type=int, default=64)
    ap.add_argument("--streams-per-sock", type=int, default=16)
    ap.add_argument("--echo-per-sock", type=int, default=2)
    ap.add_argument("--payload", type=int, default=128, help="bytes of each DATA frame")
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    a = ap.parse_args()
    import brpc_b200 as b2
    import _oracle as O
    import _streams as S
    from _compare import gather
    from _traffic import echo_frame
    from brpc_b200.abi import PinnedBuffer
    n_streams = a.socks * a.streams_per_sock
    ids = [(1 << 33) + 7919 * i for i in range(n_streams)]
    rng = random.Random(20261017)
    gpu = gpu_facts()
    kw = dict(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 14, max_runs=1024)
    ring, batch, plain = b2.Context(**kw), b2.Context(**kw), b2.Context(**kw)
    for c in (ring, batch):
        c.stream_configure(n_streams, 4096, 64 << 10)
        c.stream_open([(ids[i], ids[i] + 1, i % a.socks, 3) for i in range(n_streams)])
    ring.stream_ring_enable(64 << 10)
    pin, pin_echo = PinnedBuffer(1 << 20), PinnedBuffer(1 << 20)
    lat = {"a": [], "b": [], "c": []}
    launches = {"a": 0, "b": 0, "c": 0}
    for step in range(a.warmup + a.steps):
        chunks, echo_chunks = [], []
        for s in range(a.socks):
            e = [echo_frame(rng, step * a.socks + s + k, b"e" * rng.choice((16, 64, 200))) for k in range(a.echo_per_sock)]
            sid = ids[s + a.socks * (step % a.streams_per_sock)]
            chunks.append(e[0] + O.pack_stream_frame(sid, sid + 1, S.DATA, None, rng.randbytes(a.payload)) + b"".join(e[1:]))
            echo_chunks.append(b"".join(e))
        data, runs = b2.make_runs(chunks)
        edata, eruns = b2.make_runs(echo_chunks)
        pin.array[:len(data)] = data; pin_echo.array[:len(edata)] = edata
        l0 = ring.ring_launches()
        t0 = time.perf_counter()
        ra = ring.ring_wait(ring.ring_submit(None, runs, ptr=pin.ptr, nbytes=len(data)))
        ta = time.perf_counter() - t0
        sa = [x.copy() for x in ring.stream_results()]
        la = ring.ring_launches() - l0
        t0 = time.perf_counter()
        rb = batch.process_batch_ptr(pin.ptr, len(data), runs)
        tb = time.perf_counter() - t0
        sb = batch.stream_results()
        l0 = plain.ring_launches()
        t0 = time.perf_counter()
        rc = plain.ring_wait(plain.ring_submit(None, eruns, ptr=pin_echo.ptr, nbytes=len(edata)))
        tc = time.perf_counter() - t0
        lc = plain.ring_launches() - l0
        # (a) == (b): descriptors, replies, stream messages, events, FEEDBACK bytes; (c): the same echo replies
        for f in ("status", "frame_off", "resp_len", "correlation_id"):
            assert np.array_equal(ra[1][f], rb[1][f]), f
        assert np.array_equal(gather(ra[2], ra[1]["resp_off"], ra[1]["resp_len"]), gather(rb[2], rb[1]["resp_off"], rb[1]["resp_len"]))
        echo = ra[1]["status"] != 4
        assert np.array_equal(gather(ra[2], ra[1]["resp_off"][echo], ra[1]["resp_len"][echo]), gather(rc[2], rc[1]["resp_off"], rc[1]["resp_len"])), \
            (ra[1]["status"], rc[1]["status"], ra[1]["resp_len"], rc[1]["resp_len"])
        assert len(sa[0]) == len(sb[0]) == a.socks and len(sa[1]) == len(sb[1]) == a.socks
        key = lambda ev, ctrl: sorted((int(e["stream_id"]), int(e["flags"]), int(e["local_consumed"]), ctrl[int(e["fb_off"]):int(e["fb_off"]) + int(e["fb_len"])].tobytes()) for e in ev)
        assert key(sa[1], sa[3]) == key(sb[1], sb[3])
        assert sorted((int(m["stream_id"]), int(m["first_frame"]), int(m["len"])) for m in sa[0]) == sorted((int(m["stream_id"]), int(m["first_frame"]), int(m["len"])) for m in sb[0])
        if step >= a.warmup:
            lat["a"].append(ta * 1e6); lat["b"].append(tb * 1e6); lat["c"].append(tc * 1e6)
            launches["a"] += la; launches["b"] += rb[3]["n_launches"]; launches["c"] += lc
    pct = lambda v, q: float(np.percentile(np.asarray(v), q))
    out = {"bench": "stream pass on the ring", "socks": a.socks, "streams": n_streams, "frames_per_batch": len(ra[1]),
           "batch_bytes": len(data), "steps": a.steps, "results_equal": True, "gpu": gpu}
    for k, name in (("a", "ring_with_table"), ("b", "process_batch_with_table"), ("c", "ring_without_table_echo_only")):
        out[name] = {"p50_us": pct(lat[k], 50), "p99_us": pct(lat[k], 99), "launches_per_batch": launches[k] / a.steps}
    print(json.dumps(out))
    for c in (ring, batch, plain):
        c.close()
    pin.free(); pin_echo.free()


if __name__ == "__main__":
    main()
