"""Latency of a Stream producer's turn on the ring (b2_stream_ring_write_enable) against the same turn before it: a stream-ring ticket
followed by b2_stream_write.  A turn reads the peers' FEEDBACK frames, then writes what is queued.  Two contexts with identical tables,
alternated step by step in one process (which one goes first alternates too):
  (a) b2_stream_ring_submit + b2_stream_ring_wait;
  (b) b2_ring_submit + b2_ring_wait + b2_stream_write on a context with b2_stream_ring_enable.
Every step checks that (a) and (b) give the same descriptors, stream events, write results and frame bytes, and the same b2_stream_query
of every stream the step touched (of every stream at the end).  Workloads:
  feedback: 64 sockets x 16 windowed streams; per turn one FEEDBACK and one 4 KiB write per socket (each step a different stream of it);
  big:      16 streams; per turn one FEEDBACK and one 64 KiB write per stream, max_segment_size 16 KiB.
Prints one JSON line: p50 / p99 wall-clock microseconds per turn, launches per 1 000 turns, the ring's median phase stamps, and the GPU's
name, power limit and SM clocks read in the same run.  Writes nothing; needs a GPU.
    python bench_stream_write_ring.py --workload feedback --steps 2000 --warmup 200"""
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

SW_LAUNCHES = 7          # k_sw_route .. k_sw_copy: what one b2_stream_write launches


def gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                                       # (reported, not fatal: the number is then unlabelled)
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("feedback", "big"), default="feedback")
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    a = ap.parse_args()
    import brpc_b200 as b2
    import _streams as S
    from brpc_b200.abi import PinnedBuffer, STREAM_WRITE_DT
    if a.workload == "feedback":
        socks, per_sock, size, seg, window = 64, 16, 4096, 0, 1 << 30
    else:
        socks, per_sock, size, seg, window = 16, 1, 64 << 10, 16 << 10, 1 << 30
    n_streams = socks * per_sock
    ids = [(1 << 33) + 7919 * i for i in range(n_streams)]
    remote = {sid: sid + 1 for sid in ids}
    rng = random.Random(20261018)
    gpu = gpu_facts()
    kw = dict(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=1024, max_resp_bytes=8 << 20)
    ring, base = b2.Context(**kw), b2.Context(**kw)
    for c in (ring, base):
        c.stream_configure(n_streams, 4096, 64 << 10)
        c.stream_open([(sid, remote[sid], i % socks, 3, window) for i, sid in enumerate(ids)])
        c.stream_ring_enable(64 << 10)
    ring.stream_ring_write_enable(2 << 20, socks, 4 << 20, seg)
    pin = PinnedBuffer(4 << 20)
    out_b = np.empty(4 << 20, np.uint8)
    produced = {sid: 0 for sid in ids}
    lat = {"a": [], "b": []}
    launches = {"a": 0, "b": 0}
    phases = []
    for step in range(a.warmup + a.steps):
        touched = [ids[s + socks * (step % per_sock)] for s in range(socks)]
        chunks = [S.feedback_frame(sid, remote[sid], produced[sid]) for sid in touched]
        data, runs = b2.make_runs(chunks)
        payload_off = len(data)
        payloads = rng.randbytes(size * socks)
        n = payload_off + len(payloads)
        pin.array[:payload_off] = data
        pin.array[payload_off:n] = np.frombuffer(payloads, np.uint8)
        writes = np.zeros(socks, STREAM_WRITE_DT)
        writes["stream_id"] = touched
        writes["src_off"] = payload_off + size * np.arange(socks)
        writes["src_len"] = size
        res = {}
        for who in (("a", "b") if step % 2 == 0 else ("b", "a")):
            if who == "a":
                l0 = ring.ring_launches()
                t0 = time.perf_counter()
                t = ring.stream_ring_submit(None, runs, writes, ptr=pin.ptr, nbytes=n)
                ra = ring.stream_ring_wait(t)
                dt = time.perf_counter() - t0
                launches["a"] += ring.ring_launches() - l0 if step >= a.warmup else 0
                res["a"] = (ra[1].copy(), [x.copy() for x in ring.stream_results()], ra[4].copy(), ra[5].copy())
                if step >= a.warmup:
                    phases.append(ring.ring_phase_ns(t))
            else:
                l0 = base.ring_launches()
                t0 = time.perf_counter()
                rb = base.ring_wait(base.ring_submit(None, runs, ptr=pin.ptr, nbytes=payload_off))   # (b2_ring_submit: <= 128 KiB)
                sb = [x.copy() for x in base.stream_results()]
                wr, wo = base.stream_write(writes, pin.array[:n], seg, out=out_b)
                dt = time.perf_counter() - t0
                launches["b"] += base.ring_launches() - l0 + SW_LAUNCHES if step >= a.warmup else 0
                used = int(max(wr["out_off"].astype(np.int64) + (wr["out_len"].astype(np.int64) + 15) // 16 * 16)) if len(wr) else 0
                res["b"] = (rb[1].copy(), sb, wr.copy(), wo[:used].copy())
            if step >= a.warmup:
                lat[who].append(dt * 1e6)
        # (a) == (b): descriptors, stream events and messages, write results, frames, the touched streams' state
        (ma, sa, wa, oa), (mb, sbb, wb, ob) = res["a"], res["b"]
        assert ma.tobytes() == mb.tobytes()
        key = lambda ev: sorted((int(e["stream_id"]), int(e["flags"]), int(e["remote_consumed"]), int(e["local_consumed"])) for e in ev)
        assert key(sa[1]) == key(sbb[1]) and len(sa[0]) == len(sbb[0])
        assert wa.tobytes() == wb.tobytes() and oa.tobytes() == ob.tobytes()
        assert all(int(r["status"]) == 0 for r in wa), [int(r["status"]) for r in wa]
        for sid, r in zip(touched, wa):
            produced[sid] = int(r["produced"])
            assert ring.stream_query(sid) == base.stream_query(sid)
    for sid in ids:
        assert ring.stream_query(sid) == base.stream_query(sid)
    pct = lambda v, q: float(np.percentile(np.asarray(v), q))
    ph = np.median(np.asarray(phases, dtype=np.float64), axis=0) / 1e3
    out = {"bench": "stream producer turn on the ring", "workload": a.workload, "socks": socks, "streams": n_streams, "write_bytes": size,
           "writes_per_turn": socks, "max_segment_size": seg, "turn_bytes": n, "steps": a.steps, "results_equal": True, "gpu": gpu,
           "ring_phase_us_p50": {"header": ph[0], "pulled": ph[1], "served": ph[2], "pushed": ph[3]}}
    for k, name in (("a", "stream_ring_ticket"), ("b", "ring_ticket_then_stream_write")):
        out[name] = {"p50_us": pct(lat[k], 50), "p99_us": pct(lat[k], 99), "launches_per_1000": 1000.0 * launches[k] / a.steps}
    print(json.dumps(out))
    ring.ring_stop(); base.ring_stop()
    for c in (ring, base):
        c.close()
    pin.free()


if __name__ == "__main__":
    main()
