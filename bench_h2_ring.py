"""Latency of h2/gRPC on the ring (b2_h2_ring_submit + b2_h2_ring_wait on the resident k_h2_ring) against b2_h2_serve_batch, on two
contexts fed the same batches, alternated step by step in one process.  Every step checks that both give the same run statuses, messages,
spans and replies.  Shapes (connections x calls per connection per batch, message bytes):
  64 x 1 of 1 KiB, 64 x 1 of 4 KiB, 16 x 4 of 4 KiB — small rounds of clients that wait for each call;
  mixed: 64 x 1 of 1 KiB where one call in eight goes to an unknown path; the host answers those with b2_h2_pack_responses between
  batches on both contexts (inside the timed step), which retires k_h2_ring, so the relaunch cost shows.
Prints one JSON line: per shape the p50 / p99 wall-clock microseconds per batch of each (Python call overhead included, the same on both),
ring launches per 1 000 tickets and the median device phase stamps of the ring (b2_ring_phase_ns), with the GPU's name and power limit
read in the same run.  Writes nothing; needs a GPU.
    python bench_h2_ring.py --steps 2000 --warmup 200"""
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


def run_shape(conns, calls, size, mixed, steps, warmup):
    import brpc_b200 as b2
    import _h2serve as S
    import _h2traffic as T
    from brpc_b200.abi import H2_RESPONSE_DT, PinnedBuffer
    rng = random.Random(conns * 1000 + calls * 10 + size + mixed)
    msg_cap, out_cap, replies_cap = 1024, conns * (64 << 10), conns * (64 << 10)
    kw = dict(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=1024, max_resp_bytes=16 << 20)
    ring, batch = b2.Context(**kw), b2.Context(**kw)
    for c in (ring, batch):
        c.h2_configure(max_conns=conns, max_pending=16, stream_bytes=(64 << 10) + 4096)
        for k in range(conns):
            c.h2_conn_reset(k)
    ring.h2_ring_enable(1 << 20, msg_cap, out_cap, replies_cap)
    enc = [T.HpackEncoder(rng) for _ in range(conns)]
    sid = [1] * conns
    message = S.echo_request(bytes(rng.choice(b"abcdefghij") for _ in range(size)))
    window = T.frame(8, 0, 0, (calls * (size + 512)).to_bytes(4, "big"))
    pin = PinnedBuffer(1 << 20)
    host = np.frombuffer(b"application/grpcunimplemented\0", np.uint8)
    lat = {"ring": [], "batch": []}
    phases = []
    launches = 0
    n_host = 0

    def host_replies(ctx, msgs, conn_of):
        left = (msgs["flags"] & S.F_ANSWERED) == 0
        if not left.any():
            return []
        r = np.zeros(int(left.sum()), H2_RESPONSE_DT)
        r["conn"] = conn_of[left]; r["stream_id"] = msgs["stream_id"][left]; r["status_code"] = 200; r["flags"] = 1
        r["content_type_len"] = 16; r["grpc_status"] = 12; r["grpc_message_off"] = 16; r["grpc_message_len"] = 13
        return ctx.h2_pack_responses(host, r)

    for step in range(warmup + steps):
        chunks = []
        for k in range(conns):
            b = T.PREFACE + T.settings() + window if step == 0 else window
            for _ in range(calls):
                path = b"/other.Service/Echo" if mixed and rng.randrange(8) == 0 else b"/example.EchoService/Echo"
                b += b"".join(T.request_frames(rng, enc[k], sid[k], message=message, path=path)); sid[k] += 2
            chunks.append(b)
        data, runs = b2.make_runs(chunks)
        runs["socket_id"] = np.arange(conns)
        pin.array[:len(data)] = data
        view = pin.array[:len(data)]
        l0 = ring.ring_launches()
        t0 = time.perf_counter()
        ticket = ring.h2_ring_submit(None, runs, ptr=pin.ptr, nbytes=len(data))
        ra = ring.h2_ring_wait(ticket)
        ha = host_replies(ring, ra[1], np.repeat(np.arange(conns), ra[0]["n_msgs"]))
        ta = time.perf_counter() - t0
        la = ring.ring_launches() - l0
        ph = ring.ring_phase_ns(ticket)
        ra = tuple(x.copy() for x in ra)
        t0 = time.perf_counter()
        rb = batch.h2_serve_batch(view, runs, msg_cap=msg_cap, out_cap=out_cap, replies_cap=replies_cap)
        hb = host_replies(batch, rb[1], np.repeat(np.arange(conns), rb[0]["n_msgs"]))
        tb = time.perf_counter() - t0
        assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes() and ra[4].tobytes() == rb[4].tobytes(), step
        for s in rb[4]:
            o, n = int(s["off"]), int(s["len"])
            assert ra[3][o:o + n].tobytes() == rb[3][o:o + n].tobytes(), step
        assert ha == hb, step
        assert int(rb[4]["n_answered"].sum()) + len(hb) == conns * calls, step
        if step >= warmup:
            lat["ring"].append(ta * 1e6); lat["batch"].append(tb * 1e6)
            launches += la; phases.append(ph); n_host += len(hb)
    pct = lambda v, q: round(float(np.percentile(np.asarray(v), q)), 1)
    ph = np.median(np.asarray(phases, dtype=np.float64), axis=0) / 1e3
    out = {"conns": conns, "calls_per_conn": calls, "message_bytes": size, "mixed": bool(mixed), "batch_bytes": len(data),
           "ring": {"p50_us": pct(lat["ring"], 50), "p99_us": pct(lat["ring"], 99), "launches_per_1000_tickets": 1000.0 * launches / steps,
                    "phase_us_median": {"header_read": round(ph[0], 1), "bytes_pulled": round(ph[1], 1), "replies_packed": round(ph[2], 1),
                                        "results_pushed": round(ph[3], 1)}},
           "serve_batch": {"p50_us": pct(lat["batch"], 50), "p99_us": pct(lat["batch"], 99)},
           "host_answered_calls": n_host, "results_equal": True}
    ring.close(); batch.close(); pin.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    a = ap.parse_args()
    gpu = gpu_facts()
    shapes = [(64, 1, 1024, 0), (64, 1, 4096, 0), (16, 4, 4096, 0), (64, 1, 1024, 1)]
    res = [run_shape(c, k, s, m, a.steps, a.warmup) for c, k, s, m in shapes]
    print(json.dumps({"bench": "h2/gRPC on the ring vs b2_h2_serve_batch", "steps": a.steps, "gpu": gpu, "shapes": res}))


if __name__ == "__main__":
    main()
