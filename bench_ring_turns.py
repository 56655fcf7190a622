"""Latency of a baidu_std server's turn whose calls go (partly or all) to a host method, three ways on three contexts fed the same
batches, alternated step by step in one process.  A step reads one batch of requests and sends the host's replies to the host-method
calls of the step before:
  turns: b2_ring_turn_submit + _wait, the runs and the replies in one ticket of k_ring<RingBody::replies>;
  ring:  b2_ring_submit + _wait for the runs, then b2_pack_responses for the replies, with the ring drained between them;
  batch: b2_process_batch, then b2_pack_responses.
Every step checks that the three give the same run statuses, messages, device replies and host reply frames.  The host answers a call
with its request's message back (the serialized EchoRequest is a valid EchoResponse); gathering those bodies and building the b2_reply
records is inside each arm's timed step.  Shapes (sockets x calls per socket per batch, message bytes):
  64 x 1 of 1 KiB, one call in eight to the host method;
  64 x 1 of 1 KiB, every call to the host method;
  8 x 3 of 4 KiB, every call to the host method, the replies snappy-compressed with CRC32C (16 x 4 of 4 KiB would be 256 KiB,
  above the 128 KiB b2_ring_submit serves).
Prints one JSON line: per shape and arm the p50 / p99 wall-clock microseconds per step (Python call overhead included), ring launches per
1 000 tickets and the median device phase stamps, with the GPU's name and power limit read in the same run.  Writes nothing; needs a GPU.
    python bench_ring_turns.py --steps 1000 --warmup 100"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_h2_ring import gpu_facts  # noqa: E402

B2_MSG_HOST = 2
OFF_FIELDS = ("error_text_off", "body_off", "attachment_off", "checksum_value_off", "extra_streams_off", "user_fields_off")


def host_calls(view, msgs):
    """the host-method calls of a batch: their correlation ids and the serialized request messages, back to back"""
    from _compare import gather
    host = msgs[msgs["status"] == B2_MSG_HOST]
    lens = host["body_size"].astype(np.int64) - host["meta_size"]
    bodies = gather(view, host["frame_off"].astype(np.int64) + 12 + host["meta_size"], lens)
    return host["correlation_id"].copy(), lens, bodies


def host_replies(calls, base, snappy_crc):
    """the b2_reply records answering `calls` with their messages back, the bodies placed at `base` of the bytes"""
    from brpc_b200.abi import REPLY_DT
    cids, lens, bodies = calls
    recs = np.zeros(len(cids), REPLY_DT)
    for f in OFF_FIELDS:
        recs[f] = base
    recs["correlation_id"] = cids
    recs["body_off"] = base + np.cumsum(lens) - lens; recs["body_len"] = lens
    if snappy_crc:
        recs["compress_type"] = 1; recs["checksum_type"] = 1
    return recs


def run_shape(socks, calls, size, host_share, snappy_crc, steps, warmup):
    import brpc_b200 as b2
    import _oracle as O
    from _compare import assert_same
    from brpc_b200.abi import PinnedBuffer
    rng = random.Random(socks * 1000 + calls * 10 + size + int(host_share * 8))
    methods = (O.ECHO_METHOD, dict(O.ECHO_METHOD, method_name=b"Host", handler=0))
    kw = dict(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=1024, max_resp_bytes=16 << 20, methods=methods)
    arms = ("turns", "ring", "batch")
    ctx = {a: b2.Context(**kw) for a in arms}
    ctx["turns"].ring_turn_enable(1 << 20, 1024, 4 << 20)
    ctx["ring"].ring_start()
    pin = {a: PinnedBuffer(1 << 20) for a in arms}
    prev = {a: None for a in arms}
    lat = {a: [] for a in arms}
    launches = {a: 0 for a in ("turns", "ring")}
    phases = {a: [] for a in ("turns", "ring")}
    n_host = 0
    message = bytes(rng.choice(b"abcdefghij") for _ in range(size))

    for step in range(warmup + steps):
        chunks = []
        for k in range(socks):
            chunks.append(b"".join(O.pack_echo_request(method=b"Host" if rng.random() < host_share else b"Echo", correlation_id=(step << 20) | (k << 8) | j,
                                                       message=message) for j in range(calls)))
        data, runs = b2.make_runs(chunks)
        n = len(data)
        for a in arms:
            pin[a].array[:n] = data
        got, took, nl = {}, {}, {}
        # turns: the runs and the replies to the step before's host calls, in one ticket
        c, p = ctx["turns"], pin["turns"]; l0 = c.ring_launches()
        t0 = time.perf_counter()
        recs = host_replies(prev["turns"], n, snappy_crc) if prev["turns"] else host_replies(([], [], b""), n, snappy_crc)
        if len(recs):
            blob = prev["turns"][2]; p.array[n:n + len(blob)] = blob
        t = c.ring_turn_submit(None, runs, recs, ptr=p.ptr, nbytes=n + (len(prev["turns"][2]) if prev["turns"] else 0))
        rs, msgs, resp, _, frames = c.ring_turn_wait(t)
        prev["turns"] = host_calls(p.array, msgs)
        took["turns"] = time.perf_counter() - t0
        got["turns"] = ((rs.copy(), msgs.copy(), resp.copy()), frames)
        nl["turns"] = c.ring_launches() - l0; ph_turns = c.ring_phase_ns(t)
        # ring: the ticket, then b2_pack_responses with the ring drained
        c, p = ctx["ring"], pin["ring"]; l0 = c.ring_launches()
        t0 = time.perf_counter()
        t = c.ring_submit(None, runs, ptr=p.ptr, nbytes=n)
        rs, msgs, resp, _ = c.ring_wait(t)
        calls_now = host_calls(p.array, msgs)
        frames = []
        if prev["ring"] and len(prev["ring"][0]):
            frames = c.pack_responses(np.frombuffer(prev["ring"][2].tobytes() + b"\0" * 16, np.uint8), host_replies(prev["ring"], 0, snappy_crc), out_cap=4 << 20)
        prev["ring"] = calls_now
        took["ring"] = time.perf_counter() - t0
        got["ring"] = ((rs.copy(), msgs.copy(), resp.copy()), frames)
        nl["ring"] = c.ring_launches() - l0; ph_ring = c.ring_phase_ns(t)
        # batch: the two batch calls
        c, p = ctx["batch"], pin["batch"]
        t0 = time.perf_counter()
        rs, msgs, resp, _ = c.process_batch_ptr(p.ptr, n, runs)
        calls_now = host_calls(p.array, msgs)
        res = (rs.copy(), msgs.copy(), resp.copy())
        frames = []
        if prev["batch"] and len(prev["batch"][0]):
            frames = c.pack_responses(np.frombuffer(prev["batch"][2].tobytes() + b"\0" * 16, np.uint8), host_replies(prev["batch"], 0, snappy_crc), out_cap=4 << 20)
        prev["batch"] = calls_now
        took["batch"] = time.perf_counter() - t0
        got["batch"] = (res, frames)
        rb, fb = got["batch"]
        for a in ("turns", "ring"):
            assert_same(got[a][0], rb, "%s step %d" % (a, step))
            assert got[a][1] == fb, (a, step)
        assert all(len(f) > 0 for f in fb), step
        if step >= warmup:
            for a in arms:
                lat[a].append(took[a] * 1e6)
            for a in ("turns", "ring"):
                launches[a] += nl[a]
            phases["turns"].append(ph_turns); phases["ring"].append(ph_ring)
            n_host += len(fb)
    pct = lambda v, q: round(float(np.percentile(np.asarray(v), q)), 1)

    def stamps(v):
        m = np.median(np.asarray(v, dtype=np.float64), axis=0) / 1e3
        return {"header_read": round(m[0], 1), "bytes_pulled": round(m[1], 1), "served_and_packed": round(m[2], 1), "results_pushed": round(m[3], 1)}
    out = {"sockets": socks, "calls_per_socket": calls, "message_bytes": size, "calls_to_host": "1 in 8" if host_share < 1 else "all",
           "host_replies": "snappy + CRC32C" if snappy_crc else "plain", "batch_bytes": n, "host_replies_sent": n_host, "results_equal": True}
    for a in arms:
        out[a] = {"p50_us": pct(lat[a], 50), "p99_us": pct(lat[a], 99)}
    for a in ("turns", "ring"):
        out[a]["launches_per_1000_tickets"] = 1000.0 * launches[a] / steps
        out[a]["phase_us_median"] = stamps(phases[a])
    for c in ctx.values():
        c.close()
    for p in pin.values():
        p.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    a = ap.parse_args()
    gpu = gpu_facts()
    shapes = [(64, 1, 1024, 0.125, False), (64, 1, 1024, 1.0, False), (8, 3, 4096, 1.0, True)]
    res = [run_shape(s, k, b, h, z, a.steps, a.warmup) for s, k, b, h, z in shapes]
    print(json.dumps({"bench": "baidu_std server turns with host replies: ring turns vs ring + b2_pack_responses vs batch calls", "steps": a.steps,
                      "gpu": gpu, "shapes": res}))


if __name__ == "__main__":
    main()
