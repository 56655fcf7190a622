"""Times the stream pass (b2_stream_*: frames routed to open streams, messages reassembled, FEEDBACK written on the device) against the same
batch on a context without a stream table, and against the host doing the routing from the descriptors in Python / NumPy.
64 sockets x 16 streams, all connected with need_feedback; two workloads: one 4 KiB single-frame message per stream and batch, and 256 KiB
messages in 64 KiB segments (--big-streams of the streams carry one per batch).  The two contexts alternate step by step on the same
pinned bytes and every step checks that their descriptors are equal.  Prints one JSON line per workload with calls/s and device time both
ways, the stream kernels' times from b2_stage_times, the host routing time, and the GPU's name and power limit read in the same run.
Writes nothing; needs a GPU.
    python bench_streams.py --steps 30 --warmup 3"""
import argparse
import json
import os
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


def host_route(data, msgs, ids_sorted, local_consumed, feedback_frame, remote_of):
    """what a host has to do with the descriptors when there is no table: id lookup, frames grouped per stream in order, messages joined
    at the frame without continuation, one Consume + FEEDBACK per stream"""
    fr = np.nonzero(msgs["status"] == 4)[0]
    sid = msgs["correlation_id"][fr]
    slot = np.searchsorted(ids_sorted, sid)
    known = (slot < len(ids_sorted)) & (ids_sorted[np.minimum(slot, len(ids_sorted) - 1)] == sid)
    fr, slot = fr[known], slot[known]
    order = np.argsort(slot, kind="stable")
    fr, slot = fr[order], slot[order]
    off = msgs["frame_off"][fr].astype(np.int64) + 12 + msgs["meta_size"][fr]
    ln = (msgs["body_size"][fr] - msgs["meta_size"][fr]).astype(np.int64)
    last = (msgs["has_bits"][fr] & 256) == 0
    n_out, out, start = 0, [], 0
    ends = np.nonzero(last)[0]
    for e in ends:                                   # (traffic of this benchmark: every message completes inside the batch, in one stream)
        if e > start:
            out.append(np.concatenate([data[off[k]:off[k] + ln[k]] for k in range(start, e + 1)]))
        n_out += 1; start = e + 1
    consumed = np.bincount(slot, weights=ln, minlength=len(ids_sorted)).astype(np.int64)
    local_consumed += consumed
    fb = [feedback_frame(remote_of[s], int(ids_sorted[s]), int(local_consumed[s])) for s in np.nonzero(consumed)[0]]
    return n_out, out, fb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--socks", type=int, default=64)
    ap.add_argument("--streams-per-sock", type=int, default=16)
    ap.add_argument("--big-streams", type=int, default=128, help="streams that carry a 256 KiB message per batch in the segmented workload")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import brpc_b200
    import _oracle as O
    import _streams as S
    from brpc_b200.abi import PinnedBuffer
    n_streams = a.socks * a.streams_per_sock
    ids = np.arange(n_streams, dtype=np.int64) * 7919 + (1 << 33)
    remote = {i: int(ids[i]) + 1 for i in range(n_streams)}
    rng = np.random.default_rng(20261016)
    gpu = gpu_facts()
    for name, per_msg, seg, carriers in (("4 KiB single-frame", 4096, 4096, n_streams), ("256 KiB in 64 KiB segments", 256 << 10, 64 << 10, min(a.big_streams, n_streams))):
        chunks = [[] for _ in range(a.socks)]
        for s in range(carriers):
            sock = s % a.socks
            body = rng.integers(0, 256, per_msg, dtype=np.uint8).tobytes()
            parts = [body[o:o + seg] for o in range(0, per_msg, seg)]
            for k, p in enumerate(parts):
                chunks[sock].append(O.pack_stream_frame(int(ids[s]), remote[s], S.DATA, True if k < len(parts) - 1 else None, p))
        data_, runs = brpc_b200.make_runs([b"".join(c) for c in chunks])
        pin = PinnedBuffer(len(data_)); pin.array[:] = data_
        cap = max(64 << 20, len(data_) + (1 << 20))
        plain = brpc_b200.Context(device=0, max_batch_bytes=cap, max_msgs=1 << 16, max_runs=1024)
        table = brpc_b200.Context(device=0, max_batch_bytes=cap, max_msgs=1 << 16, max_runs=1024)
        table.stream_configure(n_streams, 256 << 10)
        table.stream_open([(int(ids[i]), remote[i], i % a.socks, 3) for i in range(n_streams)])
        local = np.zeros(n_streams, np.int64)
        t_plain, t_table, t_host, k_plain, k_table, stages = [], [], [], [], [], {}
        n_frames = sum(len(c) for c in chunks)
        for step in range(a.warmup + a.steps):
            t0 = time.perf_counter(); rp = plain.process_batch_ptr(pin.ptr, len(data_), runs); tp = time.perf_counter() - t0
            msgs_plain = rp[1].copy()
            t0 = time.perf_counter(); rt = table.process_batch_ptr(pin.ptr, len(data_), runs); sm, ev, out, ctrl, rc = table.stream_results(); tt = time.perf_counter() - t0
            assert np.array_equal(msgs_plain, rt[1]) and len(rt[1]) == n_frames, "descriptors differ"
            assert len(sm) == carriers and len(ev) == carriers and int(ev["consumed_bytes"].sum()) == carriers * per_msg and np.all(ev["fb_len"] > 0)
            t0 = time.perf_counter(); n_out, host_out, fb = host_route(pin.array, msgs_plain, ids, local, S.feedback_frame, remote); th = time.perf_counter() - t0
            assert n_out == carriers and len(fb) == carriers
            if step == 0:                            # the device's FEEDBACK bytes and reassembled bytes are the host's
                want = set(fb)
                assert {ctrl[int(e["fb_off"]):int(e["fb_off"]) + int(e["fb_len"])].tobytes() for e in ev} == want
                if host_out:
                    assert {out[int(m["off"]):int(m["off"]) + int(m["len"])].tobytes() for m in sm} == {h.tobytes() for h in host_out}
            if step >= a.warmup:
                t_plain.append(tp); t_table.append(tt); t_host.append(th); k_plain.append(rp[3]["kernel_ms"]); k_table.append(rt[3]["kernel_ms"])
                for nm, ms in table.stage_times():
                    if nm.startswith("stream_"):
                        stages.setdefault(nm, []).append(ms)
        med = lambda v: float(sorted(v)[len(v) // 2])
        print(json.dumps({"bench": "stream pass vs a context without a table", "workload": name, "streams": n_streams, "socks": a.socks,
                          "frames_per_batch": n_frames, "messages_per_batch": carriers, "batch_bytes": len(data_),
                          "median_call_s_plain": med(t_plain), "median_call_s_table": med(t_table), "calls_per_s_plain": 1 / med(t_plain),
                          "calls_per_s_table": 1 / med(t_table), "median_device_ms_plain": med(k_plain), "median_device_ms_table": med(k_table),
                          "stream_kernels_ms": {k: med(v) for k, v in stages.items()}, "median_host_routing_s": med(t_host),
                          "descriptors_equal": True, "steps": a.steps, "gpu": gpu}))
        plain.close(); table.close(); pin.free()


if __name__ == "__main__":
    main()
