"""Times b2_stream_write (brpc::StreamWrite for a batch of writes: admission, DATA frames and payload copies on the device) on four
workloads: 1 024 streams x one 4 KiB write per call and 128 streams x one 256 KiB write in 64 KiB segments, each host-sourced and as a
streaming echo (b2_process_batch of bench_streams.py's traffic, then B2_STREAM_W_FROM_MSG writes of every completed message, read where
the receive pass left it).  Streams are connected and have no window.  The first step checks every result and frame byte against the
oracle of tests/_stream_write.py.  Prints one JSON line per workload: calls/s of the write call, its device time and each k_sw_* kernel
(b2_stage_times), the copy kernel's GB/s next to a device-to-device cudaMemcpyAsync of the same number of bytes measured in the same run,
a Python / NumPy host packer of the same frames, and the GPU's name and power limit read in the same run.  Writes nothing; needs a GPU.
    python bench_stream_write.py --steps 30 --warmup 3"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_streams import gpu_facts  # noqa: E402


def host_pack(W, remote, sids, payloads, seg):
    """the same frames packed on the host, write by write, into one buffer laid out as the device lays it out"""
    parts = []
    for sid, p in zip(sids, payloads):
        body = b"".join(W.cut_frames(remote[sid], sid, p, seg))
        parts.append(body); parts.append(b"\0" * ((-len(body)) % 16))
    return np.frombuffer(b"".join(parts), np.uint8)


def d2d_ms(nbytes, reps=20):
    import torch
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda"); dst = torch.empty_like(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record(); dst.copy_(src); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(sorted(ts)[len(ts) // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import brpc_b200
    import _oracle as O
    import _stream_write as W
    import _streams as S
    from brpc_b200.abi import PinnedBuffer, STREAM_W_FROM_MSG
    gpu = gpu_facts()
    rng = np.random.default_rng(20261016)
    med = lambda v: float(sorted(v)[len(v) // 2])
    for name, n_streams, per_msg, seg in (("1024 x 4 KiB", 1024, 4096, 0), ("128 x 256 KiB in 64 KiB segments", 128, 256 << 10, 64 << 10)):
        for echo in (False, True):
            ids = np.arange(n_streams, dtype=np.int64) * 7919 + (1 << 33)
            remote = {int(ids[i]): int(ids[i]) + 1 for i in range(n_streams)}
            ctx = brpc_b200.Context(device=0, max_batch_bytes=64 << 20, max_msgs=1 << 16, max_runs=1024, max_resp_bytes=96 << 20)
            ctx.stream_configure(2 * n_streams, 256 << 10)
            ctx.stream_open([(int(ids[i]), remote[int(ids[i])], i % 64, 3) for i in range(n_streams)])
            payloads = [rng.integers(0, 256, per_msg, dtype=np.uint8).tobytes() for _ in range(n_streams)]
            sids = [int(i) for i in ids]
            if echo:                              # bench_streams.py's traffic: the peers' frames, one message per stream and batch
                chunks = [[] for _ in range(64)]
                for s, p in enumerate(payloads):
                    sub = [p[o:o + (seg or per_msg)] for o in range(0, per_msg, seg or per_msg)]
                    for k, part in enumerate(sub):
                        chunks[s % 64].append(O.pack_stream_frame(remote[sids[s]], sids[s], S.DATA, True if k < len(sub) - 1 else None, part))
                data_, runs = brpc_b200.make_runs([b"".join(c) for c in chunks])
                pin = PinnedBuffer(len(data_)); pin.array[:] = data_
                # (the receiving side is the peer's id: a second table entry per stream so the echo goes back on the forward stream)
                ctx.stream_open([(remote[s], s, 99, 3) for s in sids])
            else:
                data = np.frombuffer(b"".join(payloads), np.uint8)
                pin = PinnedBuffer(len(data)); pin.array[:] = data
                writes = [(sids[s], 0, s * per_msg, per_msg) for s in range(n_streams)]
            out = PinnedBuffer(sum(W.bound(per_msg, seg) for _ in range(n_streams)))
            t_call, t_dev, t_host, stages = [], [], [], {}
            for step in range(a.warmup + a.steps):
                if echo:
                    ctx.process_batch_ptr(pin.ptr, len(data_), runs)
                    sm = ctx.stream_results()[0]
                    assert len(sm) == n_streams
                    writes = [(int(m["stream_id"]) - 1, STREAM_W_FROM_MSG, k, 0) for k, m in enumerate(sm)]
                    src_ids = [int(m["stream_id"]) - 1 for m in sm]
                    src_payloads = [payloads[sids.index(s)] for s in src_ids] if step == 0 else None
                t0 = time.perf_counter()
                res, _ = ctx.stream_write(writes, None if echo else pin.array, seg, out=out.array)
                tc = time.perf_counter() - t0
                assert np.all(res["status"] == 0)
                if step == 0:                     # every result and frame byte is the oracle's
                    orc = W.WriteOracle()
                    for s in sids:
                        orc.open(s, remote[s], sids.index(s) % 64, True, True)
                    want, want_out = orc.write_many(list(zip(src_ids, src_payloads)) if echo else list(zip(sids, payloads)), seg)
                    for r, w in zip(res, want):
                        assert (int(r["status"]), int(r["n_frames"]), int(r["out_off"]), int(r["out_len"]), int(r["host_socket_id"])) == \
                               (w["status"], w["n_frames"], w["out_off"], w["out_len"], w["host_socket_id"])
                        assert out.array[w["out_off"]:w["out_off"] + w["out_len"]].tobytes() == b"".join(w["frames"])
                if step >= a.warmup:
                    t_call.append(tc)
                    st = [(nm, ms) for nm, ms in ctx.stage_times() if nm.startswith("stream_write_")]
                    t_dev.append(sum(ms for _, ms in st))
                    for nm, ms in st:
                        stages.setdefault(nm, []).append(ms)
                    if not echo:
                        t0 = time.perf_counter(); host_pack(W, remote, sids, payloads, seg); t_host.append(time.perf_counter() - t0)
            total = n_streams * per_msg
            copy_ms = med(stages["stream_write_copy"])
            ref_ms = d2d_ms(total)
            print(json.dumps({"bench": "b2_stream_write", "workload": name + (" echo (FROM_MSG)" if echo else " host-sourced"), "writes_per_call": n_streams,
                              "payload_bytes_per_call": total, "max_segment_size": seg or W.DEFAULT_SEGMENT, "frames_per_call": int(res["n_frames"].sum()),
                              "median_call_s": med(t_call), "calls_per_s": 1 / med(t_call), "median_device_ms": med(t_dev),
                              "write_kernels_ms": {k: med(v) for k, v in stages.items()}, "copy_GB_per_s": total / copy_ms / 1e6,
                              "d2d_memcpy_ms_same_bytes": ref_ms, "d2d_memcpy_GB_per_s": total / ref_ms / 1e6,
                              "median_host_pack_s": med(t_host) if t_host else None, "bytes_checked_vs_oracle": True, "steps": a.steps, "gpu": gpu}))
            ctx.close(); pin.free(); out.free()


if __name__ == "__main__":
    main()
