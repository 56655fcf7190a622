"""Latency of a gRPC server's turn whose calls go (partly or all) to host methods, three ways on three contexts fed the same batches,
alternated step by step in one process:
  turns: b2_h2_ring_turn_submit + _wait for the runs, then the host's replies to the calls left in a reply-only turn (no relaunch);
  ring:  b2_h2_ring_submit + _wait, then b2_h2_pack_responses between tickets (which retires k_h2_ring; the next ticket relaunches it);
  batch: b2_h2_serve_batch, then b2_h2_pack_responses.
Every step checks that the three give the same run statuses, messages, spans, device replies and host reply frames.  The host answers a
call to the Host method with its message back (grpc-status 0) and a call to an unknown path with UNIMPLEMENTED; building those records
is inside each arm's timed step.  Shapes (connections x calls per connection per batch, message bytes):
  mixed: 64 x 1 of 1 KiB, one call in eight to an unknown path (bench_h2_ring.py's mixed shape);
  64 x 1 of 1 KiB and 16 x 4 of 4 KiB, every call to the Host method.
Prints one JSON line: per shape and arm the p50 / p99 wall-clock microseconds per step (Python call overhead included), ring launches per
1 000 tickets and the median device phase stamps, with the GPU's name and power limit read in the same run.  Writes nothing; needs a GPU.
    python bench_h2_ring_turns.py --steps 1000 --warmup 100"""
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

F_ANSWERED, F_BODY_IN_INPUT = 512, 16
CT, UNIMPL = b"application/grpc", b"unimplemented"


def host_replies(data, served, conns):
    """the host's replies to the calls the device left: (bytes, H2_RESPONSE_DT records indexing them)"""
    from brpc_b200.abi import H2_RESPONSE_DT
    rs, msgs, out = served[0], served[1], served[2]
    conn_of = np.repeat(np.arange(conns), rs["n_msgs"])
    left = np.flatnonzero((msgs["flags"] & F_ANSWERED) == 0)
    r = np.zeros(len(left), H2_RESPONSE_DT)
    parts, at = [CT, UNIMPL], len(CT) + len(UNIMPL)
    for j, i in enumerate(left):
        m = msgs[i]
        r[j]["conn"] = conn_of[i]; r[j]["stream_id"] = m["stream_id"]; r[j]["status_code"] = 200; r[j]["flags"] = 1; r[j]["content_type_len"] = len(CT)
        if int(m["method_idx"]) == 1:                                     # Host: the message back
            src = data if int(m["flags"]) & F_BODY_IN_INPUT else out
            body = src[int(m["msg_off"]):int(m["msg_off"]) + int(m["msg_len"])].tobytes()
            r[j]["body_off"] = at; r[j]["body_len"] = len(body); parts.append(body); at += len(body)
        else:
            r[j]["grpc_status"] = 12; r[j]["grpc_message_off"] = len(CT); r[j]["grpc_message_len"] = len(UNIMPL)
    return np.frombuffer(b"".join(parts) + b"\0" * 16, np.uint8), r


def run_shape(conns, calls, size, mixed, steps, warmup):
    import brpc_b200 as b2
    import _h2serve as S
    import _h2traffic as T
    import _oracle as O
    from brpc_b200.abi import H2_RESPONSE_DT, PinnedBuffer
    rng = random.Random(conns * 1000 + calls * 10 + size + mixed)
    msg_cap, out_cap, replies_cap = 1024, conns * (64 << 10), conns * (64 << 10)
    methods = (O.ECHO_METHOD, dict(O.ECHO_METHOD, method_name=b"Host", handler=0))
    kw = dict(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=1024, max_resp_bytes=16 << 20, methods=methods)
    arms = ("turns", "ring", "batch")
    ctx = {a: b2.Context(**kw) for a in arms}
    for c in ctx.values():
        c.h2_configure(max_conns=conns, max_pending=16, stream_bytes=(64 << 10) + 4096)
        for k in range(conns):
            c.h2_conn_reset(k)
    ctx["turns"].h2_ring_turn_enable(1 << 20, msg_cap, out_cap, replies_cap, 1024, 4 << 20)
    ctx["ring"].h2_ring_enable(1 << 20, msg_cap, out_cap, replies_cap)
    enc = [T.HpackEncoder(rng) for _ in range(conns)]
    sid = [1] * conns
    message = S.echo_request(bytes(rng.choice(b"abcdefghij") for _ in range(size)))
    window = T.frame(8, 0, 0, (calls * (size + 512)).to_bytes(4, "big"))
    pin, pin_rep = PinnedBuffer(1 << 20), PinnedBuffer(1 << 20)
    lat = {a: [] for a in arms}
    launches = {a: 0 for a in ("turns", "ring")}
    tickets = {a: 0 for a in ("turns", "ring")}
    phases = {"turns_runs": [], "turns_replies": [], "ring": []}
    n_host = 0

    for step in range(warmup + steps):
        chunks = []
        for k in range(conns):
            b = T.PREFACE + T.settings() + window if step == 0 else window
            for _ in range(calls):
                path = (b"/other.Service/Echo" if rng.randrange(8) == 0 else b"/example.EchoService/Echo") if mixed else b"/example.EchoService/Host"
                b += b"".join(T.request_frames(rng, enc[k], sid[k], message=message, path=path)); sid[k] += 2
            chunks.append(b)
        data, runs = b2.make_runs(chunks)
        runs["socket_id"] = np.arange(conns)
        pin.array[:len(data)] = data
        view = pin.array[:len(data)]
        got, took, ph, nt, nl = {}, {}, {}, {}, {}
        # turns: the runs, then a reply-only turn with what the host produced for them
        c = ctx["turns"]; l0 = c.ring_launches()
        t0 = time.perf_counter()
        t_runs = c.h2_ring_turn_submit(None, runs, np.zeros(0, H2_RESPONSE_DT), ptr=pin.ptr, nbytes=len(data))
        st, served, _ = c.h2_ring_turn_wait(t_runs)
        blob, recs = host_replies(view, served, conns)
        frames, t_rep = [], 0
        if len(recs):
            pin_rep.array[:len(blob)] = blob
            t_rep = c.h2_ring_turn_submit(None, runs[:0], recs, ptr=pin_rep.ptr, nbytes=len(blob))
            frames = c.h2_ring_turn_wait(t_rep)[2]
        took["turns"] = time.perf_counter() - t0
        assert st == 0, step
        got["turns"] = (tuple(x.copy() for x in served), frames)
        nl["turns"] = c.ring_launches() - l0; nt["turns"] = 2 if t_rep else 1
        ph["turns_runs"] = c.ring_phase_ns(t_runs); ph["turns_replies"] = c.ring_phase_ns(t_rep) if t_rep else None
        # ring: the ticket, then b2_h2_pack_responses between tickets
        c = ctx["ring"]; l0 = c.ring_launches()
        t0 = time.perf_counter()
        t_ring = c.h2_ring_submit(None, runs, ptr=pin.ptr, nbytes=len(data))
        served = c.h2_ring_wait(t_ring)
        blob, recs = host_replies(view, served, conns)
        served = tuple(x.copy() for x in served)
        frames = c.h2_pack_responses(blob, recs) if len(recs) else []
        took["ring"] = time.perf_counter() - t0
        got["ring"] = (served, frames)
        nl["ring"] = c.ring_launches() - l0; nt["ring"] = 1
        ph["ring"] = c.ring_phase_ns(t_ring)
        # batch: the two batch calls
        c = ctx["batch"]
        t0 = time.perf_counter()
        served = c.h2_serve_batch(view, runs, msg_cap=msg_cap, out_cap=out_cap, replies_cap=replies_cap)
        blob, recs = host_replies(view, served, conns)
        frames = c.h2_pack_responses(blob, recs) if len(recs) else []
        took["batch"] = time.perf_counter() - t0
        got["batch"] = (served, frames)
        rb, fb = got["batch"]
        for a in ("turns", "ring"):
            ra, fa = got[a]
            assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes() and ra[4].tobytes() == rb[4].tobytes(), (a, step)
            for s in rb[4]:
                o, n = int(s["off"]), int(s["len"])
                assert ra[3][o:o + n].tobytes() == rb[3][o:o + n].tobytes(), (a, step)
            assert fa == fb, (a, step)
        assert int(rb[4]["n_answered"].sum()) + len(fb) == conns * calls, step
        if step >= warmup:
            for a in arms:
                lat[a].append(took[a] * 1e6)
            for a in ("turns", "ring"):
                launches[a] += nl[a]; tickets[a] += nt[a]
            for k, v in ph.items():
                if v is not None:
                    phases[k].append(v)
            n_host += len(fb)
    pct = lambda v, q: round(float(np.percentile(np.asarray(v), q)), 1)

    def stamps(v):
        m = np.median(np.asarray(v, dtype=np.float64), axis=0) / 1e3
        return {"header_read": round(m[0], 1), "bytes_pulled": round(m[1], 1), "replies_packed": round(m[2], 1), "results_pushed": round(m[3], 1)}
    out = {"conns": conns, "calls_per_conn": calls, "message_bytes": size, "calls_to_host": "1 in 8, unknown path" if mixed else "all, Host method",
           "batch_bytes": len(data), "host_answered_calls": n_host, "results_equal": True}
    for a in arms:
        out[a] = {"p50_us": pct(lat[a], 50), "p99_us": pct(lat[a], 99)}
    for a in ("turns", "ring"):
        out[a]["launches_per_1000_tickets"] = 1000.0 * launches[a] / tickets[a]; out[a]["tickets"] = tickets[a]
    out["turns"]["phase_us_median_runs"] = stamps(phases["turns_runs"])
    if phases["turns_replies"]:
        out["turns"]["phase_us_median_reply_only"] = stamps(phases["turns_replies"])
    out["ring"]["phase_us_median"] = stamps(phases["ring"])
    for c in ctx.values():
        c.close()
    pin.free(); pin_rep.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    a = ap.parse_args()
    gpu = gpu_facts()
    shapes = [(64, 1, 1024, 1), (64, 1, 1024, 0), (16, 4, 4096, 0)]
    res = [run_shape(c, k, s, m, a.steps, a.warmup) for c, k, s, m in shapes]
    print(json.dumps({"bench": "h2/gRPC server turns with host replies: ring turns vs ring + b2_h2_pack_responses vs batch calls", "steps": a.steps,
                      "gpu": gpu, "shapes": res}))


if __name__ == "__main__":
    main()
