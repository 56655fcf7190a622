"""Latency of h2/gRPC client connections on the ring (b2_h2_client_ring_submit + _wait on the resident k_h2_client_ring) against the two
batch calls (b2_h2_client_process_batch + b2_h2_pack_requests), as two closed loops alternated step by step in one process.  Each loop is
a client context and a server context whose server runs k_h2_ring with device echo (b2_h2_ring_*); a step is one round: the client reads
the server's replies to the previous round and sends the next requests (one ticket, or the two batch calls), then the server answers
them.  Only what the kernels wrote goes over the wire.  Every step checks that both clients give the same run statuses, calls, call
messages, control bytes, request results and frames, and that every call the client did not abandon ends with error 0 and its echo.
Shapes (connections x calls per connection per round, message bytes):
  64 x 1 of 1 KiB, 64 x 1 of 4 KiB, 16 x 4 of 4 KiB;
  mixed: 64 x 1 of 1 KiB where one call in eight is abandoned between rounds (b2_h2_client_abandon_streams on both clients, inside the
  timed client half), which retires k_h2_client_ring, so the relaunch cost shows.
Prints one JSON line: per shape the p50 / p99 wall-clock microseconds of the client half and of the whole round for each arm (Python call
overhead included, the same on both), ring launches per 1 000 client tickets and the median device phase stamps of the client ring
(b2_ring_phase_ns), with the GPU's name, power limit and SM clocks read in the same run.  Writes nothing; needs a GPU.
    python bench_h2_client_ring.py --steps 1000 --warmup 100"""
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

GRPC_EXTRA = ((b"te", b"trailers"), (b"grpc-accept-encoding", b"identity,gzip"))
PATH, AUTHORITY, CT = b"/example.EchoService/Echo", b"127.0.0.1:8000", b"application/grpc"
F_BODY_IN_INPUT = 16


def ticket_input(to_cli, bodies):
    """the client's input of one round: the server's bytes per connection (runs) and a request per (conn, body), fields behind them"""
    from brpc_b200.abi import H2_REQUEST_DT, RUN_DT
    live = [k for k, b in enumerate(to_cli) if b]
    runs = np.zeros(len(live), RUN_DT); parts = []; at = 0
    for r, k in enumerate(live):
        runs[r]["offset"] = at; runs[r]["length"] = len(to_cli[k]); runs[r]["socket_id"] = k; parts.append(to_cli[k]); at += len(to_cli[k])
    extra = b"".join(len(n).to_bytes(2, "little") + len(v).to_bytes(2, "little") + n + v for n, v in GRPC_EXTRA)
    reqs = np.zeros(len(bodies), H2_REQUEST_DT)
    for i, (k, body) in enumerate(bodies):
        offs = []
        for piece in (PATH, AUTHORITY, CT, body, extra):
            offs.append(at); parts.append(piece); at += len(piece)
        reqs[i] = (k, 1 | 8 | 16, offs[0], len(PATH), offs[1], len(AUTHORITY), offs[2], len(CT), offs[3], len(body), offs[4], len(extra))
    return np.frombuffer(b"".join(parts) + b"\0" * 16, np.uint8), runs, reqs


class Loop:
    """a client context (on the ring or on the batch calls) and a server context on k_h2_ring"""
    def __init__(self, ring, conns, calls):
        import brpc_b200 as b2
        from brpc_b200.abi import PinnedBuffer
        kw = dict(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=1024, max_resp_bytes=16 << 20)
        self.ring, self.conns = ring, conns
        self.cli, self.srv = b2.Context(**kw), b2.Context(**kw)
        for c, reset in ((self.cli, self.cli.h2_client_conn_reset), (self.srv, self.srv.h2_conn_reset)):
            c.h2_configure(max_conns=conns, max_pending=64, stream_bytes=(64 << 10) + 4096)
            for k in range(conns):
                reset(k)
        self.call_cap, self.out_cap, self.req_out_cap = 1024, conns * (64 << 10), 4 << 20
        self.srv.h2_ring_enable(1 << 20, 1024, conns * (64 << 10), conns * (64 << 10))
        if ring:
            self.cli.h2_client_ring_enable(1 << 20, self.call_cap, self.out_cap, conns * calls, self.req_out_cap)
        self.pin = PinnedBuffer(1 << 20)
        self.to_cli = [b""] * conns
        self.last = 0

    def client(self, data, runs, reqs):
        """the client half; returns (run_status, calls, out, request results, frames) as copies"""
        if self.ring:
            self.pin.array[:len(data)] = data
            self.last = self.cli.h2_client_ring_submit(None, runs, reqs, ptr=self.pin.ptr, nbytes=len(data))
            rs, calls, out, res, frames = self.cli.h2_client_ring_wait(self.last)
            return rs.copy(), calls.copy(), out, res.copy(), frames
        rs, calls, out = self.cli.h2_client_process_batch(data, runs, call_cap=self.call_cap, out_cap=self.out_cap) if len(runs) else \
            (runs[:0], np.zeros(0), None)
        res, frames = self.cli.h2_pack_requests(data, reqs, out_cap=self.req_out_cap)
        return rs, calls, out, res, frames

    def server(self, to_srv):
        """the server half: one k_h2_ring ticket over what the client wrote; its control bytes and replies go back to the client"""
        from brpc_b200.abi import RUN_DT
        live = [k for k, b in enumerate(to_srv) if b]
        runs = np.zeros(len(live), RUN_DT); at = 0
        for r, k in enumerate(live):
            runs[r]["offset"] = at; runs[r]["length"] = len(to_srv[k]); runs[r]["socket_id"] = k; at += len(to_srv[k])
        data = np.frombuffer(b"".join(to_srv[k] for k in live) + b"\0" * 16, np.uint8)
        rs, msgs, out, replies, spans = self.srv.h2_ring_wait(self.srv.h2_ring_submit(data, runs))
        assert int(spans["n_answered"].sum()) == len(msgs) and (rs["consumed"] == runs["length"]).all()
        for r, k in enumerate(live):
            s, sp = rs[r], spans[r]
            self.to_cli[k] += out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes() + \
                replies[int(sp["off"]):int(sp["off"]) + int(sp["len"])].tobytes()

    def close(self):
        self.cli.close(); self.srv.close(); self.pin.free()


def client_view(got, data):
    """what must be equal between the two clients: statuses, call records and messages, control bytes, request results and frames"""
    rs, calls, out, res, frames = got
    ctrl = [out[int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes() for s in rs]
    msgs = [((data if int(c["flags"]) & F_BODY_IN_INPUT else out)[int(c["msg_off"]):int(c["msg_off"]) + int(c["msg_len"])]).tobytes() for c in calls]
    return rs.tobytes(), calls.tobytes() if len(calls) else b"", ctrl, msgs, res.tobytes(), frames


def run_shape(conns, calls, size, mixed, steps, warmup):
    import _h2serve as S
    from brpc_b200.abi import H2_CALL_DT, H2_REQUEST_RESULT_DT
    rng = random.Random(conns * 1000 + calls * 10 + size + mixed)
    body = S.echo_request(bytes(rng.choice(b"abcdefghij") for _ in range(size)))
    arms = {"ring": Loop(True, conns, calls), "batch": Loop(False, conns, calls)}
    lat = {a: {"client": [], "round": []} for a in arms}
    phases = []; launches = 0; n_calls = 0; n_abandoned = 0
    open_sids, abandoned = set(), set()                              # (conn, stream id) sent and not yet ended; given up on
    for step in range(warmup + steps):
        A, B = arms["ring"], arms["batch"]
        assert A.to_cli == B.to_cli, step
        data, runs, reqs = ticket_input(A.to_cli, [(k, body) for k in range(conns) for _ in range(calls)])
        gone = [key for key in sorted(open_sids) if mixed and rng.randrange(8) == 0]
        abandoned.update(gone)
        views = {}
        for name, L in arms.items():
            l0 = L.cli.ring_launches()
            t0 = time.perf_counter()
            for k, sid in gone:                                      # given up on between rounds (AddAbandonedStream)
                L.cli.h2_client_abandon_streams(k, [sid])
            got = L.client(data, runs, reqs)
            t1 = time.perf_counter()
            L.to_cli = [b""] * conns
            for r, s in zip(runs, got[0]):
                k = int(r["socket_id"])
                L.to_cli[k] = bytes(data[int(r["offset"]) + int(s["consumed"]):int(r["offset"]) + int(r["length"])])
            to_srv = [b""] * conns
            for r, s in zip(runs, got[0]):
                to_srv[int(r["socket_id"])] += got[2][int(s["ctrl_off"]):int(s["ctrl_off"]) + int(s["ctrl_len"])].tobytes()
            for q, f in zip(reqs, got[4]):
                to_srv[int(q["conn"])] += f
            views[name] = client_view(got, data)
            t2 = time.perf_counter()
            L.server(to_srv)
            t3 = time.perf_counter()
            if step >= warmup:
                lat[name]["client"].append((t1 - t0) * 1e6); lat[name]["round"].append((t1 - t0 + t3 - t2) * 1e6)
                if L.ring:
                    launches += L.cli.ring_launches() - l0; phases.append(L.cli.ring_phase_ns(L.last))
        assert views["ring"] == views["batch"], step
        res = np.frombuffer(views["ring"][4], H2_REQUEST_RESULT_DT)
        assert (res["status"] == 0).all(), step
        for c, m in zip(np.frombuffer(views["ring"][1], H2_CALL_DT), views["ring"][3]):
            key = (int(runs[int(c["run_idx"])]["socket_id"]), int(c["stream_id"]))
            assert key in open_sids and int(c["error_code"]) == 0 and m == body, (step, key)
            open_sids.discard(key); n_calls += 1
        open_sids -= abandoned                                       # (their replies were in this ticket: reported above, or dropped)
        n_abandoned += len(gone); abandoned.clear()
        open_sids.update((int(q["conn"]), int(r["stream_id"])) for q, r in zip(reqs, res))
    pct = lambda v, q: round(float(np.percentile(np.asarray(v), q)), 1)
    ph = np.median(np.asarray(phases, dtype=np.float64), axis=0) / 1e3
    out = {"conns": conns, "calls_per_conn": calls, "message_bytes": size, "mixed": bool(mixed)}
    for name in arms:
        out[name] = {"client_p50_us": pct(lat[name]["client"], 50), "client_p99_us": pct(lat[name]["client"], 99),
                     "round_p50_us": pct(lat[name]["round"], 50), "round_p99_us": pct(lat[name]["round"], 99)}
    out["ring"]["launches_per_1000_tickets"] = 1000.0 * launches / steps
    out["ring"]["phase_us_median"] = {"header_read": round(ph[0], 1), "bytes_pulled": round(ph[1], 1), "requests_packed": round(ph[2], 1),
                                      "results_pushed": round(ph[3], 1)}
    out.update({"calls_ended": n_calls, "calls_abandoned": n_abandoned, "results_equal": True})
    for L in arms.values():
        L.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    a = ap.parse_args()
    gpu = gpu_facts()
    shapes = [(64, 1, 1024, 0), (64, 1, 4096, 0), (16, 4, 4096, 0), (64, 1, 1024, 1)]
    res = [run_shape(c, k, s, m, a.steps, a.warmup) for c, k, s, m in shapes]
    print(json.dumps({"bench": "h2/gRPC client connections on the ring vs b2_h2_client_process_batch + b2_h2_pack_requests", "steps": a.steps,
                      "gpu": gpu, "shapes": res}))


if __name__ == "__main__":
    main()
