"""Latency of baidu_std client connections on the ring (b2_client_ring_submit + _wait on the resident k_ring<true>) against today's path on
the same context (b2_ring_submit + _wait for the replies, then b2_pack_requests), as two closed loops alternated step by step in one
process.  Each loop is a client context and a server context whose server runs k_ring with device echo (b2_ring_*); a step is one round:
the client reads the server's replies to the previous round and sends the next requests (one ticket, or the ring ticket and the batch
call), then the server answers them.  Only what the kernels wrote goes over the wire.  Every step checks that both clients give the same
run statuses, descriptors and request frames, and that every reply carries error 0 and the correlation id of a request sent the round
before.
Shapes (sockets x requests per socket per round, message bytes):
  64 x 1 of 1 KiB (the client turn of BASELINE config 2: about 133 KB of bytes, above b2_ring_submit's 128 KiB), 1 x 64 of 1 KiB;
  64 x 1 of 4 KiB with snappy + CRC32C requests (the server replies snappy + CRC32C too, so that the replies fit b2_ring_submit).
Prints one JSON line: per shape the p50 / p99 wall-clock microseconds of the client half and of the whole round for each arm (Python call
overhead included, the same on both), ring launches per 1 000 client tickets and the median device phase stamps of the client ring
(b2_ring_phase_ns), with the GPU's name, power limit and SM clocks read in the same run.  Writes nothing; needs a GPU.
    python bench_client_ring.py --steps 2000 --warmup 200"""
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


def turn_input(to_cli, payloads, socks, compress, step):
    """the client's input of one round: the replies per socket (B2_RUN_CLIENT runs), then the requests' payloads behind them"""
    from brpc_b200.abi import REQUEST_DT, RUN_DT
    live = [k for k, b in enumerate(to_cli) if b]
    runs = np.zeros(len(live), RUN_DT); parts = []; at = 0
    for r, k in enumerate(live):
        runs[r] = (k, at, len(to_cli[k]), -1, 1)
        parts.append(to_cli[k] + b"\0" * (-len(to_cli[k]) % 16)); at += len(parts[-1])
    runs_end = at
    reqs = np.zeros(len(payloads), REQUEST_DT)
    for i, p in enumerate(payloads):
        reqs[i] = (0, 1, 0, 0, (step << 16) | i, step, compress, compress, 0, at, len(p), 0, 0, 0)
        parts.append(p); at += len(p)
    return np.frombuffer(b"".join(parts) + b"\0" * 16, np.uint8), runs, reqs, runs_end


class Loop:
    """a client context (on the client ring, or on k_ring plus b2_pack_requests) and a server context on k_ring"""
    def __init__(self, ring, socks, server_methods):
        import brpc_b200 as b2
        from brpc_b200.abi import PinnedBuffer
        kw = dict(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=512, max_resp_bytes=16 << 20)
        self.ring, self.socks = ring, socks
        self.cli, self.srv = b2.Context(**kw), b2.Context(methods=server_methods, **kw)
        self.req_out_cap = 4 << 20
        if ring:
            self.cli.client_ring_enable(1 << 20, 1024, self.req_out_cap)
        self.srv.ring_start()
        self.pin = PinnedBuffer(1 << 20)
        self.to_cli = [b""] * (max(socks) + 1)
        self.last = 0

    def client(self, data, runs, reqs, runs_end):
        """the client half; returns (run_status, msgs, resp, frames) as copies"""
        n = len(data)
        self.pin.array[:n] = data
        if self.ring:
            self.last = self.cli.client_ring_submit(None, runs, reqs, ptr=self.pin.ptr, nbytes=n)
            rs, msgs, resp, _, frames = self.cli.client_ring_wait(self.last)
            return rs.copy(), msgs.copy(), resp.copy(), frames
        rs, msgs, resp = runs[:0], None, None
        if len(runs):
            rs, msgs, resp, _ = self.cli.ring_wait(self.cli.ring_submit(None, runs, ptr=self.pin.ptr, nbytes=runs_end))
            rs, msgs, resp = rs.copy(), msgs.copy(), resp.copy()
        return rs, msgs, resp, self.cli.pack_requests(self.pin.array[:n], reqs, out_cap=self.req_out_cap)

    def server(self, to_srv):
        """the server half: one k_ring ticket over what the client wrote; its replies go back to the client"""
        import brpc_b200 as b2
        live = [k for k, b in enumerate(to_srv) if b]
        data, runs = b2.make_runs([to_srv[k] for k in live])
        rs, msgs, resp, _ = self.srv.ring_wait(self.srv.ring_submit(data, runs))
        assert (rs["consumed"] == runs["length"]).all() and (msgs["status"] == 0).all()
        for r, k in enumerate(live):
            ms = msgs[int(rs[r]["first_msg"]):int(rs[r]["first_msg"]) + int(rs[r]["n_msgs"])]
            self.to_cli[k] = b"".join(resp[int(m["resp_off"]):int(m["resp_off"]) + int(m["resp_len"])].tobytes() for m in ms)

    def close(self):
        self.cli.close(); self.srv.close(); self.pin.free()


def run_shape(n_socks, per_sock, size, compress, steps, warmup):
    from _compare import assert_same
    from brpc_b200.abi import ECHO_METHOD
    rng = random.Random(n_socks * 1000 + per_sock * 10 + size + compress)
    block = bytes(rng.choice(b"abcdefghij") for _ in range(64 if compress else size))
    payloads = [(block * (size // len(block) + 1))[:size] for _ in range(n_socks * per_sock)]
    socks = [k for k in range(n_socks) for _ in range(per_sock)]
    methods = (dict(ECHO_METHOD, response_compress_type=compress, response_checksum_type=compress),)
    arms = {"ring": Loop(True, socks, methods), "batch": Loop(False, socks, methods)}
    lat = {a: {"client": [], "round": []} for a in arms}
    phases = []; launches = 0; n_replies = 0
    sent = set()
    for step in range(warmup + steps):
        A, B = arms["ring"], arms["batch"]
        assert A.to_cli == B.to_cli, step
        data, runs, reqs, runs_end = turn_input(A.to_cli, payloads, socks, compress, step + 1)
        got = {}
        for name, L in arms.items():
            l0 = L.cli.ring_launches()
            t0 = time.perf_counter()
            got[name] = L.client(data, runs, reqs, runs_end)
            t1 = time.perf_counter()
            to_srv = [b""] * (n_socks)
            for k, f in zip(socks, got[name][3]):
                to_srv[k] += f
            t2 = time.perf_counter()
            L.server(to_srv)
            t3 = time.perf_counter()
            if step >= warmup:
                lat[name]["client"].append((t1 - t0) * 1e6); lat[name]["round"].append((t1 - t0 + t3 - t2) * 1e6)
                if L.ring:
                    launches += L.cli.ring_launches() - l0; phases.append(L.cli.ring_phase_ns(L.last))
        (ra, ma, pa, fa), (rb, mb, pb, fb) = got["ring"], got["batch"]
        assert fa == fb and all(len(f) > 0 for f in fa), step
        if len(runs):
            assert_same((ra, ma, pa), (rb, mb, pb), "step %d" % step)
            # B2_MSG_RESPONSE, or B2_MSG_RESPONSE_UNZ for a compressed reply (its message inflated into the resp region)
            assert np.isin(ma["status"], (7, 8)).all() and (ma["error_code"] == 0).all() and (ra["consumed"] == runs["length"]).all(), step
            assert set(int(c) for c in ma["correlation_id"]) == sent, step
            n_replies += len(ma)
        sent = set(int(c) for c in reqs["correlation_id"])
    pct = lambda v, q: round(float(np.percentile(np.asarray(v), q)), 1)
    ph = np.median(np.asarray(phases, dtype=np.float64), axis=0) / 1e3
    out = {"sockets": n_socks, "requests_per_socket": per_sock, "message_bytes": size, "snappy_crc32c": bool(compress),
           "ticket_bytes": int(len(data))}
    for name in arms:
        out[name] = {"client_p50_us": pct(lat[name]["client"], 50), "client_p99_us": pct(lat[name]["client"], 99),
                     "round_p50_us": pct(lat[name]["round"], 50), "round_p99_us": pct(lat[name]["round"], 99)}
    out["ring"]["launches_per_1000_tickets"] = 1000.0 * launches / steps
    out["ring"]["phase_us_median"] = {"header_read": round(ph[0], 1), "bytes_pulled": round(ph[1], 1), "runs_served_and_requests_packed": round(ph[2], 1),
                                      "results_pushed": round(ph[3], 1)}
    out.update({"replies_checked": n_replies, "results_equal": True})
    for L in arms.values():
        L.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    a = ap.parse_args()
    gpu = gpu_facts()
    shapes = [(64, 1, 1024, 0), (1, 64, 1024, 0), (64, 1, 4096, 1)]
    res = [run_shape(s, k, n, c, a.steps, a.warmup) for s, k, n, c in shapes]
    print(json.dumps({"bench": "baidu_std client turns on the ring vs b2_ring_submit + b2_pack_requests", "steps": a.steps, "gpu": gpu, "shapes": res}))


if __name__ == "__main__":
    main()
