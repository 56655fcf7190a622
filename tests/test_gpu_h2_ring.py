"""GPU: h2/gRPC on the latency path (b2_h2_ring_*: k_h2_ring on the submit ring) against a twin context that runs b2_h2_serve_batch on the
same batches with the same caps — run statuses, messages, the defined bytes of out, spans and replies, ticket by ticket, so that the
connection state each ticket leaves (HPACK tables, windows, deferred WINDOW_UPDATEs, the stream pool) is shown equal by the next one:
  - the mixed mutated calls of test_gpu_h2_serve.py cut across batches, one ticket at a time and eight in flight (waited out of order);
  - a call whose frames span two tickets; gunzip connections, and the recorded gzip client capture against the oracle engine;
  - state calls between tickets: conn_reset, set_gunzip, peer_update, and b2_h2_pack_responses answering the left calls zero-copy
    from the last ticket (which moves the HPACK encoder table);
  - every refused call while a ticket is outstanding; the capacity refusals; a full reply region that leaves calls to the host;
  - idle retirement and relaunch, no launch over 100 steady tickets, the rules that keep k_ring and k_h2_ring apart;
  - a live grpcio client: 1 000 calls over 8 connections through a ring variant of DeviceServeEngine."""
import os
import random
import time

import numpy as np
import pytest

import _h2serve as S
import _h2traffic as T
import _oracle as O
from _h2gzip import server_blob_used
from test_gpu_h2_serve import IDENTITY, METHODS, REGION, RREGION, WINDOW, _ctx, call, conn_stream, gz, mixed_calls, prefix

pytestmark = pytest.mark.gpu
MAX_BYTES = 1 << 20
F_BODY_IN_INPUT, F_GUNZIPPED = 16, 64


def _err(fn, *a, **kw):
    from brpc_b200.abi import B2Error
    with pytest.raises(B2Error) as e:
        fn(*a, **kw)
    return e.value.code


def _snap(res):
    return tuple(np.array(x, copy=True) for x in res)


def _same(got, want, n, region, what=""):
    """ring results == the batch call's: statuses, messages, the defined bytes of out, spans and replies"""
    rs, msgs, out, replies, spans = got
    rs0, msgs0, out0, replies0, spans0 = want
    assert rs.tobytes() == rs0.tobytes(), what
    assert msgs.tobytes() == msgs0.tobytes(), what
    assert spans.tobytes() == spans0.tobytes(), what
    for r in range(n):
        co, cl = int(rs0[r]["ctrl_off"]), int(rs0[r]["ctrl_len"])
        assert bytes(out[co:co + cl]) == bytes(out0[co:co + cl]), (what, r)
        f, c = int(rs0[r]["first_msg"]), int(rs0[r]["n_msgs"])
        b0 = r * region + region // 4
        used = server_blob_used(msgs0[f:f + c], r, region)
        assert bytes(out[b0:b0 + used]) == bytes(out0[b0:b0 + used]), (what, r)
        for m in msgs0[f:f + c]:
            if int(m["flags"]) & F_GUNZIPPED:
                o, ln = int(m["msg_off"]), int(m["msg_len"])
                assert bytes(out[o:o + ln]) == bytes(out0[o:o + ln]), (what, r)
        so, sl = int(spans0[r]["off"]), int(spans0[r]["len"])
        assert bytes(replies[so:so + sl]) == bytes(replies0[so:so + sl]), (what, r)


class Pair:
    """a ring context (b2_h2_ring_enable) and a twin that serves the same batches with b2_h2_serve_batch and the same caps"""
    def __init__(self, n, gunzip=(), methods=METHODS, identity=IDENTITY, msg_cap=None, out_cap=None, replies_cap=None):
        self.n = n
        self.msg_cap, self.out_cap, self.replies_cap = msg_cap or n * 128, out_cap or n * REGION, replies_cap or n * RREGION
        self.ring, self.twin = _ctx(methods, identity), _ctx(methods, identity)
        for k in range(n):
            for c in (self.ring, self.twin):
                c.h2_conn_reset(k)
                if k in gunzip:
                    c.h2_conn_set_gunzip(k)
        self.ring.h2_ring_enable(MAX_BYTES, self.msg_cap, self.out_cap, self.replies_cap)

    def region(self, n_runs):
        return (self.out_cap // n_runs) & ~63

    def twin_batch(self, chunks, ids=None):
        import brpc_b200
        data, runs = brpc_b200.make_runs(chunks)
        runs["socket_id"] = np.arange(len(chunks)) if ids is None else ids
        want = _snap(self.twin.h2_serve_batch(data, runs, msg_cap=self.msg_cap, out_cap=self.out_cap, replies_cap=self.replies_cap))
        return data, runs, want

    def step(self, chunks, ids=None, what=""):
        """one ticket, waited at once; returns the ring's results (views of the slot)"""
        data, runs, want = self.twin_batch(chunks, ids)
        self.last = self.ring.h2_ring_submit(data, runs)
        got = self.ring.h2_ring_wait(self.last)
        _same(got, want, len(chunks), self.region(len(chunks)), what)
        return got

    def many(self, batches, depth):
        """batches: [(data, runs, want)] the twin served in order; submitted `depth` at a time, each group waited last to first"""
        for i in range(0, len(batches), depth):
            group = batches[i:i + depth]
            tickets = [self.ring.h2_ring_submit(d, r) for d, r, _ in group]
            for (d, r, want), t in reversed(list(zip(group, tickets))):
                _same(self.ring.h2_ring_wait(t), want, len(r), self.region(len(r)), "ticket %d" % t)


def _cut(pair, streams, parts):
    """the streams cut into `parts` batches as the twin consumes them: [(data, runs, want)]"""
    n = len(streams); rest = [b""] * n; out = []
    for part in range(parts):
        now = [rest[k] + streams[k][len(streams[k]) * part // parts:len(streams[k]) * (part + 1) // parts] for k in range(n)]
        data, runs, want = pair.twin_batch(now)
        out.append((data, runs, want))
        rest = [now[k][int(want[0][k]["consumed"]):] for k in range(n)]
    assert not any(rest)
    return out


@pytest.mark.parametrize("depth", [1, 8])
def test_mixed_calls_across_tickets_equal_the_batch_call(depth):
    rng = random.Random(20261017 + depth)
    n = 8
    pair = Pair(n, gunzip=set(range(0, n, 2)))
    streams = [conn_stream(rng, k, mixed_calls(rng, k)) for k in range(n)]
    batches = _cut(pair, streams, 8)
    pair.many(batches, depth)
    answered = sum(int(w[4]["n_answered"].sum()) for _, _, w in batches)
    assert answered > 30 * n


def test_a_call_whose_frames_span_two_tickets():
    pair = Pair(2)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(2)]
    body = prefix(S.echo_request(bytes(range(97, 123)) * 1500))
    whole = [T.PREFACE + T.settings() + WINDOW + call(enc[k], 1, body, chunk=9000) for k in range(2)]
    cut = [len(whole[0]) // 2, len(whole[1]) // 3]
    got = pair.step([whole[k][:cut[k]] for k in range(2)], what="first half")
    assert int(got[4]["n_answered"].sum()) == 0
    cons = [int(got[0][k]["consumed"]) for k in range(2)]
    got = pair.step([whole[k][cons[k]:] for k in range(2)], what="second half")
    assert int(got[4]["n_answered"].sum()) == 2


def test_gunzip_connections():
    rng = random.Random(3)
    n = 4
    pair = Pair(n, gunzip=set(range(n)))
    msgs = [S.echo_request(bytes(rng.randrange(97, 100) for _ in range(2000 + 500 * i))) for i in range(6)]
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    ge = ((b"grpc-encoding", b"gzip"),)
    streams = [T.PREFACE + T.settings() + WINDOW + b"".join(call(enc[k], 1 + 2 * i, prefix(gz(m), 1), extra=ge) for i, m in enumerate(msgs))
               for k in range(n)]
    batches = _cut(pair, streams, 3)
    pair.many(batches, 3)
    assert sum(int(np.count_nonzero(w[1]["flags"] & F_GUNZIPPED)) for _, _, w in batches) == n * len(msgs)


class RingServeEngine(S.DeviceServeEngine):
    """DeviceServeEngine on the ring: one b2_h2_ring_submit + wait per feed, then b2_h2_pack_responses for the calls it left"""
    def __init__(self, ctx, gunzip=False):
        super().__init__(ctx, gunzip)
        ctx.h2_ring_enable(1 << 20, 1024, 8 << 20, 8 << 20)

    def feed(self, cid, buf):
        import brpc_b200
        from brpc_b200.abi import H2_RESPONSE_DT
        with self.lock:
            data, runs = brpc_b200.make_runs([buf]); runs["socket_id"] = cid
            rs, msgs, out, replies, spans = self.ctx.h2_ring_wait(self.ctx.h2_ring_submit(data, runs))
            co, cl, so, sl = int(rs["ctrl_off"][0]), int(rs["ctrl_len"][0]), int(spans["off"][0]), int(spans["len"][0])
            reply = bytes(out[co:co + cl]) + bytes(replies[so:so + sl])
            left = msgs[(msgs["flags"] & S.F_ANSWERED) == 0]
            self.n_answered += int(spans["n_answered"][0])
            if len(left):
                r = np.zeros(len(left), H2_RESPONSE_DT)
                r["conn"] = cid; r["stream_id"] = left["stream_id"]; r["status_code"] = 200; r["flags"] = 1
                r["content_type_len"] = 16; r["grpc_status"] = 12; r["grpc_message_off"] = 16; r["grpc_message_len"] = 13
                reply += b"".join(self.ctx.h2_pack_responses(np.frombuffer(b"application/grpcunimplemented\0", np.uint8), r))
            return int(rs["consumed"][0]), reply, int(rs["parse_error"][0]), len(msgs)


def test_recorded_gzip_client_capture_equals_the_oracle_engine():
    import gzip
    import json
    with gzip.open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "h2_gzip_capture.json.gz"), "rt") as f:
        cap = json.load(f)["server_rx"]
    ed = RingServeEngine(_ctx((O.ECHO_METHOD,), b"", 16, 192, 4096 + (256 << 10)), gunzip=True); eo = S.OracleServeEngine(gunzip=True)
    n = 0
    for cid, chunks in cap["chunks"].items():
        cid = int(cid); ed.open(cid); eo.open(cid)
        pd = po = b""
        for i, ch in enumerate(chunks):
            ch = bytes.fromhex(ch); pd += ch; po += ch
            cd, od, errd, nd = ed.feed(cid, pd)
            co, oo, erro, no = eo.feed(cid, po)
            assert (cd, errd, nd) == (co, erro, no) and od == oo, (cid, i)
            pd = pd[cd:]; po = po[co:]; n += nd
    assert n == len(cap["bodies"]) and ed.n_answered == eo.n_answered and eo.n_inflated > 30


def _zero_copy_records(msgs, out_head, sids_conn):
    """b2_h2_response records that echo each left call's raw message from where the last batch left it (B2_H2_RESP_BODY_IN_INPUT /
    _BODY_IN_OUT) with the request's content-type from the out region (B2_H2_RESP_CT_IN_OUT)"""
    from brpc_b200.abi import H2_RESPONSE_DT
    r = np.zeros(len(msgs), H2_RESPONSE_DT)
    r["conn"] = sids_conn; r["stream_id"] = msgs["stream_id"]; r["status_code"] = 200
    r["flags"] = 1 | 8 | np.where(msgs["flags"] & F_BODY_IN_INPUT, 2, 4)
    for i, m in enumerate(msgs):
        h = bytes(out_head[int(m["headers_off"]):int(m["headers_off"]) + int(m["headers_len"])])
        p = 0
        while p < len(h):
            nl, vl = h[p] | (h[p + 1] << 8), h[p + 2] | (h[p + 3] << 8)
            if h[p + 4:p + 4 + nl] == b"content-type":
                r[i]["content_type_off"] = int(m["headers_off"]) + p + 4 + nl; r[i]["content_type_len"] = vl
            p += 4 + nl + vl
    r["body_off"] = msgs["msg_off"]; r["body_len"] = msgs["msg_len"]
    return r


def test_state_calls_between_tickets():
    rng = random.Random(9)
    n = 4
    pair = Pair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    msg = S.echo_request(b"state " * 300)
    sid = [1] * n

    def calls(k, m, path=b"/example.EchoService/Echo"):
        out = b""
        for _ in range(m):
            out += call(enc[k], sid[k], prefix(msg), path=path); sid[k] += 2
        return out

    pair.step([T.PREFACE + T.settings() + WINDOW + calls(k, 3) for k in range(n)], what="open")
    # host-method calls left by the device, answered zero-copy from the last ticket on both
    got = pair.step([calls(k, 2, b"/example.EchoService/Host") + calls(k, 1) for k in range(n)], what="host calls")
    rs, msgs, out = got[0], got[1], got[2]
    left = msgs[(msgs["flags"] & S.F_ANSWERED) == 0]
    assert len(left) == 2 * n
    conn = np.repeat(np.arange(n), rs["n_msgs"])[(msgs["flags"] & S.F_ANSWERED) == 0]
    recs = _zero_copy_records(left, out, conn)
    assert pair.ring.h2_pack_responses(None, recs) == pair.twin.h2_pack_responses(None, recs)
    pair.step([calls(k, 2) for k in range(n)], what="after the host replies")
    for c in (pair.ring, pair.twin):
        c.h2_conn_peer_update(1, header_table_size=0, stream_window_size=1 << 20, conn_window_add=1 << 20)
        c.h2_conn_set_gunzip(2)
        c.h2_conn_reset(3)
    enc[3] = T.HpackEncoder(random.Random(33)); sid[3] = 1
    pair.step([calls(k, 2) if k != 3 else T.PREFACE + T.settings() + WINDOW + calls(3, 2) for k in range(n)], what="after the state calls")
    pair.step([calls(k, 3) for k in range(n)], what="one more")


def test_calls_refused_while_a_ticket_is_outstanding():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL, H2_RESPONSE_DT, H2_REQUEST_DT, REPLY_DT, REQUEST_DT
    n = 2
    pair = Pair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    msg = S.echo_request(b"x" * 100)
    pair.step([T.PREFACE + T.settings() + WINDOW + call(enc[k], 1, prefix(msg)) for k in range(n)], what="open")
    data, runs, want = pair.twin_batch([call(enc[k], 3, prefix(msg)) for k in range(n)])
    ring = pair.ring
    t = ring.h2_ring_submit(data, runs)
    small = np.zeros(64, np.uint8)
    one_run = brpc_b200.make_runs([b"\0" * 16])
    refused = [
        lambda: ring.h2_conn_reset(0), lambda: ring.h2_conn_set_gunzip(0), lambda: ring.h2_conn_peer_update(0, stream_window_size=1000),
        lambda: ring.h2_conn_set_next_stream_id(0, 5), lambda: ring.h2_client_conn_reset(1), lambda: ring.h2_client_abandon_streams(0, [1]),
        lambda: ring.h2_process_batch(*one_run), lambda: ring.h2_serve_batch(*one_run), lambda: ring.h2_client_process_batch(*one_run),
        lambda: ring.h2_scan_batch(*one_run), lambda: ring.h2_pack_responses(small, np.zeros(1, H2_RESPONSE_DT)),
        lambda: ring.h2_pack_requests(small, np.zeros(1, H2_REQUEST_DT)), lambda: ring.hpack_reset(0),
        lambda: ring.hpack_decode_batch(small, [(0, 0, 16)]), lambda: ring.process_batch(*one_run),
        lambda: ring.crc32c_batch(small, [0], [16]), lambda: ring.snappy_compress_batch(small, [0], [16], 1024),
        lambda: ring.snappy_uncompress_batch(small, [0], [16], 1024), lambda: ring.pack_requests(small, np.zeros(1, REQUEST_DT)),
        lambda: ring.pack_responses(small, np.zeros(1, REPLY_DT)),
    ]
    for i, f in enumerate(refused):
        assert _err(f) == B2_E_INVAL, i
    _same(ring.h2_ring_wait(t), want, n, pair.region(n), "the outstanding ticket")
    pair.step([call(enc[k], 5, prefix(msg)) for k in range(n)], what="after the refusals")
    ring.crc32c_batch(small, [0], [16])                            # between tickets every call works
    pair.step([call(enc[k], 7, prefix(msg)) for k in range(n)], what="after a call between tickets")


def test_capacity_refusals_and_a_full_reply_region():
    import brpc_b200
    from brpc_b200.abi import B2_E_CAPACITY, B2_E_INVAL
    c = _ctx()
    assert _err(c.h2_ring_enable, (32 << 20) + 1, 64, 1 << 20, 1 << 20) == B2_E_CAPACITY      # max_batch_bytes
    assert _err(c.h2_ring_enable, 1 << 20, (1 << 15) + 1, 1 << 20, 1 << 20) == B2_E_CAPACITY  # max_msgs
    assert _err(c.h2_ring_enable, 1 << 20, 64, (128 << 20) + 1, 1 << 20) == B2_E_CAPACITY     # 2 * max_resp_bytes
    assert _err(c.h2_ring_enable, 1 << 20, 64, 1 << 20, (64 << 20) + 1) == B2_E_CAPACITY      # max_resp_bytes
    c.h2_ring_enable(4096, 4, 1000, 1 << 16)
    data, runs = brpc_b200.make_runs([b"\0" * 32] * 5)
    runs["socket_id"] = np.arange(5)
    assert _err(c.h2_ring_submit, np.zeros(4097, np.uint8), runs[:1]) == B2_E_CAPACITY       # nbytes > max_bytes
    assert _err(c.h2_ring_submit, data, runs) == B2_E_CAPACITY                               # msg_cap / n_runs == 0
    assert _err(c.h2_ring_submit, data, runs[:4]) == B2_E_CAPACITY                           # (out_cap / 4) & ~63 = 192 < 256
    bad = runs[:2].copy(); bad["socket_id"] = 0
    assert _err(c.h2_ring_submit, data, bad) == B2_E_INVAL                                   # one run per connection
    bad = runs[:1].copy(); bad["socket_id"] = 32
    assert _err(c.h2_ring_submit, data, bad) == B2_E_INVAL                                   # connection out of range
    bad = runs[:1].copy(); bad["length"] = len(data) + 1
    assert _err(c.h2_ring_submit, data, bad) == B2_E_INVAL                                   # run outside the buffer
    # a full reply region: the run's later calls are the host's, exactly as with the batch call
    rng = random.Random(5)
    n = 4
    pair = Pair(n, replies_cap=n * 4 * 4096)
    msgs = [S.echo_request(bytes(rng.randrange(97, 123) for _ in range(3000))) for _ in range(12)]
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    got = pair.step([T.PREFACE + T.settings() + WINDOW + b"".join(call(enc[k], 1 + 2 * i, prefix(m)) for i, m in enumerate(msgs)) for k in range(n)],
                    what="full reply region")
    left = got[1][(got[1]["flags"] & S.F_ANSWERED) == 0]
    assert 0 < len(left) < n * 12
    conn = np.repeat(np.arange(n), got[0]["n_msgs"])[(got[1]["flags"] & S.F_ANSWERED) == 0]
    recs = _zero_copy_records(left, got[2], conn)
    assert pair.ring.h2_pack_responses(None, recs) == pair.twin.h2_pack_responses(None, recs)
    pair.step([b"".join(call(enc[k], 25 + 2 * i, prefix(m)) for i, m in enumerate(msgs[:2])) for k in range(n)], what="after the host")


def _steady(pair, enc, sid, steps, msg):
    for _ in range(steps):
        pair.step([call(enc[k], sid[k], prefix(msg)) for k in range(pair.n)])
        for k in range(pair.n):
            sid[k] += 2


def test_idle_retirement_relaunch_and_no_launch_over_100_steady_tickets(monkeypatch):
    monkeypatch.setenv("B2_RING_IDLE_MS", "2000")
    n = 4
    pair = Pair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    msg = S.echo_request(b"steady" * 100)
    pair.step([T.PREFACE + T.settings() + WINDOW for _ in range(n)])
    sid = [1] * n
    n0 = pair.ring.ring_launches()
    _steady(pair, enc, sid, 100, msg)
    assert pair.ring.ring_launches() == n0
    pair.ring.ring_stop()
    monkeypatch.setenv("B2_RING_IDLE_MS", "5")
    _steady(pair, enc, sid, 1, msg)                                 # relaunched by the submission, now with a 5 ms idle time
    n1 = pair.ring.ring_launches()
    assert n1 == n0 + 1
    time.sleep(0.2)                                                  # it retires and comes back with the next submission
    _steady(pair, enc, sid, 2, msg)
    assert pair.ring.ring_launches() > n1
    ph = pair.ring.ring_phase_ns(pair.last)
    assert 0 < ph[0] <= ph[1] <= ph[2] <= ph[3]


def test_one_resident_kernel_per_context():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL
    a = _ctx(); a.ring_start()
    assert _err(a.h2_ring_enable, 1 << 20, 64, 1 << 20, 1 << 20) == B2_E_INVAL
    a.ring_stop()
    b = _ctx()
    b.h2_ring_enable(1 << 20, 64, 1 << 20, 1 << 20)
    data, runs = brpc_b200.make_runs([b"\0" * 16])
    assert _err(b.ring_submit, data, runs) == B2_E_INVAL
    assert _err(b.h2_ring_enable, 1 << 20, 64, 1 << 20, 1 << 20) == B2_E_INVAL
    assert _err(b.h2_ring_wait, 1) == B2_E_INVAL                                             # no such ticket
    c = _ctx(); c.stream_configure(64, 1 << 16); c.stream_ring_enable(1 << 16)
    assert _err(c.h2_ring_enable, 1 << 20, 64, 1 << 20, 1 << 20) == B2_E_INVAL
    d = _ctx(); d.h2_ring_enable(1 << 20, 64, 1 << 20, 1 << 20); d.stream_configure(64, 1 << 16)
    assert _err(d.stream_ring_enable, 1 << 16) == B2_E_INVAL
    for x in (a, b, c, d):
        x.close()


def test_live_grpcio_client_1000_calls_over_8_connections():
    pytest.importorskip("grpc")
    from _h2loop import H2LoopServer
    eng = RingServeEngine(_ctx((O.ECHO_METHOD,), IDENTITY, 16, 128))
    srv = H2LoopServer(eng)
    reqs = S.mutation_corpus(1000, seed=8)
    try:
        got = S.grpcio_calls(srv.port, reqs, channels=8)
    finally:
        srv.close()
    assert not srv.errors, srv.errors
    assert got == [S.expected_call(r, IDENTITY) for r in reqs]
    assert eng.n_answered == 1000 and sum(1 for g in got if g[0] != "OK") > 200
