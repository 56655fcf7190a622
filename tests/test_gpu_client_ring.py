"""GPU: baidu_std client connections on the latency path (b2_client_ring_*).  A ticket is one client turn: the replies read from client
sockets (B2_RUN_CLIENT runs) are served as b2_process_batch serves them, then the queued requests are packed as b2_pack_requests packs
them, inside the resident k_ring<true>.  Every ticket is compared with a twin context running those two batch calls, and with the
oracle's process_batch, pack_echo_request and pack_stream_frame."""
import gc
import random
import time

import numpy as np
import pytest

import _oracle as O
from _compare import assert_same

pytestmark = pytest.mark.gpu
SEED = 20261018
MAX_BYTES, MAX_REQS, REQ_OUT = 1 << 20, 256, 2 << 20
CFG = O.make_config()


def _ctx():
    import brpc_b200
    return brpc_b200.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=512, max_resp_bytes=8 << 20)


def _err(fn, *a, **kw):
    from brpc_b200.abi import B2Error
    try:
        fn(*a, **kw)
    except B2Error as e:
        return e.code
    return 0


def _rnd(rng, n):
    return bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz0123456789") for _ in range(n))


class Req:
    """one queued request: its b2_request fields (payload and attachment placed later) and the oracle's frame"""

    def __init__(self, rng, cid, stream=None, method_idx=0, compress=None, size=None):
        self.payload = _rnd(rng, size if size is not None else rng.choice([0, 1, 15, 100, 600, 1024, 3000]))
        self.cid = cid
        if stream is None:
            stream = rng.random() < 0.2
        if stream:
            self.kind = 1
            self.has_src, self.cont, self.ft, self.src = rng.random() < 0.8, rng.choice([None, False, True]), rng.choice([1, 2, 3, 4]), rng.randrange(1 << 40)
            self.flags = (1 if self.has_src else 0) | (0 if self.cont is None else 2 | (4 if self.cont else 0))
            self.att = b""
        else:
            self.kind = 0
            self.has_log, self.log_id, self.to = rng.random() < 0.6, rng.choice([0, 5, 12345, 1 << 40]), rng.choice([0, 0, 100, 60000])
            self.comp = rng.choice([0, 0, 1]) if compress is None else compress
            self.cks = rng.choice([0, 1])
            self.att = _rnd(rng, rng.choice([0, 0, 0, 7, 300]))
            self.flags = (1 if self.has_log else 0) | (2 if self.to > 0 else 0)
        self.method_idx = method_idx

    def record(self, p_off, a_off):
        if self.kind == 1:
            return (1, self.flags, -1, 0, self.cid, self.src, 0, 0, self.ft, p_off, len(self.payload), 0, 0, 0)
        return (0, self.flags, self.method_idx, self.to, self.cid, self.log_id, self.comp, self.cks, 0, p_off, len(self.payload), a_off, len(self.att), 0)

    def frame(self):
        if self.kind == 1:
            return O.pack_stream_frame(self.cid, self.src if self.has_src else -1, self.ft, self.cont, self.payload)
        if self.method_idx != 0 or self.comp not in (0, 1):
            return b""
        return O.pack_echo_request(log_id=self.log_id if self.has_log else None, correlation_id=self.cid, message=self.payload,
                                   attachment=self.att, compress_type=self.comp, checksum_type=self.cks, timeout_ms=self.to)


def ticket(chunks, reqs, client=True, pad=0):
    """the bytes of one turn: the runs (chunks, 16-aligned), then every request's payload and attachment"""
    from brpc_b200.abi import REQUEST_DT, RUN_DT
    blob = bytearray(b"\0" * pad)
    runs = []
    for k, c in chunks:
        off = len(blob); blob += c; blob += b"\0" * (-len(blob) % 16)
        runs.append((k, off, len(c), -1, 1 if client else 0))
    recs = []
    for q in reqs:
        p = len(blob); blob += q.payload; a = len(blob); blob += q.att
        recs.append(q.record(p, a))
    blob += b"\0" * 16
    return np.frombuffer(bytes(blob), np.uint8), np.array(runs, RUN_DT), np.array(recs, REQUEST_DT)


def _copy(res):
    rs, msgs, resp = res[:3]
    return rs.copy(), msgs.copy(), resp.copy()


class Pair:
    """a context serving client turns on the ring, and its twin running the two batch calls"""

    def __init__(self, max_bytes=MAX_BYTES, max_reqs=MAX_REQS, req_out=REQ_OUT):
        self.ring, self.twin = _ctx(), _ctx()
        self.ring.client_ring_enable(max_bytes, max_reqs, req_out)
        self.req_out = req_out
        self.last = 0

    def twin_turn(self, data, runs, recs):
        batch = _copy(self.twin.process_batch(data, runs)) if len(runs) else None
        frames = self.twin.pack_requests(data, recs, out_cap=self.req_out) if len(recs) else []
        return batch, frames

    def check(self, got, data, runs, reqs, want, what=""):
        batch, frames = want
        if batch is None:
            assert len(got[0]) == 0 and len(got[1]) == 0, what
        else:
            assert_same(got, batch, "%s: ring vs twin" % (what,))
            assert_same(got, O.process_batch(CFG, data, runs), "%s: ring vs oracle" % (what,))
        assert len(got[4]) == len(reqs) == len(frames), what
        for i, (g, f, q) in enumerate(zip(got[4], frames, reqs)):
            assert g == f, (what, i, "ring vs twin")
            assert g == q.frame(), (what, i, "ring vs oracle")

    def turn(self, data, runs, recs, reqs, what="", **kw):
        want = self.twin_turn(data, runs, recs)
        t = self.ring.client_ring_submit(data, runs, recs, **kw)
        assert t == self.last + 1, (t, self.last)
        self.last = t
        got = self.ring.client_ring_wait(t)
        self.check(got, data, runs, reqs, want, what)
        return got

    def step(self, chunks, reqs, client=True, what=""):
        return self.turn(*ticket(chunks, reqs, client), reqs, what)

    def close(self):
        self.ring.close(); self.twin.close()


def _server_replies(rng, n_socks, per_sock, cid0=1):
    """what an echo server answers: per socket the replies to per_sock requests of every shape"""
    import brpc_b200
    srv = _ctx()
    streams = []
    for k in range(n_socks):
        frames = []
        for j in range(per_sock):
            q = Req(rng, cid0 + k * 1000 + j, stream=False)
            frames.append(q.frame())
        streams.append(b"".join(frames))
    data, runs = brpc_b200.make_runs(streams)
    rs, msgs, resp, _ = srv.process_batch(data, runs)
    out = []
    for k in range(n_socks):
        ms = msgs[rs[k]["first_msg"]:rs[k]["first_msg"] + rs[k]["n_msgs"]]
        assert (ms["status"] == 0).all()
        out.append(b"".join(bytes(resp[m["resp_off"]:m["resp_off"] + m["resp_len"]]) for m in ms))
    srv.close()
    return out


@pytest.mark.parametrize("depth", [1, 8])
def test_seeded_conversation_across_tickets(depth):
    """an echo server's replies split at random offsets across tickets (each ticket carries the unconsumed tail, as `consumed` says), with
    mixed requests in every ticket; up to `depth` tickets in flight, waited in and out of order"""
    rng = random.Random(SEED + depth)
    n_socks = 16
    replies = _server_replies(rng, n_socks, 6)
    pair = Pair()
    pos, tail = [0] * n_socks, [b""] * n_socks
    turns = []
    cid = 1 << 33
    while any(pos[k] < len(replies[k]) for k in range(n_socks)) or len(turns) < 6:
        chunks = []
        for k in range(n_socks):
            if rng.random() < 0.3 and pos[k] < len(replies[k]):
                continue
            take = rng.choice([0, 5, 12, 100, 700, 2000, 6000])
            new = replies[k][pos[k]:pos[k] + take]; pos[k] += len(new)
            if tail[k] or new:
                chunks.append((k, tail[k] + new))
        reqs = [Req(rng, cid + i) for i in range(rng.choice([0, 1, 5, 30]))]
        cid += 64
        if not chunks and not reqs:
            reqs = [Req(rng, cid)]
        data, runs, recs = ticket(chunks, reqs)
        want = pair.twin_turn(data, runs, recs)
        if want[0] is not None:
            for r, (k, c) in enumerate(chunks):
                tail[k] = c[int(want[0][0]["consumed"][r]):]
        turns.append((data, runs, recs, reqs, want))
    for g0 in range(0, len(turns), depth):
        group = turns[g0:g0 + depth]
        ts = [pair.ring.client_ring_submit(d, r, q) for d, r, q, _, _ in group]
        assert ts == list(range(pair.last + 1, pair.last + 1 + len(group)))
        pair.last = ts[-1]
        order = list(range(len(group)))
        rng.shuffle(order)
        for i in order:
            d, r, q, reqs, want = group[i]
            pair.check(pair.ring.client_ring_wait(ts[i]), d, r, reqs, want, ("turn", g0 + i))
    pair.close()


def test_ticket_shapes():
    from brpc_b200.abi import PinnedBuffer
    rng = random.Random(SEED + 2)
    pair = Pair()
    replies = _server_replies(rng, 4, 3)
    pair.step([(k, replies[k]) for k in range(4)], [], what="runs only")
    pair.step([], [Req(rng, 10 + i) for i in range(20)], what="requests only")
    pair.step([(0, replies[0][:777]), (1, replies[1])], [Req(rng, 40 + i) for i in range(9)], what="both")
    # server runs in a client ticket (a peer sent requests): answered as b2_ring_submit answers them
    server = b"".join(Req(rng, 90 + i, stream=False).frame() for i in range(5))
    q = [Req(rng, 60), Req(rng, 61)]
    data, runs, recs = ticket([(0, replies[2]), (1, server)], q)
    runs["flags"][1] = 0
    got = pair.turn(data, runs, recs, q, "server runs in a client ticket")
    assert (got[1]["status"][-5:] == 0).all()
    # requests that cannot be packed: a method index out of range, gzip: out_len 0 as in the batch call
    bad = [Req(rng, 70, stream=False, method_idx=3), Req(rng, 71, stream=False, method_idx=-1), Req(rng, 72, stream=False, compress=2), Req(rng, 73, stream=False)]
    got = pair.step([(3, replies[3])], bad, what="unpackable")
    assert [len(f) > 0 for f in got[4]] == [False, False, False, True]
    # bytes in b2_block_alloc memory are pulled in place, other bytes staged: the same results
    reqs = [Req(rng, 80 + i) for i in range(12)]
    data, runs, recs = ticket([(k, replies[k]) for k in range(4)], reqs)
    buf = PinnedBuffer(len(data) + 4096)
    buf.array[:len(data)] = data
    pair.turn(data, runs, recs, reqs, "pinned bytes", ptr=buf.ptr, nbytes=len(data))
    pair.step([(k, replies[k]) for k in range(4)], reqs, what="staged again")
    pair.close()
    buf.free()


def test_overflow_served_by_the_big_pipeline():
    """runs with more messages than the compact block holds are served through the big pipeline inside the wait; the requests of the
    same ticket still come from the kernel, and a ticket behind it in the ring is served by the kernel"""
    rng = random.Random(SEED + 3)
    pair = Pair()
    tiny = b"".join(Req(rng, 500 + i, stream=False, size=0).frame() for i in range(1100))      # 1100 > 1024 messages
    srv = _ctx()
    import brpc_b200
    d0, r0 = brpc_b200.make_runs([tiny])
    rs, msgs, resp, _ = srv.process_batch(d0, r0)
    replies = b"".join(bytes(resp[m["resp_off"]:m["resp_off"] + m["resp_len"]]) for m in msgs)
    srv.close()
    for what, client, body in (("client", True, replies), ("server", False, tiny)):
        reqs = [Req(rng, 900 + i) for i in range(17)]
        data, runs, recs = ticket([(0, body)], reqs, client=client)
        want = pair.twin_turn(data, runs, recs)
        reqs2 = [Req(rng, 950 + i) for i in range(3)]
        data2, runs2, recs2 = ticket([(1, body[:300])], reqs2, client=client)
        want2 = pair.twin_turn(data2, runs2, recs2)
        t = pair.ring.client_ring_submit(data, runs, recs)
        t2 = pair.ring.client_ring_submit(data2, runs2, recs2)
        pair.check(pair.ring.client_ring_wait(t2), data2, runs2, reqs2, want2, (what, "behind"))
        got = pair.ring.client_ring_wait(t)
        assert len(got[1]) == 1100
        pair.check(got, data, runs, reqs, want, (what, "overflow"))
        pair.last = t2
    pair.step([(0, replies[:5000])], [Req(rng, 999)], what="after the overflows")
    pair.close()


def test_refusals_and_capacity():
    import brpc_b200
    from brpc_b200.abi import B2_E_CAPACITY, B2_E_INVAL, REPLY_DT, REQUEST_DT
    rng = random.Random(SEED + 4)
    c = _ctx()
    assert _err(c.client_ring_enable, 0, 8, 1 << 16) == B2_E_INVAL                       # a zero cap
    assert _err(c.client_ring_enable, 1 << 16, 0, 1 << 16) == B2_E_INVAL
    assert _err(c.client_ring_enable, 1 << 16, 8, 0) == B2_E_INVAL
    assert _err(c.client_ring_enable, (4 << 20) + 1, 8, 1 << 16) == B2_E_CAPACITY         # max_batch_bytes
    assert _err(c.client_ring_enable, 1 << 16, (1 << 14) + 1, 1 << 16) == B2_E_CAPACITY  # max_msgs
    assert _err(c.client_ring_enable, 1 << 16, 8, (8 << 20) + 1) == B2_E_CAPACITY         # max_resp_bytes
    data, runs, recs = ticket([(0, b"\0" * 32)], [Req(rng, 1)])
    assert _err(c.client_ring_submit, data, runs, recs) == B2_E_INVAL                       # not enabled
    assert _err(c.client_ring_wait, 1) == B2_E_INVAL
    c.client_ring_enable(8192, 3, 4000)
    ok = [Req(rng, 2, stream=False, size=100, compress=0) for _ in range(3)]
    for q in ok:
        q.att = b""
    data, runs, recs = ticket([(0, b"\0" * 32), (1, b"\0" * 32)], ok)
    refused = [
        (B2_E_INVAL, (data, runs[:0], recs[:0])),                                            # neither runs nor requests
        (B2_E_CAPACITY, (np.zeros(8193, np.uint8), runs[:1], recs[:0])),                    # nbytes > max_bytes
        (B2_E_CAPACITY, (np.zeros(8192, np.uint8), np.zeros(513, runs.dtype), recs[:0])),  # 513 runs
        (B2_E_CAPACITY, (data, runs, np.concatenate([recs, recs[:1]]))),                    # n_reqs > max_reqs
    ]
    bad = runs.copy(); bad["offset"][1] = 8
    refused.append((B2_E_INVAL, (data, bad, recs)))                                          # a run not 16-aligned
    bad = runs.copy(); bad["length"][1] = len(data)
    refused.append((B2_E_INVAL, (data, bad, recs)))                                          # a run outside the bytes
    q = recs.copy(); q["payload_len"][2] = len(data)
    refused.append((B2_E_INVAL, (data, runs, q)))                                            # a payload outside the bytes
    q = recs.copy(); q["attachment_off"][0] = len(data); q["attachment_len"][0] = 1
    refused.append((B2_E_INVAL, (data, runs, q)))                                            # an attachment outside the bytes
    big = [Req(rng, 3, stream=False, size=3000, compress=0) for _ in range(2)]
    refused.append((B2_E_CAPACITY, ticket([], big)))                                         # req_out_cap too small
    for i, (code, args) in enumerate(refused):
        assert _err(c.client_ring_submit, *args) == code, i
    ts = [c.client_ring_submit(data, runs, recs) for _ in range(8)]
    assert ts == list(range(1, 9))                                                           # a failed submit takes no ticket number
    assert _err(c.client_ring_submit, data, runs, recs) == B2_E_CAPACITY                    # eight outstanding
    # every call that uploads to the context is refused while a ticket is outstanding
    small = np.zeros(64, np.uint8)
    one = brpc_b200.make_runs([b"\0" * 16])
    uploads = [
        lambda: c.process_batch(*one), lambda: c.upload(*one), lambda: c.pack_requests(small, np.zeros(1, REQUEST_DT)),
        lambda: c.pack_responses(small, np.zeros(1, REPLY_DT)), lambda: c.crc32c_batch(small, [0], [16]),
        lambda: c.snappy_compress_batch(small, [0], [16], 1024), lambda: c.snappy_uncompress_batch(small, [0], [16], 1024),
        lambda: c.hpack_reset(0), lambda: c.hpack_decode_batch(small, [(0, 0, 16)]), lambda: c.h2_scan_batch(*one),
    ]
    for i, f in enumerate(uploads):
        assert _err(f) == B2_E_INVAL, i
    for t in ts[1:]:
        c.client_ring_wait(t)
    for i, f in enumerate(uploads):
        assert _err(f) == B2_E_INVAL, ("one still outstanding", i)
    got = c.client_ring_wait(ts[0])
    assert [len(f) for f in got[4]] == [len(q.frame()) for q in ok]
    assert _err(c.client_ring_wait, ts[0]) == B2_E_INVAL                                    # already collected
    assert _err(c.client_ring_wait, 9) == B2_E_INVAL                                        # not submitted
    c.crc32c_batch(small, [0], [16])                                                         # between tickets they work again
    assert c.pack_requests(data, recs) == [q.frame() for q in ok]
    assert c.client_ring_submit(data, runs, recs) == 9
    c.client_ring_wait(9)
    c.close()


def test_one_ring_kind_per_context():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL
    caps = (1 << 16, 16, 1 << 16)
    rng = random.Random(SEED + 5)
    data, runs = brpc_b200.make_runs([b"\0" * 16])
    cq = Req(rng, 1)
    cdata, cruns, crecs = ticket([], [cq])
    a = _ctx(); a.ring_start()
    assert _err(a.client_ring_enable, *caps) == B2_E_INVAL                                  # after k_ring
    assert _err(a.client_ring_submit, cdata, cruns, crecs) == B2_E_INVAL
    a.ring_wait(a.ring_submit(data, runs))
    assert _err(a.client_ring_wait, 1) == B2_E_INVAL
    b = _ctx(); b.h2_configure(max_conns=8); b.h2_ring_enable(1 << 16, 64, 1 << 16, 1 << 16)
    assert _err(b.client_ring_enable, *caps) == B2_E_INVAL                                  # after k_h2_ring
    c = _ctx(); c.h2_configure(max_conns=8); c.h2_client_ring_enable(1 << 16, 64, 1 << 16, 16, 1 << 16)
    assert _err(c.client_ring_enable, *caps) == B2_E_INVAL                                  # after k_h2_client_ring
    d = _ctx(); d.stream_configure(64, 1 << 16)
    assert _err(d.client_ring_enable, *caps) == B2_E_INVAL                                  # a context with a stream table
    d.stream_ring_enable(1 << 16)
    assert _err(d.client_ring_enable, *caps) == B2_E_INVAL
    e = _ctx(); e.client_ring_enable(*caps)
    assert _err(e.client_ring_enable, *caps) == B2_E_INVAL                                  # twice
    for f in (lambda: e.h2_ring_enable(1 << 16, 64, 1 << 16, 1 << 16), lambda: e.h2_client_ring_enable(1 << 16, 64, 1 << 16, 16, 1 << 16),
              lambda: e.ring_submit(data, runs), lambda: e.h2_ring_submit(data, runs)):
        assert _err(f) == B2_E_INVAL
    t = e.client_ring_submit(cdata, cruns, crecs)
    assert _err(e.ring_wait, t) == B2_E_INVAL and _err(e.h2_ring_wait, t) == B2_E_INVAL and _err(e.h2_client_ring_wait, t) == B2_E_INVAL
    assert e.client_ring_wait(t)[4] == [cq.frame()]
    e.ring_stop(); e.ring_start()                                                            # b2_ring_start serves the context's own kind
    t = e.client_ring_submit(cdata, cruns, crecs)
    assert len(e.client_ring_wait(t)[4][0]) > 0
    for x in (a, b, c, d, e):
        x.close()


def _steady(pair, rng, replies, steps):
    for s in range(steps):
        got = pair.step([(k, replies[k]) for k in range(4)], [Req(rng, 5000 + 4 * s + k, stream=False, size=200) for k in range(4)])
        assert len(got[1]) == 12 and (got[1]["error_code"] == 0).all()


def test_no_launch_over_100_steady_tickets_and_idle_retirement(monkeypatch):
    gc.collect()                                                     # (no context of an earlier test is destroyed while this one counts)
    monkeypatch.setenv("B2_RING_IDLE_MS", "2000")
    rng = random.Random(SEED + 6)
    replies = _server_replies(rng, 4, 3)
    pair = Pair()
    _steady(pair, rng, replies, 1)
    n0 = pair.ring.ring_launches()
    _steady(pair, rng, replies, 100)
    assert pair.ring.ring_launches() == n0
    pair.ring.ring_stop()
    monkeypatch.setenv("B2_RING_IDLE_MS", "5")
    _steady(pair, rng, replies, 1)                                   # relaunched by the submission, now with a 5 ms idle time
    n1 = pair.ring.ring_launches()
    assert n1 == n0 + 1
    time.sleep(0.2)                                                  # it retires and comes back with the next submission
    _steady(pair, rng, replies, 2)
    assert pair.ring.ring_launches() > n1
    ph = pair.ring.ring_phase_ns(pair.last)
    assert 0 < ph[0] <= ph[1] <= ph[2] <= ph[3]
    pair.close()


def test_device_round_trip_client_ring_against_server_ring():
    """1 000 echo calls over 64 connections between a client ring context and a server k_ring context on the same GPU: each side's wire
    bytes are only what its kernel wrote (request frames, replies)"""
    import brpc_b200
    rng = random.Random(SEED + 7)
    n_conns, n_calls = 64, 1000
    client, server = _ctx(), _ctx()
    client.client_ring_enable(MAX_BYTES, MAX_REQS, REQ_OUT)
    sent, answered = {}, 0
    replies = [b""] * n_conns
    cid = 1
    while answered < n_calls:
        reqs = []
        for k in range(n_conns):
            if cid <= n_calls:
                q = Req(rng, (k << 40) | cid, stream=False, compress=0, size=rng.choice([1, 64, 300]))
                q.att, q.cks, q.has_log, q.flags = b"", 0, False, 0
                reqs.append((k, q)); sent[q.cid] = q.payload; cid += 1
        data, runs, recs = ticket([(k, replies[k]) for k in range(n_conns) if replies[k]], [q for _, q in reqs])
        got = client.client_ring_wait(client.client_ring_submit(data, runs, recs))
        rs, msgs = got[0], got[1]
        for r in range(len(rs)):
            assert rs["consumed"][r] == runs["length"][r]
        for m in msgs:
            assert m["status"] == 7 and m["error_code"] == 0
            body = bytes(data[m["frame_off"] + 12 + m["meta_size"]:m["frame_off"] + 12 + m["body_size"]])
            want = sent.pop(int(m["correlation_id"]))
            assert body == bytes([0x0a]) + _varint(len(want)) + want
            answered += 1
        frames = got[4]
        per = [b"".join(f for (k2, _), f in zip(reqs, frames) if k2 == k) for k in range(n_conns)]
        assert all(len(f) > 0 for f in frames)
        replies = [b""] * n_conns
        if any(per):
            sdata, sruns = brpc_b200.make_runs(per)
            srs, smsgs, sresp, _ = server.ring_wait(server.ring_submit(sdata, sruns))
            assert (smsgs["status"] == 0).all() and len(smsgs) == len(frames)
            for k in range(n_conns):
                ms = smsgs[srs[k]["first_msg"]:srs[k]["first_msg"] + srs[k]["n_msgs"]]
                replies[k] = b"".join(bytes(sresp[m["resp_off"]:m["resp_off"] + m["resp_len"]]) for m in ms)
    assert not sent and answered == n_calls
    client.close(); server.close()


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7f) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)
