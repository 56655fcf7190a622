"""GPU: a Stream producer's turn on the latency path (b2_stream_ring_*).  A ticket serves the frames the peers sent (the batch, then the
stream pass, as a stream-ring ticket) and then the queued writes (as b2_stream_write), inside the resident k_ring.  Every ticket is
compared with a twin context that runs b2_process_batch + b2_stream_write on the same table, and with the sequential oracles of
tests/_streams.py / tests/_stream_write.py: descriptors and replies, messages, events and control frames, every write result and frame
byte (the zero gaps included), and b2_stream_query of every stream."""
import random
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import _oracle as O  # noqa: E402
import _stream_write as W  # noqa: E402
import _streams as S  # noqa: E402
from _compare import assert_same  # noqa: E402
from _traffic import SEED, echo_frame  # noqa: E402
from test_gpu_streams import F, check_batch  # noqa: E402

MAX_BYTES, MAX_WRITES, WRITE_OUT = 2 << 20, 512, 4 << 20
RES_FIELDS = ("status", "n_frames", "out_off", "out_len", "produced", "host_socket_id")


def _ctx(b2):
    return b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=512, max_resp_bytes=8 << 20)


def _code(fn, *a):
    from brpc_b200.abi import B2Error
    try:
        fn(*a)
    except B2Error as e:
        return e.code
    return 0


def ticket_bytes(chunks, payloads, rng):
    """the runs' bytes (16-aligned runs) followed by every payload at an unaligned offset -> (data, runs, [(off, len)])"""
    import brpc_b200 as b2
    data, runs = b2.make_runs(chunks) if chunks else (np.zeros(0, np.uint8), np.zeros(0, b2.abi.RUN_DT))
    parts, spans, off = [data.tobytes()], [], len(data)
    for p in payloads:
        gap = rng.randrange(16)
        parts.append(b"\xee" * gap); off += gap
        spans.append((off, len(p))); parts.append(p); off += len(p)
    return np.frombuffer(b"".join(parts) or b"\0" * 16, np.uint8).copy(), runs, spans


class Pair:
    """the ring context, its twin, and an oracle for each"""

    def __init__(self, b2, max_streams, pending, out, seg):
        self.b2, self.seg = b2, seg
        self.ring, self.twin = _ctx(b2), _ctx(b2)
        for c in (self.ring, self.twin):
            c.stream_configure(max_streams, pending, out)
        self.ring.stream_ring_enable(out)
        self.ring.stream_ring_write_enable(MAX_BYTES, MAX_WRITES, WRITE_OUT, seg)
        self.orc = W.WriteOracle(pending_bytes=pending, out_bytes=out)
        self.orc_twin = W.WriteOracle(pending_bytes=pending, out_bytes=out)
        self.opened = []

    def open(self, streams):
        """streams: [(id, remote, sock, connected, need_feedback, max_buf)]"""
        for c in (self.ring, self.twin):
            c.stream_open([(t[0], t[1], t[2], (1 if t[3] else 0) | (2 if t[4] else 0), t[5]) for t in streams])
        for o in (self.orc, self.orc_twin):
            for t in streams:
                o.open(*t)
        self.opened += [t[0] for t in streams]

    def submit(self, chunks, writes, rng, pin=None):
        """writes: [(sid, payload)] -> (ticket, the ticket's inputs)"""
        data, runs, spans = ticket_bytes(chunks, [p for _, p in writes], rng)
        desc = [(sid, 0, off, n) for (sid, _), (off, n) in zip(writes, spans)]
        if pin is not None:
            pin.array[:len(data)] = data
            t = self.ring.stream_ring_submit(None, runs, desc, ptr=pin.ptr, nbytes=len(data))
        else:
            t = self.ring.stream_ring_submit(data, runs, desc)
        return t, (data, runs, desc, writes)

    def wait(self, t, inputs, what, query=True):
        """query=False while later tickets are outstanding: k_ring may already have moved the table past this ticket"""
        data, runs, desc, writes = inputs
        rs, msgs, resp, info, res, out = self.ring.stream_ring_wait(t)
        if len(runs):
            twin = self.twin.process_batch(data, runs)
            assert_same((rs, msgs, resp), twin[:3], what + ": descriptors and replies of the twin")
            check_batch(self.ring, self.orc, data, (rs, msgs, resp), self.opened if query else [], what + " (ring)")
            check_batch(self.twin, self.orc_twin, data, twin, self.opened, what + " (twin)")
        else:
            assert len(rs) == 0 and len(msgs) == 0
            smsgs, events, sout, ctrl, run_ctrl = self.ring.stream_results()
            assert len(smsgs) == len(events) == len(sout) == len(ctrl) == len(run_ctrl) == 0, what + ": a ticket without runs is an empty pass"
        assert len(res) == len(writes), what
        if writes:
            tres, tout = self.twin.stream_write(desc, data, self.seg)
            want, want_out = self.orc.write_many(writes, self.seg)
            self.orc_twin.write_many(writes, self.seg)
            assert res.tobytes() == tres.tobytes(), what + ": write results of the twin"
            assert out.tobytes() == tout[:len(out)].tobytes() == want_out, what + ": frames"
            for i, (r, w) in enumerate(zip(res, want)):
                assert {k: int(r[k]) for k in RES_FIELDS} == {k: w[k] for k in RES_FIELDS}, "%s write %d" % (what, i)
        else:
            assert len(out) == 0
        if query:
            for sid in self.opened:
                assert self.ring.stream_query(sid) == self.twin.stream_query(sid), "%s query %d" % (what, sid)
        return rs, msgs, resp, info, res, out

    def step(self, chunks, writes, rng, what, pin=None):
        t, inputs = self.submit(chunks, writes, rng, pin)
        return self.wait(t, inputs, what)

    def close(self):
        self.ring.ring_stop(); self.ring.close(); self.twin.close()


def producer_streams(rng, n):
    ids = rng.sample(range(1, 1 << 40), n)
    return [(sid, rng.randrange(1, 1 << 50), rng.randrange(64), rng.random() < 0.9, rng.random() < 0.7,
             rng.choice((0, 0, 300, 4096, 20000, 1 << 20))) for sid in ids]


def peer_frames(rng, p, live, remote_of):
    """what the peers send in one turn: FEEDBACK on many windowed streams (some moving remote_consumed past produced), DATA, an RST or
    CLOSE now and then, baidu_std echo requests on the same sockets -> per-socket byte strings"""
    socks = [[] for _ in range(64)]
    for sid in rng.sample(live, min(len(live), 80)):
        s = p.orc.streams[sid]
        r = rng.random()
        if r < 0.6:
            c = rng.choice((s.produced, s.produced // 2, s.remote_consumed, s.produced + 5))
            socks[s.sock].append(S.feedback_frame(sid, remote_of[sid], c))
        elif r < 0.97:
            for k in range(rng.choice((1, 1, 2))):
                socks[s.sock].append(F(sid, remote_of[sid], S.DATA, True if k == 0 and rng.random() < 0.2 else None, rng.randbytes(rng.randrange(300))))
        else:
            socks[s.sock].append(F(sid, remote_of[sid], rng.choice((S.RST, S.CLOSE))))
    for _ in range(6):
        socks[rng.randrange(64)].append(echo_frame(rng, rng.randrange(200)))
    for q in socks:
        rng.shuffle(q)
    return [b"".join(q) for q in socks]


def queued_writes(rng, p, sids):
    """host-sourced writes of 0 B to 64 KiB, mostly small"""
    def length():
        r = rng.random()
        return 0 if r < 0.03 else rng.randrange(1, 600) if r < 0.7 else rng.randrange(8 << 10) if r < 0.95 else rng.randrange((64 << 10) + 1)
    return [(rng.choice(sids), rng.randbytes(length())) for _ in range(rng.randrange(20, 60))]


@pytest.mark.parametrize("seg", [0, 4096, 100, 40])
def test_seeded_producer_traffic_one_ticket_at_a_time_and_eight_in_flight(seg):
    """about 300 streams on 64 sockets; the peers' frames arrive cut at random offsets across tickets (one at a time: the bytes a run did
    not consume come back at the head of its socket's next run); seg 40 takes the byte-wise copy branch"""
    import brpc_b200 as b2
    rng = random.Random(SEED + 60 + seg)
    streams = producer_streams(rng, 300)
    p = Pair(b2, 512, 4096, 1 << 20, seg)
    p.open(streams)
    sids = [t[0] for t in streams]
    remote_of = {t[0]: t[1] for t in streams}
    carry = [b""] * 64
    for k in range(8):
        live = [sid for sid in sids if not p.orc.streams[sid].closed]
        wire = [carry[i] + w for i, w in enumerate(peer_frames(rng, p, live, remote_of))]
        cut = [w[:rng.randrange(len(w) + 1)] if w and rng.random() < 0.5 else w for w in wire]
        chunks = [c for c in cut]
        rs = p.step(chunks, queued_writes(rng, p, sids), rng, "seg %d ticket %d" % (seg, k))[0]
        carry = [wire[i][int(rs[i]["consumed"]):] for i in range(64)]
        assert all(int(rs[i]["consumed"]) <= len(cut[i]) for i in range(64))
    # eight tickets in flight before the first wait: whole frames (every run is consumed), the oracle's windows as of the submission
    live = [sid for sid in sids if not p.orc.streams[sid].closed]
    pending = []
    for k in range(8):
        wire = peer_frames(rng, p, live, remote_of)
        if k == 0:
            wire = [carry[i] + w for i, w in enumerate(wire)]
        pending.append(p.submit(wire, queued_writes(rng, p, sids), rng))
    for k, (t, inputs) in enumerate(pending):
        p.wait(t, inputs, "seg %d in flight %d" % (seg, k), query=k == len(pending) - 1)
    p.close()


def test_order_inside_a_ticket_read_then_write():
    """a FEEDBACK in the runs admits the same ticket's write; a CLOSE or RST in the runs makes the same ticket's writes EINVAL; WRITABLE
    keeps its meaning"""
    import brpc_b200 as b2
    rng = random.Random(SEED + 61)
    p = Pair(b2, 16, 4096, 1 << 16, 0)
    p.open([(1, 101, 0, True, True, 100), (2, 102, 0, True, True, 0), (3, 103, 1, True, True, 0), (4, 104, 1, True, True, 50)])
    res = p.step([], [(1, b"x" * 100), (1, b"y" * 10), (4, b"z" * 60)], rng, "fill the windows")[4]
    assert [int(r["status"]) for r in res] == [0, W.EAGAIN, 0]
    res = p.step([S.feedback_frame(1, 101, 100), F(2, 102, S.CLOSE)], [(1, b"a" * 7), (2, b"b"), (4, b"c")], rng, "read, then write")[4]
    assert [int(r["status"]) for r in res] == [0, W.EINVAL, W.EAGAIN]
    _, events, _, _, _ = p.ring.stream_results()
    ev = {int(e["stream_id"]): int(e["flags"]) for e in events}
    assert ev[1] & W.EV_WRITABLE and ev[2] & S.EV_CLOSE
    res = p.step([F(3, 103, S.RST) + S.feedback_frame(4, 104, 10)], [(3, b"d"), (4, b"e" * 3)], rng, "rst, then write")[4]
    assert [int(r["status"]) for r in res] == [W.EINVAL, W.EAGAIN]
    _, events, _, _, _ = p.ring.stream_results()
    assert {int(e["stream_id"]): int(e["flags"]) & W.EV_WRITABLE for e in events} == {3: 0, 4: 0}     # 60 >= 10 + 50: still full
    p.close()


def test_ticket_shapes_pinned_bytes_and_streams_that_cannot_take_writes():
    """write-only and runs-only tickets, pinned (pulled in place) and staged bytes, a stream that is not connected and one the receive
    pass handed over"""
    import brpc_b200 as b2
    rng = random.Random(SEED + 62)
    p = Pair(b2, 16, 1024, 1 << 16, 4096)
    p.open([(1, 101, 0, True, True, 1 << 16), (2, 0, 0, False, False, 0), (3, 103, 1, True, True, 0)])
    pin = b2.abi.PinnedBuffer(1 << 20)
    p.step([], [(1, rng.randbytes(5000)), (2, b"early"), (3, rng.randbytes(20))], rng, "write-only, staged")
    p.step([F(3, 103, S.DATA, True, b"p" * 2000)], [], rng, "runs-only: stream 3 handed over")
    assert p.ring.stream_query(3)["flags"] & b2.abi.STREAM_HANDED_OVER
    res = p.step([S.feedback_frame(1, 101, 5000)], [(1, rng.randbytes(9000)), (2, b"still early"), (3, b"to a handed-over stream")], rng, "pinned", pin)[4]
    assert [int(r["status"]) for r in res] == [0, W.NOT_CONNECTED, W.HANDED_OVER]
    p.step([], [(1, rng.randbytes(64 << 10))], rng, "write-only, pinned", pin)
    pin.free()
    p.close()


def test_an_overflowing_ticket_with_writes_and_tickets_queued_behind_it():
    import brpc_b200 as b2
    rng = random.Random(SEED + 63)
    p = Pair(b2, 64, 4096, 1 << 16, 1000)
    p.open([(sid, 1000 + sid, sid % 4, True, True, 3000) for sid in range(1, 33)])
    sids = list(range(1, 33))
    echoes = b"".join(echo_frame(rng, i, b"") for i in range(1500))
    queued = [p.submit([F(sid, 1000 + sid, S.DATA, None, rng.randbytes(20)) for sid in sids[:8]], [(sid, rng.randbytes(1500)) for sid in sids], rng),
              p.submit([echoes, b"".join(S.feedback_frame(sid, 1000 + sid, 1500) for sid in sids)], [(sid, rng.randbytes(2000)) for sid in sids], rng),
              p.submit([b"".join(S.feedback_frame(sid, 1000 + sid, 3500) for sid in sids[:16])], [(sid, rng.randbytes(700)) for sid in sids], rng),
              p.submit([], [(sid, rng.randbytes(100)) for sid in sids], rng)]
    with pytest.raises(b2.B2Error):
        p.ring.stream_ring_wait(queued[1][0])     # tickets of a table context are collected in order
    for k, (t, inputs) in enumerate(queued):
        dev = p.wait(t, inputs, "queued %d" % k, query=k == len(queued) - 1)
        if k == 1:
            assert len(dev[1]) > 1024 and any(int(r["status"]) == 0 for r in dev[4])
    p.close()


def test_idle_retirement_and_no_launches_over_steady_tickets(monkeypatch):
    import brpc_b200 as b2
    rng = random.Random(SEED + 64)
    monkeypatch.setenv("B2_RING_IDLE_MS", "5")
    p = Pair(b2, 64, 4096, 1 << 16, 0)
    p.open([(sid, 2000 + sid, sid % 8, True, True, 30000) for sid in range(1, 33)])
    p.step([S.feedback_frame(sid, 2000 + sid, 0) for sid in range(1, 9)], [(sid, rng.randbytes(40000)) for sid in range(1, 33)], rng, "before the sleep")
    n0 = p.ring.ring_launches()
    time.sleep(0.2)                            # the kernel retires after its idle time and comes back with the next submission
    res = p.step([], [(sid, rng.randbytes(100)) for sid in range(1, 33)], rng, "after the sleep")[4]
    assert p.ring.ring_launches() > n0
    assert all(int(r["status"]) == W.EAGAIN for r in res)                # the windows survived the relaunch
    monkeypatch.setenv("B2_RING_IDLE_MS", "2000")
    time.sleep(0.05)
    p.step([S.feedback_frame(1, 2001, 40000)], [(1, b"warm")], rng, "warm")
    n1 = p.ring.ring_launches()
    for k in range(100):
        sid = 1 + k % 32
        s = p.orc.streams[sid]
        t, inputs = p.submit([S.feedback_frame(sid, 2000 + sid, s.produced)], [(sid, rng.randbytes(rng.randrange(1, 4096)))], rng)
        p.wait(t, inputs, "steady %d" % k, query=k % 25 == 24)
    assert p.ring.ring_launches() == n1
    p.close()


def test_refusals_and_the_one_kind_rules():
    import brpc_b200 as b2
    INVAL, CAP = b2.abi.B2_E_INVAL, b2.abi.B2_E_CAPACITY
    # enable order
    c = _ctx(b2)
    assert _code(c.stream_ring_write_enable, MAX_BYTES, MAX_WRITES, WRITE_OUT) == INVAL        # no stream ring
    c.stream_configure(8, 1024)
    assert _code(c.stream_ring_write_enable, MAX_BYTES, MAX_WRITES, WRITE_OUT) == INVAL        # a table, no stream ring yet
    c.stream_ring_enable(4096)
    assert _code(c.stream_ring_write_enable, 0, MAX_WRITES, WRITE_OUT) == INVAL
    assert _code(c.stream_ring_write_enable, MAX_BYTES, 0, WRITE_OUT) == INVAL
    assert _code(c.stream_ring_write_enable, MAX_BYTES, MAX_WRITES, 0) == INVAL
    assert _code(c.stream_ring_write_enable, (4 << 20) + 1, MAX_WRITES, WRITE_OUT) == CAP
    assert _code(c.stream_ring_write_enable, MAX_BYTES, (1 << 14) + 1, WRITE_OUT) == CAP
    assert _code(c.stream_ring_write_enable, MAX_BYTES, MAX_WRITES, (8 << 20) + 1) == CAP
    c.stream_ring_write_enable(64 << 10, 4, 4096, 1000)
    assert _code(c.stream_ring_write_enable, 64 << 10, 4, 4096, 1000) == INVAL                 # twice
    c.close()
    c = _ctx(b2)
    c.stream_configure(8, 1024); c.stream_ring_enable(4096); c.ring_start()
    assert _code(c.stream_ring_write_enable, MAX_BYTES, MAX_WRITES, WRITE_OUT) == INVAL        # after the first ring call
    c.ring_stop(); c.close()
    c = _ctx(b2)
    c.client_ring_enable(1 << 16, 4, 1 << 16)
    assert _code(c.stream_ring_write_enable, MAX_BYTES, MAX_WRITES, WRITE_OUT) == INVAL        # another kind
    assert _code(c.stream_ring_submit, np.zeros(16, np.uint8), [], [(1, 0, 0, 1)]) == INVAL
    c.close()
    # submit checks against the enable-time caps: nothing claimed, the ticket numbers go on
    rng = random.Random(SEED + 65)
    p = Pair(b2, 16, 1024, 1 << 16, 0)
    p.ring.close(); p.ring = _ctx(b2)
    p.ring.stream_configure(16, 1024, 1 << 16); p.ring.stream_ring_enable(1 << 16); p.ring.stream_ring_write_enable(64 << 10, 4, 4096, 1000)
    p.open([(1, 101, 0, True, True, 0), (2, 102, 0, True, True, 0)])
    r = p.ring
    data, runs = b2.make_runs([F(1, 101, S.DATA, None, b"hello")])
    big = np.zeros(64 << 10, np.uint8)
    t0 = r.stream_ring_submit(data, runs, [(1, 0, 0, 4)])
    r.stream_ring_wait(t0)
    bad_runs = runs.copy(); bad_runs[0]["offset"] = 3
    assert _code(r.stream_ring_submit, data, [], []) == INVAL                                   # neither runs nor writes
    assert _code(r.stream_ring_submit, np.zeros((64 << 10) + 16, np.uint8), [], [(1, 0, 0, 1)]) == CAP     # above max_bytes
    assert _code(r.stream_ring_submit, data, bad_runs, []) == INVAL                            # a run not 16-aligned
    assert _code(r.stream_ring_submit, data, np.zeros(513, b2.abi.RUN_DT), []) == CAP          # more than 512 runs
    assert _code(r.stream_ring_submit, data, [], [(1, 0, 0, 1)] * 5) == CAP                    # above max_writes
    assert _code(r.stream_ring_submit, data, [], [(1, 2, 0, 1)]) == INVAL                      # an unknown flag
    assert _code(r.stream_ring_submit, data, [], [(1, b2.abi.STREAM_W_FROM_MSG, 0, 0)]) == INVAL     # FROM_MSG in a ticket
    assert _code(r.stream_ring_submit, data, [], [(1, 0, len(data) - 2, 3)]) == INVAL          # outside bytes
    assert _code(r.stream_ring_submit, big, [], [(1, 0, 0, 4000), (2, 0, 0, 100)]) == CAP      # frames above write_out_cap
    assert _code(r.ring_submit, data, runs) == INVAL                                           # b2_ring_submit on this kind
    assert _code(r.ring_wait, t0) == INVAL
    assert _code(r.client_ring_submit, data, runs, np.zeros(0, b2.abi.REQUEST_DT)) == INVAL
    # while a ticket is outstanding the table calls and b2_stream_write are refused; between tickets they work
    t = r.stream_ring_submit(data, runs, [(2, 0, 0, 4)])
    assert t == t0 + 1
    for call in (lambda: r.stream_open([(3, 0, 0, 0)]), lambda: r.stream_set_connected(1, 9, 2), lambda: r.stream_close(2),
                 lambda: r.stream_take_pending(2, 64), lambda: r.stream_write([(2, 0, 0, 4)], data=b"abcd"),
                 lambda: r.stream_write([(1, b2.abi.STREAM_W_FROM_MSG, 0, 0)])):
        assert _code(call) == INVAL
    assert _code(r.ring_wait, t) == INVAL
    res = r.stream_ring_wait(t)[4]
    assert [int(x["status"]) for x in res] == [0]
    # a FROM_MSG b2_stream_write between tickets: served against the most recent ticket's message
    msgs = r.stream_results()[0]
    assert len(msgs) == 1
    wres, wout = r.stream_write([(2, b2.abi.STREAM_W_FROM_MSG, 0, 0)])
    assert wout[int(wres[0]["out_off"]):int(wres[0]["out_off"]) + int(wres[0]["out_len"])].tobytes() == W.data_frame(102, 2, False, b"hello")
    r.stream_open([(3, 103, 0, 3)])
    assert r.stream_close(3) != b""
    t = r.stream_ring_submit(data, [], [(3, 0, 0, 1), (1, 0, 0, 0)])
    assert [int(x["status"]) for x in r.stream_ring_wait(t)[4]] == [W.EINVAL, W.EINVAL]
    r.ring_stop(); r.close(); p.twin.close()
