"""GPU: the stream pass on the latency path (b2_stream_ring_enable): k_ring runs it after each ticket's batch.  Every ticket is checked
against the sequential oracles of tests/_streams.py / tests/_stream_write.py (messages and their bytes, events, control frames, RST per
run, b2_stream_query of every stream) and against a twin context that runs b2_process_batch with the same table on the same sequence."""
import random
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import _stream_write as W  # noqa: E402
import _streams as S  # noqa: E402
from _compare import assert_same  # noqa: E402
from _traffic import SEED, echo_frame  # noqa: E402
from test_gpu_streams import F, check_batch, traffic  # noqa: E402

RING_BYTES = 120 << 10       # a ticket: at most 128 KiB of input


def frames_of(wire):
    """a socket's bytes cut back into its frames (STRM and PRPC share the 12-byte head with the body size at 4..8)"""
    out, p = [], 0
    while p < len(wire):
        n = 12 + int.from_bytes(wire[p + 4:p + 8], "big")
        out.append(wire[p:p + n]); p += n
    return out


def tickets_of(rng, socks, n):
    """every socket's frames in order, cut into n tickets (frames whole, so a batch consumes all of it); a ticket above RING_BYTES
    is cut further"""
    per = [frames_of(s) for s in socks]
    out = []
    for k in range(n):
        chunks = []
        for fr in per:
            left = len(fr)
            take = left if k == n - 1 else min(left, rng.randrange(0, 2 * left // max(1, n - k) + 2))
            chunks.append(fr[:take]); del fr[:take]
        while sum(len(b"".join(c)) + 16 for c in chunks) > RING_BYTES:
            i = max(range(len(chunks)), key=lambda j: len(b"".join(chunks[j])))
            h = len(chunks[i]) // 2
            out.append([b"".join(c[:h]) if j == i else b"" for j, c in enumerate(chunks)])
            chunks[i] = chunks[i][h:]
        out.append([b"".join(c) for c in chunks])
    return out


class Pair:
    """the ring context and its twin (b2_process_batch), each with its own oracle"""

    def __init__(self, b2, max_streams, pending, out, oracle=S.StreamOracle):
        self.b2 = b2
        self.ring = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=512)
        self.twin = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=512)
        for c in (self.ring, self.twin):
            c.stream_configure(max_streams, pending, out)
        self.ring.stream_ring_enable(out)
        self.orc = oracle(pending_bytes=pending, out_bytes=out)
        self.orc_twin = oracle(pending_bytes=pending, out_bytes=out)
        self.opened = []

    def open(self, streams):
        """streams: [(id, remote, sock, connected, need_feedback[, max_buf])]"""
        for c in (self.ring, self.twin):
            c.stream_open([(t[0], t[1], t[2], (1 if t[3] else 0) | (2 if t[4] else 0)) + tuple(t[5:]) for t in streams])
        for o in (self.orc, self.orc_twin):
            for t in streams:
                o.open(*t)
        self.opened += [t[0] for t in streams]

    def submit(self, chunks):
        data, runs = self.b2.make_runs(chunks)
        return self.ring.ring_submit(data, runs), data, runs

    def wait(self, ticket, data, runs, what, query=True):
        """query=False while later tickets are outstanding: k_ring may already have moved the table past this ticket"""
        dev = self.ring.ring_wait(ticket)
        twin = self.twin.process_batch(data, runs)
        assert_same(dev, twin[:3], what + ": descriptors and replies of the twin")
        check_batch(self.ring, self.orc, data, dev, self.opened if query else [], what + " (ring)")
        check_batch(self.twin, self.orc_twin, data, twin, self.opened, what + " (twin)")
        return dev

    def step(self, chunks, what):
        t, data, runs = self.submit(chunks)
        return self.wait(t, data, runs, what)

    def close(self):
        self.ring.ring_stop(); self.ring.close(); self.twin.close()


def test_seeded_traffic_one_ticket_at_a_time_and_eight_in_flight():
    import brpc_b200 as b2
    rng = random.Random(SEED + 40)
    streams, socks = traffic(rng, 300, 16, 900, 4)
    p = Pair(b2, 512, 16 << 10, 256 << 10)
    p.open(streams)
    tickets = tickets_of(rng, socks, 14)
    assert len(tickets) >= 14
    for k, chunks in enumerate(tickets[:6]):
        p.step(chunks, "ticket %d" % k)
    # eight tickets in flight before the first wait; messages straddle them through the pending pool
    rest = tickets[6:14]
    inflight = [p.submit(c) for c in rest]
    for k, (t, data, runs) in enumerate(inflight):
        p.wait(t, data, runs, "in flight %d" % k, query=k == len(inflight) - 1)
    for k, chunks in enumerate(tickets[14:]):
        p.step(chunks, "tail %d" % k)
    p.close()


def test_hand_over_from_a_small_out_region_then_take_pending():
    import brpc_b200 as b2
    p = Pair(b2, 8, 1024, 4096)
    p.open([(sid, 100 + sid, 9, True, True) for sid in (1, 2, 3)])
    a, b = bytes(range(200)) * 4, b"z" * 700
    batches = [[F(1, cont=True, data=a), F(2, data=b"whole"), F(3, cont=True, data=b"q" * 1000)],
               [F(1, cont=True, data=b), F(2, cont=True, data=b"p" * 3000), F(2, cont=True, data=b"p" * 3000), F(2, data=b"tail"), F(3, data=b"fits")],
               [F(1, 4, data=b"frames of a handed-over stream are described only"), F(2, 4, S.CLOSE), F(3, data=b"still served")]]
    for k, frames in enumerate(batches):
        p.step([b"".join(frames)], "hand-over ticket %d" % k)
    assert p.ring.stream_query(1)["flags"] & 8 and p.ring.stream_query(2)["flags"] & 8
    assert p.ring.stream_take_pending(1, 4096) == a and p.ring.stream_take_pending(1, 4096) == b""
    p.close()


def test_table_calls_between_tickets_and_refused_while_one_is_outstanding():
    import brpc_b200 as b2
    p = Pair(b2, 16, 4096, 1 << 16)
    p.open([(1, 0, 7, False, False), (2, 102, 7, True, True)])
    p.step([F(1, 9, data=b"before the settings") + F(2, 5, cont=True, data=b"half")], "unconnected")
    t, data, runs = p.submit([F(2, 5, data=b" and half")])
    r = p.ring
    for call in (lambda: r.stream_open([(3, 0, 0, 0)]), lambda: r.stream_set_connected(1, 9, 2), lambda: r.stream_close(2),
                 lambda: r.stream_take_pending(2, 64), lambda: r.stream_write([(2, 0, 0, 4)], data=b"abcd")):
        with pytest.raises(b2.B2Error):
            call()
    p.wait(t, data, runs, "after the refusals")
    assert p.ring.stream_set_connected(1, 9, 2) == p.orc.set_connected(1, 9, True) != b""
    assert p.twin.stream_set_connected(1, 9, 2) == p.orc_twin.set_connected(1, 9, True)
    p.open([(3, 103, 8, True, True)])
    p.step([F(1, 9, data=b"now connected") + F(3, 5, data=b"new")], "connected")
    assert p.ring.stream_close(2) == p.orc.close(2) != b""
    assert p.twin.stream_close(2) == p.orc_twin.close(2)
    p.opened.remove(2)
    p.step([F(2, 5, data=b"closed locally") + F(3, 5, data=b"again")], "after close")
    p.close()


def test_from_msg_writes_between_tickets_and_writable_after_feedback():
    import brpc_b200 as b2
    p = Pair(b2, 16, 4096, 1 << 16, oracle=W.WriteOracle)
    p.open([(1, 101, 4, True, True, 8), (2, 102, 5, True, False, 0)])
    body = bytes(range(256)) * 3
    dev = p.step([F(1, 5, data=b"single frame") + F(2, 5, cont=True, data=body[:300]) + F(2, 5, data=body[300:])], "data")
    msgs = p.ring.stream_results()[0]
    assert len(msgs) == 2
    order = {int(m["stream_id"]): i for i, m in enumerate(msgs)}
    writes = [(1, b2.abi.STREAM_W_FROM_MSG, order[1], 0), (2, b2.abi.STREAM_W_FROM_MSG, order[2], 0), (1, b2.abi.STREAM_W_FROM_MSG, order[1], 0)]
    want, want_out = p.orc.write_many([(1, b"single frame"), (2, body), (1, b"single frame")])
    for c in (p.ring, p.twin):
        tm = c.stream_results()[0]
        tw = [(w[0], w[1], {int(m["stream_id"]): i for i, m in enumerate(tm)}[w[0]], 0) for w in writes]
        res, out = c.stream_write(tw)
        got = [(int(r["status"]), int(r["n_frames"]), out[int(r["out_off"]):int(r["out_off"]) + int(r["out_len"])].tobytes(), int(r["produced"])) for r in res]
        assert got == [(w["status"], w["n_frames"], b"".join(w["frames"]), w["produced"]) for w in want]
    p.orc_twin.write_many([(1, b"single frame"), (2, body), (1, b"single frame")])
    assert want[2]["status"] == W.EAGAIN            # the window of stream 1 is full now
    dev = p.step([S.feedback_frame(1, 101, 100)], "feedback")
    ev = p.ring.stream_results()[1]
    assert int(ev[0]["flags"]) & W.EV_WRITABLE
    # FROM_MSG resolves against the most recent ticket: a single-frame message in the ring's device copy of its input, a multi-frame
    # one in the ring's out region; a call that uploads other bytes overwrites the input, not the out region
    p.step([F(2, 5, data=b"one frame") + F(2, 5, cont=True, data=body[:100]) + F(2, 5, data=body[100:200])], "one more")
    msgs = p.ring.stream_results()[0]
    assert [int(m["n_frames"]) for m in msgs] == [1, 2]
    with pytest.raises(b2.B2Error):
        p.ring.stream_write([(2, b2.abi.STREAM_W_FROM_MSG, 2, 0)])
    res, out = p.ring.stream_write([(2, b2.abi.STREAM_W_FROM_MSG, 0, 0)])
    assert out[int(res[0]["out_off"]):int(res[0]["out_off"]) + int(res[0]["out_len"])].tobytes() == W.data_frame(102, 2, False, b"one frame")
    p.ring.crc32c_batch(np.zeros(64, np.uint8), np.zeros(1, np.uint32), np.full(1, 64, np.uint32))
    with pytest.raises(b2.B2Error):
        p.ring.stream_write([(2, b2.abi.STREAM_W_FROM_MSG, 0, 0)])
    res, out = p.ring.stream_write([(2, b2.abi.STREAM_W_FROM_MSG, 1, 0)])
    assert out[int(res[0]["out_off"]):int(res[0]["out_off"]) + int(res[0]["out_len"])].tobytes() == W.data_frame(102, 2, False, body[:200])
    p.close()


def test_idle_retirement_and_an_overflowing_ticket_with_tickets_behind_it():
    import brpc_b200 as b2
    rng = random.Random(SEED + 41)
    p = Pair(b2, 64, 4096, 1 << 16)
    p.open([(sid, 1000 + sid, sid % 4, True, True) for sid in range(1, 33)])
    p.step([F(sid, 5, cont=True, data=rng.randbytes(40)) for sid in range(1, 33)], "before the sleep")
    n0 = p.ring.ring_launches()
    time.sleep(0.25)                       # the kernel retires after its idle time and comes back with the next submission
    p.step([F(sid, 5, data=rng.randbytes(30)) for sid in range(1, 17)], "after the sleep")
    assert p.ring.ring_launches() > n0
    # the middle ticket has more messages than the compact block holds: the big pipeline serves it inside ring_wait while k_ring
    # waits before the tickets behind it
    echoes = b"".join(echo_frame(rng, i, b"") for i in range(1500))
    queued = [p.submit([F(sid, 5, cont=True, data=rng.randbytes(20)) for sid in range(17, 33)]),
              p.submit([echoes, b"".join(F(sid, 5, data=rng.randbytes(25)) for sid in range(1, 33))]),
              p.submit([b"".join(F(sid, 5, data=rng.randbytes(10)) for sid in range(9, 33))]),
              p.submit([S.feedback_frame(sid, 1000 + sid, 7) + F(sid, 5, S.RST) for sid in range(1, 5)])]
    with pytest.raises(b2.B2Error):
        p.ring.ring_wait(queued[1][0])     # tickets of a table context are collected in order
    for k, (t, data, runs) in enumerate(queued):
        dev = p.wait(t, data, runs, "queued %d" % k, query=k == len(queued) - 1)
        if k == 1:
            assert len(dev[1]) > 1500
    p.close()


def test_the_ring_without_the_opt_in_and_the_opt_in_rules():
    import brpc_b200 as b2
    ctx = b2.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=16)
    with pytest.raises(b2.B2Error):
        ctx.stream_ring_enable(4096)       # no table
    ctx.stream_configure(8, 1024)
    data, runs = b2.make_runs([F(1, data=b"x")])
    with pytest.raises(b2.B2Error):
        ctx.ring_submit(data, runs)        # a table without the opt-in
    ctx.stream_ring_enable(4096)
    with pytest.raises(b2.B2Error):
        ctx.stream_ring_enable(4096)       # twice
    t = ctx.ring_submit(data, runs)
    assert len(ctx.ring_wait(t)[1]) == 1
    ctx.ring_stop(); ctx.close()
    ctx = b2.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=16)
    ctx.stream_configure(8, 1024)
    ctx.ring_start()
    with pytest.raises(b2.B2Error):
        ctx.stream_ring_enable(4096)       # after the first ring call
    ctx.ring_stop(); ctx.close()
