"""GPU: the stream pass (b2_stream_*) against the sequential oracle of tests/_streams.py — completed messages and their bytes, events,
control frames (RST per run, FEEDBACK / CLOSE per stream) and b2_stream_query state, over seeded traffic whose messages and frames
straddle batches, with baidu_std echo requests on the same sockets (answered exactly as a context without a table answers them)."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import _oracle as O  # noqa: E402
import _streams as S  # noqa: E402
from _compare import assert_same  # noqa: E402
from _traffic import SEED, echo_frame  # noqa: E402

NONE = 0xffffffff


def F(sid, src=-1, t=S.DATA, cont=None, data=b""):
    return O.pack_stream_frame(sid, src, t, cont, data)


def check_batch(ctx, orc, data, dev, opened, what):
    """device == oracle for one collected batch"""
    rs, msgs = dev[0], dev[1]
    smsgs, events, out, ctrl, run_ctrl = ctx.stream_results()
    want_msgs, want_ev, want_rst = orc.process(data, rs, msgs)
    data = np.asarray(data)
    assert sorted(int(e["stream_id"]) for e in events) == sorted(want_ev), what
    total_ctrl = 0
    for e in events:
        sid = int(e["stream_id"]); w = want_ev[sid]; tag = "%s stream %d" % (what, sid)
        got = dict(flags=int(e["flags"]), n_msgs=int(e["n_msgs"]), consumed=int(e["consumed_bytes"]), local_consumed=int(e["local_consumed"]),
                   remote_consumed=int(e["remote_consumed"]), pending_bytes=int(e["pending_bytes"]), sock=int(e["host_socket_id"]),
                   handover_msg=None if int(e["handover_msg"]) == NONE else int(e["handover_msg"]),
                   fb=ctrl[int(e["fb_off"]):int(e["fb_off"]) + int(e["fb_len"])].tobytes(), close=ctrl[int(e["close_off"]):int(e["close_off"]) + int(e["close_len"])].tobytes())
        assert got == {k: w[k] for k in got}, tag
        if got["fb"] and got["close"]:
            assert int(e["close_off"]) == int(e["fb_off"]) + int(e["fb_len"]), tag        # FEEDBACK before CLOSE
        total_ctrl += len(got["fb"]) + len(got["close"])
        mine = smsgs[int(e["first_msg"]):int(e["first_msg"]) + int(e["n_msgs"])]
        assert len(mine) == len(want_msgs[sid]), tag
        for m, (first, nfr, body) in zip(mine, want_msgs[sid]):
            src = data if int(m["flags"]) & 1 else out
            assert (int(m["stream_id"]), int(m["first_frame"]), int(m["n_frames"]), int(m["len"])) == (sid, first, nfr, len(body)), tag
            assert (int(m["flags"]) & 1) == (1 if nfr == 1 else 0), tag
            assert src[int(m["off"]):int(m["off"]) + int(m["len"])].tobytes() == body, tag
    assert len(smsgs) == sum(len(v) for v in want_msgs.values()), what
    assert len(run_ctrl) == len(rs)
    for r in range(len(rs)):
        off, ln = int(run_ctrl[r][0]), int(run_ctrl[r][1])
        assert ctrl[off:off + ln].tobytes() == want_rst[r], "%s run %d RST" % (what, r)
        total_ctrl += ln
    assert len(ctrl) == total_ctrl, what
    for sid in opened:
        q, w = ctx.stream_query(sid), orc.query(sid)
        assert (q["local_consumed"], q["remote_consumed"], q["pending_bytes"], bool(q["flags"] & 4), bool(q["flags"] & 8), q["error_code"]) == \
               (w["local_consumed"], w["remote_consumed"], w["pending_bytes"], w["closed"], w["handed_over"], w["error_code"]), "%s query %d" % (what, sid)


def traffic(rng, n_streams, n_socks, max_part, n_msgs):
    """-> (streams [(id, remote, sock, connected, need_feedback)], per-socket byte strings)"""
    ids = rng.sample(range(1, 1 << 40), n_streams + 8)
    streams = [(ids[i], rng.randrange(1, 1 << 50), rng.randrange(n_socks), rng.random() < 0.8, rng.random() < 0.7) for i in range(n_streams)]
    unknown = ids[n_streams:]
    queues = []                                   # per stream: its frames in order, each with the socket it travels on
    for sid, remote, sock, _, _ in streams:
        q = []
        for _ in range(rng.randrange(1, n_msgs + 1)):
            parts = rng.choice((1, 1, 1, 2, 3, 5))
            for p in range(parts):
                body = rng.randbytes(rng.choice((0, 1, 15, 16, 17, rng.randrange(max_part))))
                last = p == parts - 1
                q.append(F(sid, remote if rng.random() < 0.7 else -1, S.DATA, (False if rng.random() < 0.3 else None) if last else True, body))
            r = rng.random()
            if r < 0.25:
                q.append(S.feedback_frame(sid, remote, rng.randrange(1 << 20)))
            elif r < 0.30:
                q.append(F(sid, remote, rng.choice((0, S.DATA + 97))))       # FRAME_TYPE_UNKNOWN / an enum value proto2 does not know
            elif r < 0.36:
                q.append(F(sid, remote if rng.random() < 0.5 else -1, rng.choice((S.RST, S.CLOSE))))
        # a few streams travel on two sockets: their order is the order of msgs[]
        queues.append([(sock if rng.random() < 0.95 else rng.randrange(n_socks), f) for f in q])
    socks = [[] for _ in range(n_socks)]
    live = [q for q in queues if q]
    while live:
        q = rng.choice(live)
        sock, f = q.pop(0)
        socks[sock].append(f)
        if not q:
            live.remove(q)
        r = rng.random()
        if r < 0.15:
            socks[rng.randrange(n_socks)].append(echo_frame(rng, rng.randrange(200)))
        elif r < 0.22:
            u = rng.choice(unknown)
            socks[rng.randrange(n_socks)].append(rng.choice((F(u, 7, S.DATA, None, b"lost"), F(u, -1, S.DATA, None, b"lost"), S.feedback_frame(u, 9, 5), F(u, 11, S.CLOSE))))
    return streams, [b"".join(s) for s in socks]


@pytest.mark.parametrize("shape,mode", [("small", "copy"), ("big", "copy"), ("small", "pull"), ("big", "pull")])
def test_seeded_traffic_equals_the_oracle(shape, mode):
    import brpc_b200 as b2
    rng = random.Random(SEED + (1 if shape == "big" else 0) + (2 if mode == "pull" else 0))
    n_streams, n_socks, max_part, n_msgs = (24, 5, 400, 3) if shape == "small" else (320, 24, 6000, 4)
    streams, socks = traffic(rng, n_streams, n_socks, max_part, n_msgs)
    ctx = b2.Context(device=0, max_batch_bytes=16 << 20, max_msgs=1 << 15, max_runs=256)
    twin = b2.Context(device=0, max_batch_bytes=16 << 20, max_msgs=1 << 15, max_runs=256)
    ctx.stream_configure(512, 64 << 10)
    ctx.stream_open([(sid, remote, sock, (1 if conn else 0) | (2 if fb else 0)) for sid, remote, sock, conn, fb in streams])
    orc = S.StreamOracle(pending_bytes=64 << 10, out_bytes=16 << 20)
    for sid, remote, sock, conn, fb in streams:
        orc.open(sid, remote, sock, conn, fb)
    pin = None
    if mode == "pull":
        ctx.set_modes(b2.abi.INPUT_PULL, b2.abi.RESP_COPY)
        pin = b2.abi.PinnedBuffer(16 << 20)
    pos, step, n_batches, big_seen, small_seen = [0] * n_socks, 0, 5, False, False
    while any(pos[i] < len(socks[i]) for i in range(n_socks)):
        chunks = []
        for i in range(n_socks):
            left = len(socks[i]) - pos[i]
            take = left if step >= n_batches - 1 else min(left, rng.randrange(0, 2 * len(socks[i]) // (n_batches - 1) + 2))
            chunks.append(socks[i][pos[i]:pos[i] + take])
        data, runs = b2.make_runs(chunks)
        if pin is not None:
            pin.array[:len(data)] = data
            dev = ctx.process_batch_ptr(pin.ptr, len(data), runs)
        else:
            dev = ctx.process_batch(data, runs)
        assert_same(dev, twin.process_batch(data, runs)[:3], "%s batch %d: descriptors and replies of a context without a table" % (shape, step))
        check_batch(ctx, orc, data, dev, [s[0] for s in streams], "%s/%s batch %d" % (shape, mode, step))
        big_seen |= len(data) > (128 << 10); small_seen |= len(data) <= (128 << 10)
        for i in range(n_socks):
            pos[i] += int(dev[0]["consumed"][i])
        step += 1
        assert step < 40
    assert step >= 3 and (big_seen if shape == "big" else small_seen)
    # local close: the CLOSE frame of a connected stream the peer has not closed; afterwards the id is unknown
    for sid, remote, sock, conn, fb in streams[:6]:
        assert ctx.stream_close(sid) == orc.close(sid)
    data, runs = b2.make_runs([F(streams[0][0], 5, data=b"after close")])
    dev = ctx.process_batch(data, runs) if pin is None else (pin.array.__setitem__(slice(0, len(data)), data), ctx.process_batch_ptr(pin.ptr, len(data), runs))[1]
    check_batch(ctx, orc, data, dev, [s[0] for s in streams[6:]], "after close")


def test_hand_over_and_take_pending():
    import brpc_b200 as b2
    ctx = b2.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=16)
    ctx.stream_configure(8, 1024, 4096)
    orc = S.StreamOracle(pending_bytes=1024, out_bytes=4096)
    for sid in (1, 2, 3):
        ctx.stream_open([(sid, 100 + sid, 9, 3)]); orc.open(sid, 100 + sid, 9, True, True)
    a, b = bytes(range(200)) * 4, b"z" * 700
    batches = [[F(1, cont=True, data=a), F(2, data=b"whole"), F(3, cont=True, data=b"q" * 1000)],
               [F(1, cont=True, data=b), F(2, cont=True, data=b"p" * 3000), F(2, cont=True, data=b"p" * 3000), F(2, data=b"tail"), F(3, data=b"fits")],
               [F(1, 4, data=b"frames of a handed-over stream are described only"), F(2, 4, S.CLOSE), F(3, data=b"still served")]]
    for k, frames in enumerate(batches):
        data, runs = b2.make_runs([b"".join(frames)])
        dev = ctx.process_batch(data, runs)
        check_batch(ctx, orc, data, dev, (1, 2, 3), "hand-over batch %d" % k)
    assert ctx.stream_query(1)["flags"] & 8 and ctx.stream_query(2)["flags"] & 8
    assert ctx.stream_take_pending(1, 4096) == a and ctx.stream_take_pending(1, 4096) == b""     # handed out once
    assert ctx.stream_close(1) == O.pack_stream_frame(101, 1, S.CLOSE)
    with pytest.raises(b2.B2Error):
        ctx.ring_submit(np.zeros(64, np.uint8), b2.make_runs([b"x"])[1])


def test_set_connected_and_the_round_trip_between_two_contexts():
    """frames packed by b2_pack_requests on the writer are received by the reader; the reader's FEEDBACK bytes go back to the writer,
    whose remote_consumed then says what the reader consumed"""
    import brpc_b200 as b2
    writer = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 12, max_runs=16)
    reader = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 12, max_runs=16)
    writer.stream_configure(16, 4096); reader.stream_configure(16, 1 << 20)
    W, R = 0x1111, 0x2222                        # the writer's stream id and the reader's
    writer.stream_open([(W, R, 1, 3)])
    reader.stream_open([(R, 0, 2, 0)])           # a client-side stream whose settings have not arrived
    payload = np.frombuffer(random.Random(SEED).randbytes(200000), np.uint8)
    reqs, off = np.zeros(4, b2.abi.REQUEST_DT), 0
    for i, n in enumerate((65536, 65536, 65536, 200000 - 3 * 65536)):
        reqs[i]["kind"], reqs[i]["correlation_id"], reqs[i]["log_id"], reqs[i]["frame_type"] = 1, R, W, S.DATA
        reqs[i]["flags"] = 1 | (2 | 4 if i < 3 else 0)
        reqs[i]["payload_off"], reqs[i]["payload_len"] = off, n
        off += n
    frames = writer.pack_requests(payload, reqs)
    wire = b"".join(frames)
    cut = len(wire) // 2 + 13                    # the batches cut a frame in two
    data, runs = b2.make_runs([wire[:cut]])
    done = int(reader.process_batch(data, runs)[0]["consumed"][0])
    assert 0 < done < cut and reader.stream_query(R)["pending_bytes"] == 65536
    data, runs = b2.make_runs([wire[done:]])
    reader.process_batch(data, runs)
    smsgs, events, out, ctrl, _ = reader.stream_results()
    assert len(smsgs) == 1 and int(smsgs[0]["n_frames"]) == 4 and out[int(smsgs[0]["off"]):int(smsgs[0]["off"]) + 200000].tobytes() == payload.tobytes()
    assert int(events[0]["fb_len"]) == 0 and reader.stream_query(R)["local_consumed"] == 200000
    fb = reader.stream_set_connected(R, W, 2)     # SetConnected: the first FEEDBACK of a stream that consumed before
    assert fb == S.feedback_frame(W, R, 200000)
    data, runs = b2.make_runs([fb])
    writer.process_batch(data, runs)
    _, wev, _, _, _ = writer.stream_results()
    assert int(wev[0]["flags"]) == S.EV_MOVED and writer.stream_query(W)["remote_consumed"] == 200000


def test_bad_meta_connect_mid_traffic_and_slot_reuse():
    """a frame whose StreamFrameMeta does not parse is dropped; a stream opened unconnected writes no FEEDBACK until SetConnected, then
    the first one; ids closed and opened again (and new ids that land on the freed table slots) resolve to the new streams"""
    import brpc_b200 as b2
    ctx = b2.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=16)
    ctx.stream_configure(4, 4096)                 # a table of 16 slots: 4 open ids out of 40 collide and reuse tombstones
    orc = S.StreamOracle(pending_bytes=4096, out_bytes=1 << 20)
    bad = b"STRM" + (5).to_bytes(4, "big") + (2).to_bytes(4, "big") + b"\x08\xff" + b"abc"      # stream_id's varint runs off the meta
    ctx.stream_open([(1, 0, 7, 0)]); orc.open(1, 0, 7, False, False)
    opened = [1]

    def step(frames, what):
        data, runs = b2.make_runs([b"".join(frames)])
        dev = ctx.process_batch(data, runs)
        check_batch(ctx, orc, data, dev, opened, what)
        return dev
    dev = step([F(1, 9, data=b"before the settings"), bad, F(1, 9, cont=True, data=b"half")], "unconnected")
    assert list(dev[1]["status"]) == [4, 5, 4]
    assert ctx.stream_set_connected(1, 9, 2) == orc.set_connected(1, 9, True) != b""
    step([F(1, 9, data=b" and half"), bad], "connected")
    rng = random.Random(SEED)
    for rnd in range(10):
        for sid in opened:
            assert ctx.stream_close(sid) == orc.close(sid)
        old, opened = opened, rng.sample(range(1, 41), 4)
        ctx.stream_open([(sid, 100 + sid, rnd, 3) for sid in opened])
        for sid in opened:
            orc.open(sid, 100 + sid, rnd, True, True)
        frames = [F(sid, 5, cont=(True if rng.random() < 0.5 else None), data=rng.randbytes(rng.randrange(40))) for sid in opened + old + list(range(41, 44))]
        rng.shuffle(frames)
        step(frames, "reuse round %d" % rnd)
    with pytest.raises(b2.B2Error):
        ctx.stream_open([(99, 0, 0, 0)])          # full
