"""GPU: a gRPC server's turn on the latency path (b2_h2_ring_turn_*: k_h2_ring serves the runs, then packs the replies the host produced)
against a twin context that runs b2_h2_serve_batch + b2_h2_pack_responses on the same bytes with the same caps — run statuses, messages,
the defined bytes of out, spans, device replies and every host reply's frames, turn by turn, and at the end one more serve and one more
pack on both contexts, so that the connection state the turns leave (HPACK tables, windows, deferred WINDOW_UPDATEs, the stream pool) is
shown equal too:
  - mixed traffic whose calls to host methods and unknown paths are answered in the next turn, one turn at a time and eight in flight;
  - replies for connections without a run in the turn, and reply-only turns;
  - a SETTINGS (max_frame_size, header_table_size 0) or WINDOW_UPDATE in the runs that governs the same turn's replies, and a connection
    window too small for a reply (RST_STREAM(FLOW_CONTROL_ERROR));
  - a body over several DATA frames with the longest content-type and grpc-message; gunzip connections; pinned and staged bytes;
  - idle retirement and relaunch, no launch over 100 steady turns that carry host replies; every refusal; b2_h2_ring_submit on a
    turn-enabled context equal to a plain one;
  - a live grpcio client: 1 000 calls over 8 connections to the device echo method and a host-answered method."""
import random
import time

import numpy as np
import pytest

import _h2serve as S
import _h2traffic as T
from test_gpu_h2_ring import MAX_BYTES, _err, _same, _snap
from test_gpu_h2_serve import IDENTITY, METHODS, REGION, RREGION, WINDOW, _ctx, call, conn_stream, gz, host_records, mixed_calls, prefix

pytestmark = pytest.mark.gpu
F_BODY_IN_INPUT, F_GUNZIPPED = 16, 64
HOST = b"/example.EchoService/Host"
CT = b"application/grpc"


def turn_bytes(chunks, items):
    """a turn's bytes and lists: chunks [(conn, bytes)] as 16-byte aligned runs, then the fields of the host replies items
    [(conn, stream_id, content-type, body, grpc-status, grpc-message)], which the records index in the same buffer"""
    import brpc_b200
    from brpc_b200.abi import RUN_DT
    if chunks:
        data, runs = brpc_b200.make_runs([b for _, b in chunks])
        runs["socket_id"] = [k for k, _ in chunks]
    else:
        data, runs = np.zeros(16, np.uint8), np.zeros(0, RUN_DT)
    blob, resps = host_records(items)
    for f in ("content_type_off", "body_off", "grpc_message_off"):
        resps[f] += len(data)
    return np.concatenate([data, blob]), runs, resps


class TurnPair:
    """a turn-enabled ring context and a twin running b2_h2_serve_batch + b2_h2_pack_responses with the same caps"""
    def __init__(self, n, gunzip=(), max_resps=512, resp_out_cap=8 << 20):
        self.n = n
        self.msg_cap, self.out_cap, self.replies_cap, self.resp_out_cap = n * 128, n * REGION, n * RREGION, resp_out_cap
        self.ring, self.twin = _ctx(), _ctx()
        for k in range(n):
            for c in (self.ring, self.twin):
                c.h2_conn_reset(k)
                if k in gunzip:
                    c.h2_conn_set_gunzip(k)
        self.ring.h2_ring_turn_enable(MAX_BYTES, self.msg_cap, self.out_cap, self.replies_cap, max_resps, resp_out_cap)

    def region(self, n_runs):
        return (self.out_cap // n_runs) & ~63

    def twin_turn(self, chunks, items=()):
        """the turn on the twin: (data, runs, resps, served or None, frames)"""
        data, runs, resps = turn_bytes(chunks, items)
        want = None
        if len(runs):
            want = _snap(self.twin.h2_serve_batch(data, runs, msg_cap=self.msg_cap, out_cap=self.out_cap, replies_cap=self.replies_cap))
        frames = self.twin.h2_pack_responses(data, resps, out_cap=self.resp_out_cap) if len(resps) else []
        return data, runs, resps, want, frames

    def check(self, got, turn, what=""):
        _, runs, _, want, frames = turn
        status, served, got_frames = got
        assert status == 0, what
        if want is None:
            assert len(served[0]) == 0 and len(served[1]) == 0, what
        else:
            _same(served, want, len(runs), self.region(len(runs)), what)
        assert got_frames == frames, what

    def step(self, chunks, items=(), what="", pinned=None):
        """one turn, waited at once; pinned: a PinnedBuffer the bytes are copied into and pulled from in place"""
        turn = self.twin_turn(chunks, items)
        data, runs, resps = turn[:3]
        if pinned is not None:
            pinned.array[:len(data)] = data
            self.last = self.ring.h2_ring_turn_submit(None, runs, resps, ptr=pinned.ptr, nbytes=len(data))
        else:
            self.last = self.ring.h2_ring_turn_submit(data, runs, resps)
        self.check(self.ring.h2_ring_turn_wait(self.last), turn, what)
        return turn

    def many(self, turns, depth):
        """turns the twin ran in order, submitted `depth` at a time, each group waited last to first"""
        for i in range(0, len(turns), depth):
            group = turns[i:i + depth]
            tickets = [self.ring.h2_ring_turn_submit(d, r, q) for d, r, q, _, _ in group]
            for turn, t in reversed(list(zip(group, tickets))):
                self.check(self.ring.h2_ring_turn_wait(t), turn, "ticket %d" % t)

    def finish(self, chunks, items):
        """one more serve and one more pack on both contexts: the state the turns left is equal"""
        data, runs, resps = turn_bytes(chunks, items)
        caps = dict(msg_cap=self.msg_cap, out_cap=self.out_cap, replies_cap=self.replies_cap)
        got, want = _snap(self.ring.h2_serve_batch(data, runs, **caps)), _snap(self.twin.h2_serve_batch(data, runs, **caps))
        _same(got, want, len(runs), self.region(len(runs)), "serve after the turns")
        assert self.ring.h2_pack_responses(data, resps) == self.twin.h2_pack_responses(data, resps)


def host_items(turn):
    """the host's replies to the calls a turn left: a Host call gets its message back (grpc-status 0), every other one UNIMPLEMENTED"""
    data, runs, _, want, _ = turn
    if want is None:
        return []
    rs, msgs, out = want[0], want[1], want[2]
    conns = np.repeat(runs["socket_id"], rs["n_msgs"])
    items = []
    for m, k in zip(msgs, conns):
        f = int(m["flags"])
        if f & S.F_ANSWERED:
            continue
        if int(m["method_idx"]) == 1:
            src = data if (f & F_BODY_IN_INPUT) and not (f & F_GUNZIPPED) else out
            items.append((int(k), int(m["stream_id"]), CT, bytes(src[int(m["msg_off"]):int(m["msg_off"]) + int(m["msg_len"])]), 0, b""))
        else:
            items.append((int(k), int(m["stream_id"]), CT, b"", 12, b"unimplemented"))
    return items


def _turns(pair, streams, parts):
    """the streams cut into `parts` turns as the twin consumes them, each carrying the host replies to the calls the one before left,
    then a reply-only turn for the last ones: [turn]"""
    n = len(streams); rest = [b""] * n; out = []; items = []
    for part in range(parts):
        now = [rest[k] + streams[k][len(streams[k]) * part // parts:len(streams[k]) * (part + 1) // parts] for k in range(n)]
        turn = pair.twin_turn(list(enumerate(now)), items)
        out.append(turn)
        rest = [now[k][int(turn[3][0][k]["consumed"]):] for k in range(n)]
        items = host_items(turn)
    assert not any(rest)
    if items:
        out.append(pair.twin_turn([], items))
    return out


def _calls(enc, sid, k, m, msg, path=b"/example.EchoService/Echo"):
    out = b""
    for _ in range(m):
        out += call(enc[k], sid[k], prefix(msg), path=path); sid[k] += 2
    return out


@pytest.mark.parametrize("depth", [1, 8])
def test_mixed_turns_equal_the_two_batch_calls(depth):
    rng = random.Random(20261018 + depth)
    n = 8
    pair = TurnPair(n, gunzip=set(range(0, n, 2)))
    streams = [conn_stream(rng, k, mixed_calls(rng, k)) for k in range(n)]
    turns = _turns(pair, streams, 8)
    pair.many(turns, depth)
    assert sum(len(t[2]) for t in turns) >= 6 * n and sum(1 for t in turns if len(t[2]) and len(t[1])) >= 6
    pair.finish([(k, T.frame(6, 0, 0, b"\0" * 8)) for k in range(n)], [(k, 99, CT, b"late", 0, b"") for k in range(n)])   # a PING per connection


def test_replies_for_connections_without_a_run_and_reply_only_turns():
    n = 4
    pair = TurnPair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    sid = [1] * n
    msg = S.echo_request(b"turn " * 200)
    t = pair.step([(k, T.PREFACE + T.settings() + WINDOW + _calls(enc, sid, k, 2, msg, HOST) + _calls(enc, sid, k, 1, msg)) for k in range(n)],
                  what="open")
    left = host_items(t)
    assert len(left) == 2 * n
    # runs on 0 and 1 only, replies on 2 and 3 only
    t = pair.step([(k, _calls(enc, sid, k, 1, msg, HOST) + _calls(enc, sid, k, 1, msg)) for k in (0, 1)], [i for i in left if i[0] >= 2],
                  what="replies without runs")
    left = [i for i in left if i[0] < 2] + host_items(t)
    pair.step([], sorted(left), what="reply-only")
    pair.step([], [(3, 999, CT, b"x" * 5000, 0, b"")], what="reply-only, one connection")
    pair.step([(2, _calls(enc, sid, 2, 2, msg))], what="runs only")
    pair.finish([(k, _calls(enc, sid, k, 1, msg)) for k in range(n)], [(k, 777, CT, b"y" * 300, 0, b"") for k in range(n)])


def test_settings_and_window_updates_in_the_runs_govern_the_same_turns_replies():
    n = 4
    pair = TurnPair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    sid = [1] * n
    msg = S.echo_request(b"s" * 100)
    big = bytes(random.Random(1).randrange(256) for _ in range(70000))
    # 0: max_frame_size 64 KiB, then back to 16 KiB in the reply's turn; 1: header_table_size 0 in the reply's turn;
    # 2: the default 65 535-byte connection window; 3: the same, widened by a WINDOW_UPDATE in the reply's turn
    opens = [T.settings([(5, 65536)]) + WINDOW, WINDOW, b"", b""]
    t = pair.step([(k, T.PREFACE + T.settings() + opens[k] + _calls(enc, sid, k, 1, msg, HOST)) for k in range(n)], what="open")
    left = host_items(t)
    assert len(left) == n
    items = [(k, s, CT, big, 0, b"") for k, s, _, _, _, _ in left] + [(1, 1001, b"application/grpc+proto", b"ab", 0, b"")]
    items.sort(key=lambda i: i[0])
    runs = [(0, T.settings([(5, 16384)])), (1, T.settings([(1, 0)])), (3, T.frame(8, 0, 0, (1 << 20).to_bytes(4, "big")))]
    t = pair.step(runs, items, what="governed by the same turn")
    frames = t[4]
    heads = lambda b: [(int.from_bytes(b[p:p + 3], "big"), b[p + 3]) for p in _frame_starts(b)]
    assert max(ln for ln, ty in heads(frames[0]) if ty == 0) == 16384
    assert heads(frames[3]) == [(4, 3)] and frames[3][9:13] == (3).to_bytes(4, "big")      # RST_STREAM(FLOW_CONTROL_ERROR)
    assert any(ty == 0 for _, ty in heads(frames[4]))                                      # the widened window covers it
    pair.step([], [(2, 2001, CT, b"z" * 1000, 0, b"")], what="after the RST")
    pair.finish([(k, _calls(enc, sid, k, 1, msg)) for k in range(n)], [(k, 3001, CT, b"w" * 100, 0, b"") for k in range(n)])


def _frame_starts(b):
    p = 0
    while p + 9 <= len(b):
        yield p
        p += 9 + int.from_bytes(b[p:p + 3], "big")


def test_a_body_over_several_data_frames_and_the_longest_fields():
    n = 2
    pair = TurnPair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    sid = [1] * n
    rng = random.Random(7)
    body = bytes(rng.randrange(256) for _ in range(100000))
    ct = b"application/grpc+proto;" + b"p" * (256 - 23)
    gm = bytes(rng.randrange(32, 127) for _ in range(512))
    pair.step([(k, T.PREFACE + T.settings() + WINDOW) for k in range(n)], what="open")
    items = [(0, 101, ct, body, 2, gm), (0, 103, CT, body[:40000], 0, b""), (1, 101, ct, b"", 13, gm), (1, 103, ct, body[:16379], 0, gm[:1])]
    for _ in range(2):                                                # the second time the encoder tables hold these headers
        t = pair.step([(k, _calls(enc, sid, k, 1, S.echo_request(b"e" * 50))) for k in range(n)], items, what="long")
        items = [(k, s + 100, c, b, st, m) for k, s, c, b, st, m in items]
    assert sum(1 for _, ty in [(0, b[p + 3]) for b in t[4][:1] for p in _frame_starts(b)] if ty == 0) >= 7
    pair.finish([(k, _calls(enc, sid, k, 1, S.echo_request(b"f"))) for k in range(n)], items)


def test_gunzip_connections():
    rng = random.Random(3)
    n = 4
    pair = TurnPair(n, gunzip=set(range(n)))
    msgs = [S.echo_request(bytes(rng.randrange(97, 100) for _ in range(2000 + 500 * i))) for i in range(6)]
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    ge = ((b"grpc-encoding", b"gzip"),)
    streams = [T.PREFACE + T.settings() + WINDOW + b"".join(call(enc[k], 1 + 2 * i, prefix(gz(m), 1), extra=ge, path=HOST if i % 2 else
                                                                 b"/example.EchoService/Echo") for i, m in enumerate(msgs)) for k in range(n)]
    turns = _turns(pair, streams, 3)
    pair.many(turns, 3)
    assert sum(int(np.count_nonzero(t[3][1]["flags"] & F_GUNZIPPED)) for t in turns if t[3] is not None) == n * len(msgs)
    assert sum(len(t[2]) for t in turns) == n * len(msgs) // 2


def test_pinned_and_staged_bytes():
    from brpc_b200.abi import PinnedBuffer
    n = 4
    pair = TurnPair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    sid = [1] * n
    msg = S.echo_request(b"pin " * 300)
    buf = PinnedBuffer(1 << 20)
    try:
        t = pair.step([(k, T.PREFACE + T.settings() + WINDOW + _calls(enc, sid, k, 2, msg, HOST)) for k in range(n)], what="open", pinned=buf)
        for i in range(6):
            t = pair.step([(k, _calls(enc, sid, k, 1, msg, HOST) + _calls(enc, sid, k, 1, msg)) for k in range(n)], host_items(t),
                          what="turn %d" % i, pinned=buf if i % 2 else None)
        pair.step([], host_items(t), what="reply-only, pinned", pinned=buf)
    finally:
        pair.ring.ring_stop()
        buf.free()


def _steady(pair, enc, sid, steps, msg, items):
    for _ in range(steps):
        t = pair.step([(k, _calls(enc, sid, k, 1, msg, HOST) + _calls(enc, sid, k, 1, msg)) for k in range(pair.n)], items)
        items = host_items(t)
    return items


def test_idle_retirement_relaunch_and_no_launch_over_100_steady_turns_with_host_replies(monkeypatch):
    monkeypatch.setenv("B2_RING_IDLE_MS", "2000")
    n = 4
    pair = TurnPair(n)
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    sid = [1] * n
    msg = S.echo_request(b"steady" * 100)
    t = pair.step([(k, T.PREFACE + T.settings() + WINDOW) for k in range(n)])
    items = _steady(pair, enc, sid, 1, msg, [])
    n0 = pair.ring.ring_launches()
    items = _steady(pair, enc, sid, 100, msg, items)
    assert pair.ring.ring_launches() == n0
    pair.ring.ring_stop()
    monkeypatch.setenv("B2_RING_IDLE_MS", "5")
    items = _steady(pair, enc, sid, 1, msg, items)                  # relaunched by the submission, now with a 5 ms idle time
    n1 = pair.ring.ring_launches()
    assert n1 == n0 + 1
    time.sleep(0.2)                                                  # it retires and comes back with the next turn, the state intact
    items = _steady(pair, enc, sid, 2, msg, items)
    assert pair.ring.ring_launches() > n1
    ph = pair.ring.ring_phase_ns(pair.last)
    assert 0 < ph[0] <= ph[1] <= ph[2] <= ph[3]
    pair.step([], items, what="reply-only after the relaunch")
    pair.finish([(k, _calls(enc, sid, k, 1, msg)) for k in range(n)], [(k, 9999, CT, b"e", 0, b"") for k in range(n)])


def test_refusals():
    import brpc_b200
    from brpc_b200.abi import B2_E_CAPACITY, B2_E_INVAL, H2_RESPONSE_DT, RUN_DT
    n = 2
    pair = TurnPair(n, max_resps=4, resp_out_cap=1 << 16)
    ring = pair.ring
    enc = [T.HpackEncoder(random.Random(k)) for k in range(n)]
    sid = [1] * n
    msg = S.echo_request(b"r" * 100)
    pair.step([(k, T.PREFACE + T.settings() + WINDOW + _calls(enc, sid, k, 1, msg)) for k in range(n)], what="open")
    no_runs = np.zeros(0, RUN_DT)

    def refused(items, patch=None):
        data, _, resps = turn_bytes([], items)
        if patch:
            patch(resps)
        return _err(ring.h2_ring_turn_submit, data, no_runs, resps)

    one = [(0, 11, CT, b"abc", 0, b"")]
    for flag in (2, 4, 8):                                          # B2_H2_RESP_BODY_IN_INPUT, _BODY_IN_OUT, _CT_IN_OUT
        assert refused(one, lambda r: r.__setitem__("flags", 1 | flag)) == B2_E_INVAL, flag
    assert refused([(0, 11, CT, b"", 0, b""), (1, 13, CT, b"", 0, b""), (0, 15, CT, b"", 0, b"")]) == B2_E_INVAL   # not adjacent
    assert refused([(32, 11, CT, b"", 0, b"")]) == B2_E_INVAL                                                        # connection out of range
    assert refused([(0, 11, b"c" * 257, b"", 0, b"")]) == B2_E_INVAL                                                 # content-type > 256
    assert refused([(0, 11, CT, b"", 2, b"m" * 513)]) == B2_E_INVAL                                                  # grpc-message > 512
    assert refused(one, lambda r: r.__setitem__("body_off", 1 << 20)) == B2_E_INVAL                                  # outside the bytes
    assert refused([(0, 11 + 2 * i, CT, b"", 0, b"") for i in range(5)]) == B2_E_CAPACITY                            # > max_resps
    assert refused([(0, 11, CT, b"b" * 40000, 0, b""), (0, 13, CT, b"b" * 40000, 0, b"")]) == B2_E_CAPACITY            # > resp_out_cap
    assert _err(ring.h2_ring_turn_submit, np.zeros(16, np.uint8), no_runs, np.zeros(0, H2_RESPONSE_DT)) == B2_E_INVAL   # an empty turn
    bad = brpc_b200.make_runs([b"\0" * 16])[1]; bad["socket_id"] = 0
    bad = np.concatenate([bad, bad])
    assert _err(ring.h2_ring_turn_submit, np.zeros(32, np.uint8), bad, np.zeros(0, H2_RESPONSE_DT)) == B2_E_INVAL       # the runs' checks
    # while a turn is outstanding the batch calls are refused; the refused submissions above changed nothing
    t = pair.twin_turn([(k, _calls(enc, sid, k, 1, msg, HOST)) for k in range(n)], [(1, 11, CT, b"abc", 0, b"")])
    ticket = ring.h2_ring_turn_submit(*t[:3])
    assert _err(ring.h2_pack_responses, np.zeros(64, np.uint8), np.zeros(1, H2_RESPONSE_DT)) == B2_E_INVAL
    assert _err(ring.h2_serve_batch, *brpc_b200.make_runs([b"\0" * 16])) == B2_E_INVAL
    pair.check(ring.h2_ring_turn_wait(ticket), t, "the outstanding turn")
    pair.step([], host_items(t), what="after the refusals")
    # the enable rules
    c = _ctx()
    assert _err(c.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, 0, 1 << 16) == B2_E_INVAL
    assert _err(c.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, 64, 0) == B2_E_INVAL
    assert _err(c.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, (1 << 15) + 1, 1 << 16) == B2_E_CAPACITY     # max_msgs
    assert _err(c.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, 64, (64 << 20) + 1) == B2_E_CAPACITY         # max_resp_bytes
    assert _err(c.h2_ring_turn_enable, 1 << 20, 64, (128 << 20) + 1, 1 << 20, 64, 1 << 16) == B2_E_CAPACITY        # b2_h2_ring_enable's
    c.h2_ring_turn_enable(1 << 20, 64, 1 << 20, 1 << 20, 64, 1 << 16)
    assert _err(c.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, 64, 1 << 16) == B2_E_INVAL                    # twice
    assert _err(c.h2_ring_enable, 1 << 20, 64, 1 << 20, 1 << 20) == B2_E_INVAL
    assert _err(c.h2_ring_turn_wait, 1) == B2_E_INVAL                                                               # no such ticket
    a = _ctx(); a.ring_start()
    assert _err(a.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, 64, 1 << 16) == B2_E_INVAL                    # after a ring call
    a.ring_stop()
    b = _ctx(); b.h2_client_ring_enable(1 << 20, 64, 1 << 20, 16, 1 << 16)
    assert _err(b.h2_ring_turn_enable, 1 << 20, 64, 1 << 20, 1 << 20, 64, 1 << 16) == B2_E_INVAL                    # another ring kind
    p = _ctx(); p.h2_ring_enable(1 << 20, 64, 1 << 20, 1 << 20)
    data, _, resps = turn_bytes([], one)
    assert _err(p.h2_ring_turn_submit, data, no_runs, resps) == B2_E_INVAL                                          # a plain h2 ring
    assert _err(p.h2_ring_turn_wait, 1) == B2_E_INVAL
    for x in (c, a, b, p):
        x.close()


def test_plain_tickets_on_a_turn_enabled_context_equal_a_plain_context():
    import brpc_b200
    n = 4
    rng = random.Random(11)
    plain, turns = _ctx(), _ctx()
    for c in (plain, turns):
        for k in range(n):
            c.h2_conn_reset(k)
    caps = (MAX_BYTES, n * 128, n * REGION, n * RREGION)
    plain.h2_ring_enable(*caps)
    turns.h2_ring_turn_enable(*caps, 64, 1 << 20)
    streams = [conn_stream(rng, k, mixed_calls(rng, k)) for k in range(n)]
    rest = [b""] * n
    for part in range(4):
        now = [rest[k] + streams[k][len(streams[k]) * part // 4:len(streams[k]) * (part + 1) // 4] for k in range(n)]
        data, runs = brpc_b200.make_runs(now)
        runs["socket_id"] = np.arange(n)
        want = _snap(plain.h2_ring_wait(plain.h2_ring_submit(data, runs)))
        _same(turns.h2_ring_wait(turns.h2_ring_submit(data, runs)), want, n, (n * REGION // n) & ~63, "part %d" % part)
        rest = [now[k][int(want[0][k]["consumed"]):] for k in range(n)]
    assert not any(rest)
    for c in (plain, turns):
        c.close()


class TurnServeEngine(S.DeviceServeEngine):
    """DeviceServeEngine on ring turns: one turn per feed, then the calls it left answered by a reply-only turn — Host calls with their
    message back, every other one UNIMPLEMENTED"""
    def __init__(self, ctx):
        super().__init__(ctx)
        ctx.h2_ring_turn_enable(1 << 20, 1024, 8 << 20, 8 << 20, 1024, 8 << 20)
        self.n_host = 0

    def feed(self, cid, buf):
        from brpc_b200.abi import H2_RESPONSE_DT
        with self.lock:
            data, runs, _ = turn_bytes([(cid, buf)], [])
            st, served, _ = self.ctx.h2_ring_turn_wait(self.ctx.h2_ring_turn_submit(data, runs, np.zeros(0, H2_RESPONSE_DT)))
            assert st == 0
            rs, msgs, out, replies, spans = served
            co, cl, so, sl = int(rs["ctrl_off"][0]), int(rs["ctrl_len"][0]), int(spans["off"][0]), int(spans["len"][0])
            reply = bytes(out[co:co + cl]) + bytes(replies[so:so + sl])
            self.n_answered += int(spans["n_answered"][0])
            items = host_items((data, runs, None, _snap(served), None))
            if items:
                self.n_host += sum(1 for i in items if i[4] == 0)
                d, r, q = turn_bytes([], items)
                st, _, frames = self.ctx.h2_ring_turn_wait(self.ctx.h2_ring_turn_submit(d, r, q))
                reply += b"".join(frames)
            return int(rs["consumed"][0]), reply, int(rs["parse_error"][0]), len(msgs)


def _grpcio_two_methods(port, requests, channels):
    """request i as a call to Echo (even i) or Host (odd i), round-robin over `channels` connections: (code name, details, reply) per call"""
    import threading
    import grpc
    opts = [("grpc.max_receive_message_length", 1 << 24), ("grpc.max_send_message_length", 1 << 24), ("grpc.use_local_subchannel_pool", 1)]
    chans = [grpc.insecure_channel("127.0.0.1:%d" % port, options=opts) for _ in range(channels)]
    try:
        calls = [[ch.unary_unary(p, request_serializer=lambda b: b, response_deserializer=lambda b: b) for p in ("/example.EchoService/Echo", HOST.decode())]
                 for ch in chans]
        gate = threading.BoundedSemaphore(64); futs = []
        for i, b in enumerate(requests):
            gate.acquire()
            f = calls[i % channels][(i // channels) % 2].future(b, timeout=120)
            f.add_done_callback(lambda _f: gate.release())
            futs.append(f)
        out = []
        for f in futs:
            try:
                out.append(("OK", "", f.result()))
            except grpc.RpcError as e:
                out.append((e.code().name, e.details(), None))
        return out
    finally:
        for ch in chans:
            ch.close()


def test_live_grpcio_client_1000_calls_over_8_connections_device_and_host_methods():
    pytest.importorskip("grpc")
    from _h2loop import H2LoopServer
    eng = TurnServeEngine(_ctx(METHODS, IDENTITY, 16, 128))
    srv = H2LoopServer(eng)
    reqs = S.mutation_corpus(1000, seed=18)
    try:
        got = _grpcio_two_methods(srv.port, reqs, 8)
    finally:
        srv.close()
    assert not srv.errors, srv.errors
    want = [S.expected_call(r, IDENTITY) if (i // 8) % 2 == 0 else ("OK", "", r) for i, r in enumerate(reqs)]
    assert got == want
    n_echo = sum(1 for i in range(len(reqs)) if (i // 8) % 2 == 0)
    assert eng.n_answered == n_echo and eng.n_host == len(reqs) - n_echo
