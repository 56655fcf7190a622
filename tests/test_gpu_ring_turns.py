"""GPU: baidu_std server turns on the latency path (b2_ring_turn_*).  A ticket is one server turn: the bytes read from server sockets are
served as b2_process_batch serves them, then the replies user code produced for B2_HANDLER_HOST methods are packed as b2_pack_responses
packs them, inside the resident k_ring<RingBody::replies>.  Every turn is compared with a twin context running those two batch calls, and
with the oracle's process_batch and pack_response."""
import ctypes as C
import gc
import random
import time

import numpy as np
import pytest

import _oracle as O
from _compare import MSG_FIELDS, RUN_FIELDS, assert_same
from _replies import ReplyBatch
from _traffic import echo_frame, mixed_frames, rnd62

pytestmark = pytest.mark.gpu
SEED = 20261019
MAX_BYTES, MAX_RESPS, RESP_OUT, MAX_REQS_CLIENT = 1 << 20, 256, 2 << 20, 256
METHODS = (O.ECHO_METHOD, dict(O.ECHO_METHOD, method_name=b"Host", handler=0))      # a device echo method and a B2_HANDLER_HOST method
CFG = O.make_config(METHODS)
OFF_FIELDS = ("error_text_off", "body_off", "attachment_off", "checksum_value_off", "extra_streams_off", "user_fields_off")
SHAPES = ("ok", "ok", "snappy", "crc", "snappy_crc", "attachment", "error", "error-1", "error_text", "stream", "user_fields", "gzip")


def _ctx():
    import brpc_b200
    return brpc_b200.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 14, max_runs=512, max_resp_bytes=8 << 20, methods=METHODS)


def _err(fn, *a, **kw):
    from brpc_b200.abi import B2Error
    try:
        fn(*a, **kw)
    except B2Error as e:
        return e.code
    return 0


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7f) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


def host_replies(rng, cids, shape=None, size=None):
    """what user code answers to host-method calls: one reply per correlation id, of every shape SendRpcResponse writes"""
    rb = ReplyBatch()
    for cid in cids:
        s = shape or rng.choice(SHAPES)
        n = size if size is not None else rng.choice([0, 1, 30, 200, 1000, 5000])
        body = rng.choice([rnd62(rng, n), b"r" * n])
        kw = dict(correlation_id=int(cid), body=b"\x0a" + _varint(len(body)) + body)
        if s in ("snappy", "snappy_crc"):
            kw["compress_type"] = 1
        if s in ("crc", "snappy_crc"):
            kw["checksum_type"] = 1
        if s == "attachment":
            kw["attachment"] = rnd62(rng, rng.choice([1, 33, 4000]))
        if s.startswith("error"):
            kw["error_code"] = -1 if s == "error-1" else rng.choice([1003, 2002])
            kw["error_text"] = rnd62(rng, rng.choice([3, 90])) if s == "error_text" else b""
            kw["request_checksum"] = rnd62(rng, rng.choice([0, 4]))
        if s == "stream":
            kw["stream"] = dict(stream_id=rng.getrandbits(62), need_feedback=rng.random() < 0.5, writable=rng.random() < 0.5,
                                extra=[rng.getrandbits(rng.choice([3, 30, 62])) for _ in range(rng.choice([0, 1, 5]))])
        if s == "user_fields":
            kw["user_fields"] = [(rnd62(rng, rng.choice([1, 9])), rnd62(rng, rng.choice([0, 40, 300]))) for _ in range(rng.choice([1, 3]))]
        if s == "gzip":
            kw["compress_type"] = 2                      # not packed: length 0, as from b2_pack_responses
        rb.add(**kw)
    return rb


def turn(chunks, rb=None, client=False):
    """the bytes of one turn: the runs (chunks, 16-aligned), then the replies' buffer, the records' offsets moved behind the runs"""
    from brpc_b200.abi import REPLY_DT, RUN_DT
    blob, runs = bytearray(), []
    for k, c in chunks:
        off = len(blob); blob += c; blob += b"\0" * (-len(blob) % 16)
        runs.append((k, off, len(c), -1, 1 if client else 0))
    recs = np.zeros(0, REPLY_DT)
    if rb is not None and rb.recs:
        base = len(blob); blob += rb.buf
        recs = np.array(rb.recs, REPLY_DT)
        for f in OFF_FIELDS:
            recs[f] += base
    blob += b"\0" * 16
    return np.frombuffer(bytes(blob), np.uint8), np.array(runs, RUN_DT), recs


def _copy(res):
    rs, msgs, resp = res[:3]
    return rs.copy(), msgs.copy(), resp.copy()


class Pair:
    """a context serving server turns on the ring, and its twin running the two batch calls"""

    def __init__(self, max_bytes=MAX_BYTES, max_resps=MAX_RESPS, resp_out=RESP_OUT):
        self.ring, self.twin = _ctx(), _ctx()
        self.ring.ring_turn_enable(max_bytes, max_resps, resp_out)
        self.resp_out = resp_out
        self.last = 0

    def twin_turn(self, data, runs, recs):
        batch = _copy(self.twin.process_batch(data, runs)) if len(runs) else None
        frames = self.twin.pack_responses(data, recs, out_cap=self.resp_out) if len(recs) else []
        return batch, frames

    def check(self, got, data, runs, recs, want, what=""):
        batch, frames = want
        if batch is None:
            assert len(got[0]) == 0 and len(got[1]) == 0, what
        else:
            assert_same(got, batch, "%s: ring vs twin" % (what,))
            assert_same(got, O.process_batch(CFG, data, runs), "%s: ring vs oracle" % (what,))
        assert len(got[4]) == len(recs) == len(frames), what
        for i, (g, f) in enumerate(zip(got[4], frames)):
            assert g == f, (what, i, "ring vs twin")
            assert g == O.pack_response(recs[i], data), (what, i, "ring vs oracle")

    def turn(self, data, runs, recs, what="", **kw):
        want = self.twin_turn(data, runs, recs)
        t = self.ring.ring_turn_submit(data, runs, recs, **kw)
        assert t == self.last + 1, (t, self.last)
        self.last = t
        got = self.ring.ring_turn_wait(t)
        self.check(got, data, runs, recs, want, what)
        return got

    def step(self, chunks, rb=None, what=""):
        return self.turn(*turn(chunks, rb), what)

    def close(self):
        self.ring.close(); self.twin.close()


def _requests(rng, n_socks, per_sock, host_share=0.4):
    """per socket the frames of per_sock requests: mixed traffic (every ProcessRpcRequest branch) and calls to the host method"""
    out = []
    for k in range(n_socks):
        frames = mixed_frames(rng, per_sock)
        for j in range(len(frames)):
            if rng.random() < host_share:
                frames[j] = echo_frame(rng, k * 1000 + j, rnd62(rng, rng.choice([0, 10, 300])), method=b"Host")
        out.append(b"".join(frames))
    return out


@pytest.mark.parametrize("depth", [1, 8])
def test_seeded_traffic_across_turns(depth):
    """mixed requests split at random offsets across turns (each turn carries the unconsumed tail, as `consumed` says); the host answers
    the previous turn's host-method calls in the next one, with every reply shape; up to `depth` turns in flight, waited out of order"""
    rng = random.Random(SEED + depth)
    n_socks = 16
    streams = _requests(rng, n_socks, 10)
    pair = Pair()
    pos, tail, pending = [0] * n_socks, [b""] * n_socks, []
    turns = []
    while any(pos[k] < len(streams[k]) for k in range(n_socks)) or pending or len(turns) < 6:
        chunks, budget = [], 96 << 10                          # (the runs stay inside the compact block: no overflow among turns in flight)
        for k in range(n_socks):
            if rng.random() < 0.3 and pos[k] < len(streams[k]) or budget < len(tail[k]) + 6000:
                continue
            take = rng.choice([0, 5, 12, 100, 700, 2000, 6000])
            new = streams[k][pos[k]:pos[k] + take]; pos[k] += len(new)
            if tail[k] or new:
                chunks.append((k, tail[k] + new)); budget -= len(chunks[-1][1])
        rb = host_replies(rng, pending)
        if not chunks and not pending:
            rb = host_replies(rng, [rng.getrandbits(62)])          # a reply-only turn
        data, runs, recs = turn(chunks, rb)
        want = pair.twin_turn(data, runs, recs)
        pending = []
        if want[0] is not None:
            rs, msgs = want[0][0], want[0][1]
            for r, (k, c) in enumerate(chunks):
                tail[k] = c[int(rs["consumed"][r]):]
                if rs["parse_error"][r]:                       # the reference closes the socket
                    tail[k], pos[k] = b"", len(streams[k])
            pending = [int(m["correlation_id"]) for m in msgs if m["status"] == 2]
        turns.append((data, runs, recs, want))
        assert len(turns) < 400
    assert sum(len(t[2]) for t in turns) > 10
    for g0 in range(0, len(turns), depth):
        group = turns[g0:g0 + depth]
        ts = [pair.ring.ring_turn_submit(d, r, q) for d, r, q, _ in group]
        assert ts == list(range(pair.last + 1, pair.last + 1 + len(group)))
        pair.last = ts[-1]
        order = list(range(len(group)))
        rng.shuffle(order)
        for i in order:
            d, r, q, want = group[i]
            pair.check(pair.ring.ring_turn_wait(ts[i]), d, r, q, want, ("turn", g0 + i))
    pair.close()


def test_turn_shapes():
    from brpc_b200.abi import PinnedBuffer
    rng = random.Random(SEED + 2)
    pair = Pair()
    reqs = _requests(rng, 4, 6)
    pair.step([(k, reqs[k]) for k in range(4)], what="runs only")
    pair.step([], host_replies(rng, range(20)), what="replies only")
    pair.step([(0, reqs[0][:777]), (1, reqs[1])], host_replies(rng, range(100, 109)), what="both")
    for s in SHAPES:
        pair.step([(2, reqs[2])], host_replies(rng, range(200, 204), shape=s), what=s)
    # a turn larger than b2_ring_submit's 128 KiB because of its reply bodies
    data, runs, recs = turn([(k, reqs[k]) for k in range(4)], host_replies(rng, range(300, 304), shape="snappy_crc", size=60000))
    assert len(data) > 128 << 10
    pair.turn(data, runs, recs, "over 128 KiB")
    # bytes in b2_block_alloc memory are pulled in place, other bytes staged: the same results
    data, runs, recs = turn([(k, reqs[k]) for k in range(4)], host_replies(rng, range(400, 412)))
    buf = PinnedBuffer(len(data) + 4096)
    buf.array[:len(data)] = data
    pair.turn(data, runs, recs, "pinned bytes", ptr=buf.ptr, nbytes=len(data))
    pair.turn(data, runs, recs, "staged again")
    pair.close()
    buf.free()


def test_by_ref_and_iovec_apply_to_the_runs():
    """B2_RESP_BY_REF / B2_RESP_IOVEC shape the runs' replies as in b2_ring_wait; the host replies come back as whole frames"""
    from test_gpu_modes import replies
    rng = random.Random(SEED + 3)
    pair = Pair()
    frames = [echo_frame(rng, i, rnd62(rng, rng.choice([100, 1024]))) for i in range(40)] + \
             [echo_frame(rng, 99, b"x" * 50, method=b"Host"), echo_frame(rng, 98, b"y" * 70, checksum_type=1)]
    for rm in (1, 2):
        pair.ring.set_modes(0, rm); pair.twin.set_modes(0, rm)
        data, runs, recs = turn([(0, b"".join(frames[:20])), (1, b"".join(frames[20:]))], host_replies(rng, range(7), shape="snappy_crc"))
        tw = pair.twin.process_batch(data, runs)
        t_rs, t_msgs, t_info = tw[0].copy(), tw[1].copy(), tw[3]
        t_refs = None if t_info["refs"] is None else t_info["refs"].copy()
        t_frames = pair.twin.pack_responses(data, recs, out_cap=RESP_OUT)
        pair.last = pair.ring.ring_turn_submit(data, runs, recs)
        rs, msgs, resp, info, got = pair.ring.ring_turn_wait(pair.last)
        o_rs, o_msgs, o_resp = O.process_batch(CFG, data, runs)
        for f in RUN_FIELDS:
            assert np.array_equal(rs[f], t_rs[f]) and np.array_equal(rs[f], o_rs[f]), (rm, f)
        for f in MSG_FIELDS:
            assert np.array_equal(msgs[f], t_msgs[f]) and np.array_equal(msgs[f], o_msgs[f]), (rm, f)
        want = replies(data, o_msgs, o_resp, None)
        if rm == 1:
            assert info["refs"] is not None and np.array_equal(info["refs"], t_refs)
            assert replies(data, msgs, resp, info["refs"]) == want
        else:
            iov = info["iov"]
            assert iov is not None and len(iov) == 2 * len(msgs)
            answered = (msgs["status"] == 0) | (msgs["status"] == 1)
            for k in range(len(msgs)):
                g = b"".join(C.string_at(int(iov["base"][j]), int(iov["len"][j])) for j in (2 * k, 2 * k + 1) if iov["len"][j])
                assert g == (want[k] if answered[k] else b""), (k, int(msgs["status"][k]))
        assert got == t_frames == [O.pack_response(r, data) for r in recs], rm
    pair.ring.set_modes(0, 0); pair.twin.set_modes(0, 0)
    pair.close()


def test_overflow_served_by_the_big_pipeline():
    """runs with more messages than the compact block holds are served through the big pipeline inside the wait; the replies of the same
    turn still come from the kernel, and a turn behind it in the ring is served by the kernel"""
    rng = random.Random(SEED + 4)
    pair = Pair()
    tiny = b"".join(echo_frame(rng, i, b"") for i in range(1100))                    # 1100 > 1024 messages
    data, runs, recs = turn([(0, tiny)], host_replies(rng, range(17)))
    want = pair.twin_turn(data, runs, recs)
    data2, runs2, recs2 = turn([(1, tiny[:3000])], host_replies(rng, range(50, 53)))
    want2 = pair.twin_turn(data2, runs2, recs2)
    t = pair.ring.ring_turn_submit(data, runs, recs)
    t2 = pair.ring.ring_turn_submit(data2, runs2, recs2)
    pair.check(pair.ring.ring_turn_wait(t2), data2, runs2, recs2, want2, "behind")
    got = pair.ring.ring_turn_wait(t)
    assert len(got[1]) == 1100
    pair.check(got, data, runs, recs, want, "overflow")
    pair.last = t2
    pair.step([(0, tiny[:5000])], host_replies(rng, [999]), what="after the overflow")
    pair.close()


def test_refusals_and_capacity():
    import brpc_b200
    from brpc_b200.abi import B2_E_CAPACITY, B2_E_INVAL, REPLY_DT, REQUEST_DT
    rng = random.Random(SEED + 5)
    c = _ctx()
    assert _err(c.ring_turn_enable, 0, 8, 1 << 16) == B2_E_INVAL                          # a zero cap
    assert _err(c.ring_turn_enable, 1 << 16, 0, 1 << 16) == B2_E_INVAL
    assert _err(c.ring_turn_enable, 1 << 16, 8, 0) == B2_E_INVAL
    assert _err(c.ring_turn_enable, (4 << 20) + 1, 8, 1 << 16) == B2_E_CAPACITY            # max_batch_bytes
    assert _err(c.ring_turn_enable, 1 << 16, (1 << 14) * 64 // 88 + 1, 1 << 16) == B2_E_CAPACITY   # max_resps * 88 > max_msgs * 64
    assert _err(c.ring_turn_enable, 1 << 16, 8, (8 << 20) + 1) == B2_E_CAPACITY            # max_resp_bytes
    data, runs, recs = turn([(0, b"\0" * 32)], host_replies(rng, [1]))
    assert _err(c.ring_turn_submit, data, runs, recs) == B2_E_INVAL                          # not enabled
    assert _err(c.ring_turn_wait, 1) == B2_E_INVAL
    c.ring_turn_enable(8192, 3, 4000)
    data, runs, recs = turn([(0, b"\0" * 32), (1, b"\0" * 32)], host_replies(rng, [2, 3, 4], shape="ok", size=100))
    refused = [
        (B2_E_INVAL, (data, runs[:0], recs[:0])),                                            # neither runs nor replies
        (B2_E_CAPACITY, (np.zeros(8193, np.uint8), runs[:1], recs[:0])),                    # nbytes > max_bytes
        (B2_E_CAPACITY, (np.zeros(8192, np.uint8), np.zeros(513, runs.dtype), recs[:0])),  # 513 runs
        (B2_E_CAPACITY, (data, runs, np.concatenate([recs, recs[:1]]))),                    # n_replies > max_resps
    ]
    bad = runs.copy(); bad["offset"][1] = 8
    refused.append((B2_E_INVAL, (data, bad, recs)))                                          # a run not 16-aligned
    bad = runs.copy(); bad["length"][1] = len(data)
    refused.append((B2_E_INVAL, (data, bad, recs)))                                          # a run outside the bytes
    for field, value in (("body_len", len(data)), ("attachment_off", len(data)), ("error_text_len", len(data)),
                         ("checksum_value_off", len(data)), ("user_fields_off", len(data) + 1), ("n_user_fields", 1), ("extra_streams_off", 4)):
        q = recs.copy(); q[field][2] = value
        if field == "attachment_off":
            q["attachment_len"][2] = 1
        if field == "checksum_value_off":
            q["checksum_value_len"][2] = 1
        if field == "n_user_fields":
            q["user_fields_off"][2] = len(data) - 4
        refused.append((B2_E_INVAL, (data, runs, q)))                                        # a reply field outside the bytes
    refused.append((B2_E_CAPACITY, turn([], host_replies(rng, [5, 6], shape="ok", size=3000))))   # resp_out_cap too small
    for i, (code, args) in enumerate(refused):
        assert _err(c.ring_turn_submit, *args) == code, i
    ts = [c.ring_turn_submit(data, runs, recs) for _ in range(8)]
    assert ts == list(range(1, 9))                                                           # a failed submit takes no ticket number
    assert _err(c.ring_turn_submit, data, runs, recs) == B2_E_CAPACITY                      # eight outstanding
    # every call that uploads to the context is refused while a turn is outstanding
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
        c.ring_turn_wait(t)
    for i, f in enumerate(uploads):
        assert _err(f) == B2_E_INVAL, ("one still outstanding", i)
    got = c.ring_turn_wait(ts[0])
    assert got[4] == [O.pack_response(r, data) for r in recs]
    assert _err(c.ring_turn_wait, ts[0]) == B2_E_INVAL                                      # already collected
    assert _err(c.ring_turn_wait, 9) == B2_E_INVAL                                          # not submitted
    c.crc32c_batch(small, [0], [16])                                                         # between turns they work again
    assert c.pack_responses(data, recs, out_cap=4000) == got[4]
    assert c.ring_turn_submit(data, runs, recs) == 9
    c.ring_turn_wait(9)
    c.close()


def test_one_ring_kind_per_context():
    import brpc_b200
    from brpc_b200.abi import H2_RESPONSE_DT, REQUEST_DT
    from brpc_b200.abi import B2_E_INVAL
    caps = (1 << 16, 16, 1 << 16)
    rng = random.Random(SEED + 6)
    data, runs = brpc_b200.make_runs([b"\0" * 16])
    tdata, truns, trecs = turn([], host_replies(rng, [1], shape="ok"))
    a = _ctx(); a.ring_start()
    assert _err(a.ring_turn_enable, *caps) == B2_E_INVAL                                    # after k_ring
    assert _err(a.ring_turn_submit, tdata, truns, trecs) == B2_E_INVAL
    a.ring_wait(a.ring_submit(data, runs))
    assert _err(a.ring_turn_wait, 1) == B2_E_INVAL
    b = _ctx(); b.h2_configure(max_conns=8); b.h2_ring_enable(1 << 16, 64, 1 << 16, 1 << 16)
    assert _err(b.ring_turn_enable, *caps) == B2_E_INVAL                                    # after k_h2_ring
    c = _ctx(); c.client_ring_enable(*caps)
    assert _err(c.ring_turn_enable, *caps) == B2_E_INVAL                                    # after the client ring
    assert _err(c.ring_turn_submit, tdata, truns, trecs) == B2_E_INVAL
    d = _ctx(); d.stream_configure(64, 1 << 16)
    assert _err(d.ring_turn_enable, *caps) == B2_E_INVAL                                    # a context with a stream table
    e = _ctx(); e.ring_turn_enable(*caps)
    assert _err(e.ring_turn_enable, *caps) == B2_E_INVAL                                    # twice
    for f in (lambda: e.h2_ring_enable(1 << 16, 64, 1 << 16, 1 << 16), lambda: e.client_ring_enable(*caps), lambda: e.stream_ring_enable(1 << 16),
              lambda: e.ring_submit(data, runs), lambda: e.h2_ring_submit(data, runs), lambda: e.client_ring_submit(data, runs, np.zeros(0, REQUEST_DT)),
              lambda: e.h2_ring_turn_submit(data, runs, np.zeros(0, H2_RESPONSE_DT))):
        assert _err(f) == B2_E_INVAL
    t = e.ring_turn_submit(tdata, truns, trecs)
    for w in (e.ring_wait, e.h2_ring_wait, e.client_ring_wait, e.h2_ring_turn_wait, e.stream_ring_wait):
        assert _err(w, t) == B2_E_INVAL
    assert e.ring_turn_wait(t)[4] == [O.pack_response(trecs[0], tdata)]
    e.ring_stop(); e.ring_start()                                                            # b2_ring_start serves the context's own kind
    t = e.ring_turn_submit(tdata, truns, trecs)
    assert len(e.ring_turn_wait(t)[4][0]) > 0
    for x in (a, b, c, d, e):
        x.close()


def _steady(pair, rng, reqs, steps):
    for s in range(steps):
        got = pair.step([(k, reqs[k]) for k in range(4)], host_replies(rng, range(4 * s, 4 * s + 4), shape=rng.choice(["ok", "snappy_crc"]), size=200))
        assert len(got[1]) == 12 and len(got[4]) == 4 and all(got[4])


def test_no_launch_over_100_steady_turns_and_idle_retirement(monkeypatch):
    gc.collect()                                                     # (no context of an earlier test is destroyed while this one counts)
    monkeypatch.setenv("B2_RING_IDLE_MS", "2000")
    rng = random.Random(SEED + 7)
    reqs = [b"".join(echo_frame(rng, 10 * k + j, rnd62(rng, 100), method=rng.choice([b"Echo", b"Host"])) for j in range(3)) for k in range(4)]
    pair = Pair()
    _steady(pair, rng, reqs, 1)
    n0 = pair.ring.ring_launches()
    _steady(pair, rng, reqs, 100)
    assert pair.ring.ring_launches() == n0
    pair.ring.ring_stop()
    monkeypatch.setenv("B2_RING_IDLE_MS", "5")
    _steady(pair, rng, reqs, 1)                                      # relaunched by the submission, now with a 5 ms idle time
    n1 = pair.ring.ring_launches()
    assert n1 == n0 + 1
    time.sleep(0.2)                                                  # it retires and comes back with the next submission
    _steady(pair, rng, reqs, 2)
    assert pair.ring.ring_launches() > n1
    ph = pair.ring.ring_phase_ns(pair.last)
    assert 0 < ph[0] <= ph[1] <= ph[2] <= ph[3]
    pair.close()


def test_device_round_trip_client_ring_against_turn_ring():
    """1 000 calls over 64 connections between a client ring context and a server turn context on the same GPU.  A quarter go to the host
    method and are answered in the server's next turn with snappy + CRC32C replies; every call completes exactly once, with its own body,
    and each side's wire bytes are only what its kernel wrote"""
    from test_gpu_client_ring import Req, ticket as client_ticket
    rng = random.Random(SEED + 8)
    n_conns, n_calls = 64, 1000
    client, server = _ctx(), _ctx()
    client.client_ring_enable(MAX_BYTES, MAX_REQS_CLIENT, RESP_OUT)
    server.ring_turn_enable(MAX_BYTES, MAX_RESPS, RESP_OUT)
    sent, answered, host_calls = {}, 0, 0
    to_client = [b""] * n_conns
    pending = []                                                     # host-method calls the server answers in its next turn
    cid, rounds = 1, 0
    while answered < n_calls:
        rounds += 1
        assert rounds < 100
        reqs = []
        for k in range(n_conns):
            if cid <= n_calls:
                host = rng.random() < 0.25
                q = Req(rng, (k << 40) | cid, stream=False, compress=0, size=rng.choice([1, 64, 300]), method_idx=1 if host else 0)
                q.att, q.cks, q.has_log, q.flags = b"", 0, False, 0
                reqs.append((k, q)); sent[q.cid] = q.payload; cid += 1; host_calls += host
        data, runs, recs = client_ticket([(k, to_client[k]) for k in range(n_conns) if to_client[k]], [q for _, q in reqs])
        got = client.client_ring_wait(client.client_ring_submit(data, runs, recs))
        rs, msgs, resp = got[0], got[1], got[2]
        for r in range(len(rs)):
            assert rs["consumed"][r] == runs["length"][r]
        for m in msgs:
            assert m["status"] in (7, 8) and m["error_code"] == 0, (int(m["status"]), int(m["error_code"]))
            src = data if m["status"] == 7 else resp
            body = bytes(src[m["resp_off"]:m["resp_off"] + m["resp_len"]])
            assert body == sent.pop(int(m["correlation_id"]))
            answered += 1
        assert all(len(f) > 0 for f in got[4])
        per = [b"".join(f for (k2, _), f in zip(reqs, got[4]) if k2 == k) for k in range(n_conns)]
        to_client = [b""] * n_conns
        if not any(per) and not pending:
            continue
        rb = ReplyBatch()
        for c_id, payload in pending:
            rb.add(correlation_id=c_id, body=b"\x0a" + _varint(len(payload)) + payload, compress_type=1, checksum_type=1)
        sdata, sruns, srecs = turn([(k, per[k]) for k in range(n_conns) if per[k]], rb)
        srs, smsgs, sresp, _, sframes = server.ring_turn_wait(server.ring_turn_submit(sdata, sruns, srecs))
        assert np.isin(smsgs["status"], (0, 2)).all()
        pending = []
        for r in range(len(srs)):
            k = int(sruns["socket_id"][r])
            ms = smsgs[srs[r]["first_msg"]:srs[r]["first_msg"] + srs[r]["n_msgs"]]
            to_client[k] += b"".join(bytes(sresp[m["resp_off"]:m["resp_off"] + m["resp_len"]]) for m in ms if m["status"] == 0)
            for m in ms[ms["status"] == 2]:
                c_id = int(m["correlation_id"])
                pending.append((c_id, sent[c_id]))
        for rec, f in zip(srecs, sframes):
            assert len(f) > 0
            to_client[int(rec["correlation_id"]) >> 40] += f
    assert not sent and answered == n_calls and host_calls > 150
    client.close(); server.close()

