"""GPU: b2_stream_write (the sending side of brpc's Stream) against the sequential oracle of tests/_stream_write.py — statuses, produced,
n_frames, host_socket_id, out offsets and every frame byte — over seeded write lists interleaving hundreds of streams whose windows
fill mid-list, receive batches between the calls whose FEEDBACK reopens them (B2_STREAM_EV_WRITABLE), every alignment of source and
frame head, FROM_MSG writes of what the receive pass left on the device, and a round trip between two contexts."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import _oracle as O  # noqa: E402
import _stream_write as W  # noqa: E402
import _streams as S  # noqa: E402
from _traffic import SEED  # noqa: E402

EV_FIELDS = ("flags", "remote_consumed", "local_consumed", "consumed_bytes", "n_msgs", "pending_bytes")


def layout(rng, payloads):
    """the payloads at unaligned offsets of one buffer -> (data, [(off, len)])"""
    parts, spans, off = [], [], 0
    for p in payloads:
        gap = rng.randrange(16)
        parts.append(rng.randbytes(gap)); off += gap
        spans.append((off, len(p))); parts.append(p); off += len(p)
    return b"".join(parts), spans


def check_write(ctx, orc, sids, payloads, seg, what, rng=None, writes=None, data=None):
    """host-sourced writes of payloads[i] to sids[i] (or the given FROM_MSG records): device == oracle"""
    if writes is None:
        data, spans = layout(rng, payloads)
        writes = [(sid, 0, off, n) for sid, (off, n) in zip(sids, spans)]
    res, out = ctx.stream_write(writes, data, seg)
    want, want_out = orc.write_many(list(zip(sids, payloads)), seg)
    assert len(res) == len(want)
    assert out[:len(want_out)].tobytes() == want_out, what          # every write's frames, and zero bytes in the alignment gaps
    for i, (r, w) in enumerate(zip(res, want)):
        got = {k: int(r[k]) for k in ("status", "n_frames", "out_off", "out_len", "produced", "host_socket_id")}
        assert got == {k: w[k] for k in got}, "%s write %d" % (what, i)
        if w["status"] == 0:
            assert out[w["out_off"]:w["out_off"] + w["out_len"]].tobytes() == b"".join(w["frames"]), "%s write %d bytes" % (what, i)
    return res, out


def check_events(ctx, orc, data, dev, what):
    rs, msgs = dev[0], dev[1]
    _, events, _, _, _ = ctx.stream_results()
    _, want, _ = orc.process(data, rs, msgs)
    assert sorted(int(e["stream_id"]) for e in events) == sorted(want), what
    for e in events:
        w = want[int(e["stream_id"])]
        got = {k: int(e[k]) for k in EV_FIELDS}
        assert got == {"flags": w["flags"], "remote_consumed": w["remote_consumed"], "local_consumed": w["local_consumed"],
                       "consumed_bytes": w["consumed"], "n_msgs": w["n_msgs"], "pending_bytes": w["pending_bytes"]}, "%s stream %d" % (what, int(e["stream_id"]))
    return events


def receive(ctx, orc, frames, what, pin=None):
    import brpc_b200 as b2
    data, runs = b2.make_runs(frames)
    if pin is not None:
        pin.array[:len(data)] = data
        dev = ctx.process_batch_ptr(pin.ptr, len(data), runs)
    else:
        dev = ctx.process_batch(data, runs)
    return data, dev, check_events(ctx, orc, data, dev, what)


def rand_id(rng, negative=True):
    """ids of every varint length class; local ids stay non-negative here because the receive oracle's CLOSE frame takes a negative
    source_stream_id for "absent" (negative local ids are covered by test_every_alignment_of_source_and_frame_head)"""
    return rng.choice((rng.randrange(1, 1 << 14), rng.randrange(1, 1 << 40), rng.randrange(1 << 62, 1 << 63)) + ((-rng.randrange(1, 1 << 63),) if negative else ()))


@pytest.mark.parametrize("seg", [0, 1, 4096, 65536])
def test_seeded_write_lists_equal_the_oracle(seg):
    import brpc_b200 as b2
    rng = random.Random(SEED + seg)
    ctx = b2.Context(device=0, max_batch_bytes=32 << 20, max_msgs=1 << 14, max_runs=64, max_resp_bytes=96 << 20)
    ctx.stream_configure(512, 4096)
    orc = W.WriteOracle()
    n_streams, n_writes, top = (120, 400, 600) if seg == 1 else (240, 1500, 300 << 10)
    ids = list({rand_id(rng, False) for _ in range(n_streams + 8)})
    rng.shuffle(ids)
    sids, unknown = ids[:n_streams], ids[n_streams:]
    streams = []
    for sid in sids:
        conn = rng.random() < 0.9
        win = 0 if rng.random() < 0.25 else rng.choice((1, 700, 8 << 10, 256 << 10, 2 << 20)) if seg != 1 else rng.choice((0, 1, 300, 2000))
        streams.append((sid, rand_id(rng), rng.randrange(1 << 60), conn, win))
    ctx.stream_open([(sid, remote, sock, (1 if conn else 0) | 2, win) for sid, remote, sock, conn, win in streams])
    for sid, remote, sock, conn, win in streams:
        orc.open(sid, remote, sock, conn, True, win)
    remote_of = {sid: remote for sid, remote, _, _, _ in streams}

    def length():
        r = rng.random()
        return 0 if r < 0.03 else rng.randrange(1, 65) if r < 0.4 else rng.randrange(top // 16 + 1) if r < 0.95 else rng.randrange(top + 1)
    for rnd in range(3):
        ws = [rng.choice(unknown) if rng.random() < 0.02 else rng.choice(sids) for _ in range(n_writes)]
        payloads = [rng.randbytes(length()) for _ in ws]
        res, _ = check_write(ctx, orc, ws, payloads, seg, "seg %d round %d" % (seg, rnd), rng)
        sts = set(int(s) for s in res["status"])
        assert {0, W.EAGAIN, W.EINVAL, W.NOT_CONNECTED} <= sts, sts
        # the peers answer: FEEDBACK (some moving remote_consumed past produced, some not), a few RST / CLOSE, a late SetConnected
        frames = []
        for sid in rng.sample(sids, n_streams // 2):
            s = orc.streams.get(sid)
            if s is None or s.closed:
                continue
            c = rng.choice((s.produced, s.produced // 2, s.remote_consumed, s.produced + 5))
            frames.append(S.feedback_frame(sid, remote_of[sid], c))
        for sid in rng.sample(sids, 3):
            frames.append(O.pack_stream_frame(sid, remote_of[sid], rng.choice((S.RST, S.CLOSE))))
        rng.shuffle(frames)
        _, _, events = receive(ctx, orc, [b"".join(frames[k::4]) for k in range(4)], "seg %d feedback %d" % (seg, rnd))
        assert any(int(e["flags"]) & W.EV_WRITABLE for e in events)
        assert all(not (int(e["flags"]) & W.EV_WRITABLE) for e in events if orc.streams[int(e["stream_id"])].max_buf == 0)
        for sid, remote, _, conn, _ in streams:
            s = orc.streams.get(sid)
            if s is not None and not s.connected and not s.closed and rng.random() < 0.5:
                assert ctx.stream_set_connected(sid, remote, 2) == orc.set_connected(sid, remote, True)
        gone = rng.choice([sid for sid in sids if sid in orc.streams])
        assert ctx.stream_close(gone) == orc.close(gone)


def id_of_varint_len(v, k):
    """an id (k = 1 .. 127 tells them apart) whose varint is v bytes long: 10 bytes is every negative id"""
    return -k if v == 10 else k if v == 1 else (1 << (7 * (v - 1))) + k


def test_every_alignment_of_source_and_frame_head():
    """source offset mod 16 x meta length 8 .. 26 (so every residue of the 12 + meta head), single frames and segmented ones"""
    import brpc_b200 as b2
    rng = random.Random(SEED + 7)
    ctx = b2.Context(device=0, max_batch_bytes=8 << 20, max_msgs=1 << 12, max_runs=16)
    ctx.stream_configure(64, 4096)
    orc = W.WriteOracle()
    pairs, metas = [], set()
    for vr in range(1, 11):
        for vi in range(1, 11):
            ml = 2 + vr + vi + 4
            if ml in metas:
                continue
            metas.add(ml)
            remote, sid = id_of_varint_len(vr, 1), id_of_varint_len(vi, 11 * vr + vi)
            assert 2 + len(W._varint(remote)) + len(W._varint(sid)) + 4 == ml
            pairs.append((sid, remote))
    assert sorted(metas) == list(range(8, 27))
    ctx.stream_open([(sid, remote, 5, 3) for sid, remote in pairs])
    for sid, remote in pairs:
        orc.open(sid, remote, 5, True, True)
    for seg, n in ((0, 100), (0, 33), (1000, 4500)):
        sids, payloads, writes, parts, off = [], [], [], [], 0
        for sid, _ in pairs:
            for r in range(16):
                gap = (r - off) % 16
                parts.append(b"\xee" * gap); off += gap
                p = rng.randbytes(n)
                parts.append(p); writes.append((sid, 0, off, n)); off += n
                sids.append(sid); payloads.append(p)
        data = b"".join(parts)
        assert sorted({w[2] % 16 for w in writes}) == list(range(16))
        check_write(ctx, orc, sids, payloads, seg, "alignment seg %d len %d" % (seg, n), writes=writes, data=data)


@pytest.mark.parametrize("shape,mode", [("small", "copy"), ("big", "copy"), ("small", "pull"), ("big", "pull")])
def test_from_msg_echo_reads_the_last_batch_in_place(shape, mode):
    """FROM_MSG writes of every completed message (single-frame: the input bytes; multi-frame: the out region) on the reverse stream;
    b2_stream_results stays byte-identical across the write calls"""
    import brpc_b200 as b2
    rng = random.Random(SEED + (1 if shape == "big" else 0) + (2 if mode == "pull" else 0))
    ctx = b2.Context(device=0, max_batch_bytes=16 << 20, max_msgs=1 << 14, max_runs=64)
    ctx.stream_configure(256, 64 << 10)
    orc = W.WriteOracle()
    n, size = (16, 300) if shape == "small" else (160, 20000)
    pairs = [(1000 + 2 * i, 5000 + i) for i in range(n)]     # (id, the peer's id)
    ctx.stream_open([(sid, remote, i % 7, 3, 1 << 20) for i, (sid, remote) in enumerate(pairs)])
    for i, (sid, remote) in enumerate(pairs):
        orc.open(sid, remote, i % 7, True, True, 1 << 20)
    pin = None
    if mode == "pull":
        ctx.set_modes(b2.abi.INPUT_PULL, b2.abi.RESP_COPY)
        pin = b2.abi.PinnedBuffer(16 << 20)
    for rnd in range(2):
        socks = [[] for _ in range(4)]
        for sid, remote in pairs:
            for _ in range(rng.randrange(1, 3)):
                parts = rng.choice((1, 1, 3))
                for p in range(parts):
                    socks[sid % 4].append(O.pack_stream_frame(sid, remote, S.DATA, True if p < parts - 1 else None, rng.randbytes(rng.randrange(1, size))))
        data, dev, events = receive(ctx, orc, [b"".join(s) for s in socks], "%s/%s batch %d" % (shape, mode, rnd), pin)
        assert (len(data) > (128 << 10)) == (shape == "big")
        before = [np.array(a, copy=True) for a in ctx.stream_results()]
        smsgs = before[0]
        assert np.any(smsgs["flags"] & 1) and np.any(~smsgs["flags"] & 1)
        src = np.asarray(data)
        payloads = [(src if int(m["flags"]) & 1 else before[2])[int(m["off"]):int(m["off"]) + int(m["len"])].tobytes() for m in smsgs]
        sids = [int(m["stream_id"]) for m in smsgs]
        writes = [(sid, b2.abi.STREAM_W_FROM_MSG, k, 0) for k, sid in enumerate(sids)]
        for seg in (0, 4096):
            check_write(ctx, orc, sids, payloads, seg, "%s/%s echo %d seg %d" % (shape, mode, rnd, seg), writes=writes)
        after = ctx.stream_results()
        assert all(np.array_equal(a, b) for a, b in zip(before, after))
        with pytest.raises(b2.B2Error):
            ctx.stream_write([(sids[0], b2.abi.STREAM_W_FROM_MSG, len(smsgs), 0)])


def test_hand_over_refusals_capacity_and_a_round_trip():
    import brpc_b200 as b2
    A = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 12, max_runs=16)
    B = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 12, max_runs=16)
    A.stream_configure(16, 1024); B.stream_configure(16, 1 << 20)
    oa, ob = W.WriteOracle(pending_bytes=1024, out_bytes=4 << 20), W.WriteOracle()
    AID, BID, H = 0x1111, -0x2222, 77
    A.stream_open([(AID, BID, 3, 3, 300000), (H, 9, 4, 3, 0)]); oa.open(AID, BID, 3, True, True, 300000); oa.open(H, 9, 4, True, True)
    B.stream_open([(BID, AID, 8, 3)]); ob.open(BID, AID, 8, True, True)
    # a stream handed over by the receive pass refuses writes: its FEEDBACK now reaches only the host
    receive(A, oa, [O.pack_stream_frame(H, 9, S.DATA, True, b"p" * 2000)], "hand-over")
    assert A.stream_query(H)["flags"] & 8
    # refused between submit and collect: the table belongs to the submitted batch
    data, runs = b2.make_runs([b"x" * 16])
    pin = b2.abi.PinnedBuffer(4096); pin.array[:len(data)] = data
    A.submit_ptr(pin.ptr, len(data), runs)
    with pytest.raises(b2.B2Error):
        A.stream_write([(AID, 0, 0, 1)], b"y")
    A.collect()
    rng = random.Random(SEED + 11)
    payloads = [rng.randbytes(n) for n in (100000, 150000, 60000, 60000, 70000)]     # the fourth overshoots the window of 300 000
    sids = [AID, AID, H, AID, AID]
    # capacity: nothing changes
    with pytest.raises(b2.B2Error) as e:
        A.stream_write([(AID, 0, 0, 100000)], payloads[0], 0, out_cap=100000)
    assert e.value.code == b2.abi.B2_E_CAPACITY
    res, out = check_write(A, oa, sids, payloads, 65536, "writer", rng)
    assert [int(s) for s in res["status"]] == [0, 0, W.HANDED_OVER, 0, W.EAGAIN]
    wire = b"".join(out[int(r["out_off"]):int(r["out_off"]) + int(r["out_len"])].tobytes() for r in res if int(r["status"]) == 0)
    _, _, ev = receive(B, ob, [wire], "reader")
    smsgs, _, bout, _, _ = B.stream_results()
    assert [bout[int(m["off"]):int(m["off"]) + int(m["len"])].tobytes() if not int(m["flags"]) & 1 else None for m in smsgs][:2] == payloads[:2]
    assert len(smsgs) == 3 and int(ev[0]["fb_len"]) > 0
    ctrl = B.stream_results()[3]
    fb = ctrl[int(ev[0]["fb_off"]):int(ev[0]["fb_off"]) + int(ev[0]["fb_len"])].tobytes()
    _, _, aev = receive(A, oa, [fb], "feedback to the writer")
    assert int(aev[0]["flags"]) == S.EV_MOVED | W.EV_WRITABLE
    check_write(A, oa, [AID], [payloads[4]], 65536, "after the FEEDBACK", rng)


@pytest.mark.parametrize("mode", ["copy", "pull"])
def test_from_msg_after_a_call_that_overwrote_the_input(mode):
    """a call that uploads other bytes (b2_crc32c_batch, b2_pack_responses) between the batch and the write: in copy mode a FROM_MSG
    write of a single-frame message (its bytes were the device copy of the input) is refused; multi-frame messages in the out region,
    and every message of a B2_INPUT_PULL batch, are still written from the right bytes"""
    import brpc_b200 as b2
    rng = random.Random(SEED + 13)
    ctx = b2.Context(device=0, max_batch_bytes=4 << 20, max_msgs=1 << 12, max_runs=16)
    ctx.stream_configure(8, 4096)
    orc = W.WriteOracle()
    ctx.stream_open([(1, 2, 7, 3)]); orc.open(1, 2, 7, True, True)
    pin = None
    if mode == "pull":
        ctx.set_modes(b2.abi.INPUT_PULL, b2.abi.RESP_COPY)
        pin = b2.abi.PinnedBuffer(1 << 20)
    one, two = rng.randbytes(200), rng.randbytes(3000)
    receive(ctx, orc, [O.pack_stream_frame(1, 2, S.DATA, None, one) + O.pack_stream_frame(1, 2, S.DATA, True, two[:1000]) +
                       O.pack_stream_frame(1, 2, S.DATA, None, two[1000:])], "batch", pin)
    smsgs = ctx.stream_results()[0]
    assert [int(m["flags"]) & 1 for m in smsgs] == [1, 0]
    check_write(ctx, orc, [1, 1], [one, two], 0, "before", writes=[(1, b2.abi.STREAM_W_FROM_MSG, 0, 0), (1, b2.abi.STREAM_W_FROM_MSG, 1, 0)])
    assert ctx.crc32c_batch(np.frombuffer(b"Z" * 4096, np.uint8), [0], [4096]) is not None
    rep = np.zeros(1, b2.abi.REPLY_DT); rep[0]["body_len"] = 4096
    assert len(ctx.pack_responses(np.frombuffer(b"Z" * 4096, np.uint8), rep)[0]) > 4096
    if mode == "copy":
        with pytest.raises(b2.B2Error) as e:
            ctx.stream_write([(1, b2.abi.STREAM_W_FROM_MSG, 0, 0)])
        assert e.value.code == b2.abi.B2_E_INVAL and "overwrote" in str(e.value)
        check_write(ctx, orc, [1], [two], 0, "out region after", writes=[(1, b2.abi.STREAM_W_FROM_MSG, 1, 0)])
    else:
        check_write(ctx, orc, [1, 1], [one, two], 0, "pull after", writes=[(1, b2.abi.STREAM_W_FROM_MSG, 0, 0), (1, b2.abi.STREAM_W_FROM_MSG, 1, 0)])
    assert [int(m["flags"]) & 1 for m in ctx.stream_results()[0]] == [1, 0]          # the results themselves stay
