"""CPU: the write oracle (tests/_stream_write.py) against python-protobuf, the reference's own StreamWrite cases and the order of the
rules, and a round trip through the receive oracle."""
import struct

import pytest

import _oracle as O
import _stream_write as W
import _streams as S

pytest.importorskip("google.protobuf")
from test_oracle_streams import _frame_meta_class, batch  # noqa: E402

Meta = _frame_meta_class()


def split(frame):
    assert frame[:4] == b"STRM"
    body, meta = struct.unpack(">II", frame[4:12])
    assert len(frame) == 12 + body
    return frame[12:12 + meta], frame[12 + meta:]


@pytest.mark.parametrize("nbytes", range(1, 11))
def test_data_metas_equal_python_protobuf(nbytes):
    """ids whose varints are 1 .. 10 bytes long: 10 bytes is every negative id"""
    ids = [(1 << (7 * (nbytes - 1))) + 3 if nbytes < 10 else -5, (1 << (7 * nbytes)) - 1 if nbytes < 10 else -(1 << 62)]
    for remote in ids:
        for sid in ids:
            for cont in (False, True):
                m = Meta(stream_id=remote, source_stream_id=sid, frame_type=S.DATA, has_continuation=cont)
                meta, payload = split(W.data_frame(remote, sid, cont, b"xyz"))
                assert meta == m.SerializeToString() and payload == b"xyz"
                assert len(meta) <= W.HEAD_MAX - 12
                if sid >= 0:                 # the C oracle's packer (a negative source_stream_id means "absent" there)
                    assert W.data_frame(remote, sid, cont, b"xyz") == O.pack_stream_frame(remote, sid, S.DATA, cont, b"xyz")
    (f,) = W.cut_frames(ids[0], ids[1], b"abc")
    assert Meta.FromString(split(f)[0]).HasField("has_continuation")          # set_has_continuation(false): on the wire


def oracle_with(sid=1, remote=2, max_buf=0, connected=True, sock=7):
    o = W.WriteOracle()
    o.open(sid, remote, sock, connected, True, max_buf)
    return o


def test_block():
    """brpc_streaming_rpc_unittest.cpp:441-535: max_buf_size = 4 N; N writes of 4 bytes fill it, the next one is EAGAIN; FEEDBACK of
    what the peer consumed reopens the window for N more"""
    N = 1000
    o = oracle_with(max_buf=4 * N)
    for i in range(N):
        assert o.write(1, struct.pack(">I", i))[0] == 0
    assert o.write(1, b"\0\0\0\0")[:3] == (W.EAGAIN, [], 4 * N)
    o.streams[1].remote_consumed = 4 * N
    for i in range(N):
        assert o.write(1, struct.pack(">I", N + i))[0] == 0
    assert o.write(1, b"\0\0\0\0")[0] == W.EAGAIN and o.streams[1].produced == 8 * N


def test_batch_create_stream_feedback_race():
    """:160-190: 64 bytes at max_buf_size 64 are accepted (the check is before the add); the next byte is EAGAIN until the client's
    FEEDBACK of 64 arrives, and that FEEDBACK sets WRITABLE (a FEEDBACK that does not move remote_consumed changes nothing)"""
    o = oracle_with(max_buf=64)
    assert o.write(1, b"a" * 64)[:3] == (0, [O.pack_stream_frame(2, 1, S.DATA, False, b"a" * 64)], 64)
    assert o.write(1, b"b")[0] == W.EAGAIN
    for consumed, writable in ((0, False), (64, True)):
        data, rs, msgs = batch([[S.feedback_frame(1, 2, consumed)]])
        _, ev, _ = o.process(data, rs, msgs)
        assert bool(ev[1]["flags"] & W.EV_WRITABLE) == writable
        assert o.write(1, b"b")[0] == (0 if writable else W.EAGAIN)
    assert o.streams[1].produced == 65


def test_overshoot_by_one_write():
    o = oracle_with(max_buf=10)
    assert [o.write(1, b"x" * n)[0] for n in (9, 100, 1)] == [0, 0, W.EAGAIN] and o.streams[1].produced == 109


def test_segment_stream_data_automatically():
    """:812-865: -stream_write_max_segment_size=1: every byte its own frame, has_continuation on all but the last"""
    o = oracle_with()
    st, frames, _, _ = o.write(1, struct.pack(">I", 0x01020304), seg=1)
    assert st == 0 and len(frames) == 4
    for k, f in enumerate(frames):
        meta, payload = split(f)
        m = Meta.FromString(meta)
        assert (m.stream_id, m.source_stream_id, m.frame_type, m.has_continuation, payload) == (2, 1, S.DATA, k < 3, bytes([k + 1]))


@pytest.mark.parametrize("seg", [1, 7, 4096])
def test_segment_boundaries(seg):
    o = oracle_with()
    for n, want in ((seg - 1, 1), (seg, 1), (seg + 1, 2), (3 * seg, 3)):
        if n == 0:
            continue
        body = bytes(range(256)) * (n // 256 + 1)
        st, frames, _, _ = o.write(1, body[:n], seg=seg)
        assert st == 0 and len(frames) == want
        assert b"".join(split(f)[1] for f in frames) == body[:n]
        assert [Meta.FromString(split(f)[0]).has_continuation for f in frames] == [True] * (want - 1) + [False]
        assert sum(len(f) for f in frames) + 15 & ~15 <= W.bound(n, seg)


def test_the_order_of_the_rules():
    o = W.WriteOracle()
    o.open(1, 11, 3, True, True, 8)                 # window 8
    o.open(2, 0, 4, False, False, 8)                # not connected
    o.open(3, 13, 5, True, True, 0)                 # no window
    o.open(4, 14, 6, True, True, 0)
    o.streams[4].handed_over = True
    assert o.write(99, b"x")[:2] == (W.EINVAL, [])                      # never opened
    assert o.write(1, b"")[0] == W.EINVAL                               # empty, not full
    assert o.write(1, b"123456789")[0] == 0                             # overshoots
    assert o.write(1, b"")[0] == W.EAGAIN                               # full is checked before empty
    assert o.write(2, b"")[0] == W.EINVAL and o.write(2, b"abc")[0] == W.NOT_CONNECTED and o.streams[2].produced == 0
    o.streams[2].produced = 8                                           # (full) before not connected
    assert o.write(2, b"abc")[0] == W.EAGAIN
    assert o.write(3, b"abc")[:3] == (0, W.cut_frames(13, 3, b"abc"), 0)    # no window: nothing kept
    assert o.write(4, b"abc")[:2] == (W.HANDED_OVER, [])
    data, rs, msgs = batch([[O.pack_stream_frame(3, 9, S.RST)]])
    o.process(data, rs, msgs)
    assert o.write(3, b"abc")[:2] == (W.EINVAL, [])                     # closed by the peer
    o.close(1)
    assert o.write(1, b"abc")[:2] == (W.EINVAL, [])                     # closed locally


def test_round_trip_through_the_receive_oracle():
    """the writer's frames, cut by the cut loop and fed to StreamOracle.process, give the messages back; the reader's FEEDBACK fed to
    the writer sets WRITABLE and lets the next write through"""
    wr, rd = W.WriteOracle(), W.WriteOracle()
    wr.open(10, 20, 1, True, True, 1469)              # 700 + 768 + 1 fill it exactly
    rd.open(20, 10, 2, True, True)
    msgs_in = [b"m" * 700, bytes(range(256)) * 3, b"z"]
    res, out = wr.write_many([(10, m) for m in msgs_in], seg=256)
    assert [r["status"] for r in res] == [0, 0, 0] and wr.write(10, b"more")[0] == W.EAGAIN
    data, rs, msgs = batch([[f for r in res for f in r["frames"]]])
    got, ev, _ = rd.process(data, rs, msgs)
    assert [body for _, _, body in got[20]] == msgs_in
    data, rs, msgs = batch([[ev[20]["fb"]]])
    _, wev, _ = wr.process(data, rs, msgs)
    assert wev[10]["flags"] == S.EV_MOVED | W.EV_WRITABLE and wr.write(10, b"more")[0] == 0
