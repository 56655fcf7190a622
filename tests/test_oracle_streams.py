"""CPU: the stream oracle (tests/_streams.py) against python-protobuf and the rules of brpc's Stream, case by case."""
import numpy as np
import pytest

import _oracle as O
import _streams as S

pb = pytest.importorskip("google.protobuf")
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory  # noqa: E402


def _frame_meta_class():
    """brpc's streaming_rpc_meta.proto (StreamFrameMeta, Feedback, FrameType), declared here field by field."""
    f = descriptor_pb2.FileDescriptorProto(name="b2_test_streaming_rpc_meta.proto", package="b2test", syntax="proto2")
    e = f.enum_type.add(name="FrameType")
    for i, n in enumerate(["FRAME_TYPE_UNKNOWN", "FRAME_TYPE_RST", "FRAME_TYPE_CLOSE", "FRAME_TYPE_DATA", "FRAME_TYPE_FEEDBACK"]):
        e.value.add(name=n, number=i)
    fb = f.message_type.add(name="Feedback")
    fb.field.add(name="consumed_size", number=1, type=3, label=1)
    m = f.message_type.add(name="StreamFrameMeta")
    m.field.add(name="stream_id", number=1, type=3, label=2)
    m.field.add(name="source_stream_id", number=2, type=3, label=1)
    m.field.add(name="frame_type", number=3, type=14, label=1, type_name=".b2test.FrameType")
    m.field.add(name="has_continuation", number=4, type=8, label=1)
    m.field.add(name="feedback", number=5, type=11, label=1, type_name=".b2test.Feedback")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(f)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("b2test.StreamFrameMeta"))


Meta = _frame_meta_class()


def parse(frame):
    assert frame[:4] == b"STRM"
    body, meta = int.from_bytes(frame[4:8], "big"), int.from_bytes(frame[8:12], "big")
    assert body == meta and len(frame) == 12 + body
    m = Meta(); m.ParseFromString(frame[12:])
    assert m.SerializeToString() == frame[12:]
    return m


def batch(frames_per_run):
    """-> (data, rs, msgs) of the cut loop over one run per entry"""
    chunks = [b"".join(r) for r in frames_per_run]
    off, parts, runs = 0, [], np.zeros(len(chunks), O.RUN_DT)
    for i, c in enumerate(chunks):
        runs[i] = (i, off, len(c), -1, 0)
        pad = (-len(c)) % 16
        parts.append(c + b"\0" * pad); off += len(c) + pad
    data = b"".join(parts)
    rs, msgs, _ = O.process_batch(O.make_config(), data, runs)
    return data, rs, msgs


def F(sid, src=-1, t=S.DATA, cont=None, data=b""):
    return O.pack_stream_frame(sid, src, t, cont, data)


def test_control_frames_equal_python_protobuf():
    o = S.StreamOracle()
    o.open(7, remote=1 << 40, sock=3, connected=True, need_feedback=True)
    o.open(8, remote=5, sock=3, connected=True, need_feedback=False)
    data, rs, msgs = batch([[F(7, 9, data=b"x" * 300), F(8, 9, S.CLOSE), F(99, 12345678901, data=b"y")]])
    messages, events, rst = o.process(data, rs, msgs)
    fb = parse(events[7]["fb"])
    assert (fb.stream_id, fb.source_stream_id, fb.frame_type, fb.feedback.consumed_size, fb.HasField("has_continuation")) == (1 << 40, 7, 4, 300, False)
    cl = parse(events[8]["close"])
    assert (cl.stream_id, cl.source_stream_id, cl.frame_type, cl.HasField("feedback")) == (5, 8, 2, False)
    r = parse(rst[0])
    assert (r.stream_id, r.frame_type, r.HasField("source_stream_id")) == (12345678901, 1, False)
    assert parse(o.close(7)).frame_type == 2 and o.close(8) == b""       # (8 was closed by the peer: its CLOSE went out with the batch)
    for v in (1, 127, 128, (1 << 63) - 1, -1):
        m = parse(S.feedback_frame(v, -v, v))
        assert (m.stream_id, m.source_stream_id, m.feedback.consumed_size) == (v, -v, v)


def test_rst_only_for_frames_with_a_source_that_are_not_feedback():
    o = S.StreamOracle()
    fbk = S.feedback_frame(50, 77, 10)           # a FEEDBACK for unknown id 50 that names its source
    data, rs, msgs = batch([[F(50, 77), F(50), fbk, F(50, 78, S.RST), F(50, 79, S.CLOSE), F(50, 80, 0)]])
    _, events, rst = o.process(data, rs, msgs)
    got, p = [], 0
    while p < len(rst[0]):
        n = 12 + int.from_bytes(rst[0][p + 4:p + 8], "big"); got.append(parse(rst[0][p:p + n]).stream_id); p += n
    assert got == [77, 78, 79, 80] and events == {}


def test_frames_after_a_close_in_the_same_batch():
    o = S.StreamOracle()
    o.open(1, remote=2, connected=True, need_feedback=True)
    data, rs, msgs = batch([[F(1, 2, data=b"abc"), F(1, 2, cont=True, data=b"partial"), F(1, 2, S.RST)], [F(1, 2, data=b"late"), F(1, data=b"late2")]])
    messages, events, rst = o.process(data, rs, msgs)
    assert [b for _, _, b in messages[1]] == [b"abc"]
    ev = events[1]
    assert ev["flags"] == S.EV_RST and ev["consumed"] == 3 and ev["pending_bytes"] == 0 and o.query(1)["error_code"] == 104
    assert parse(ev["fb"]).feedback.consumed_size == 3 and parse(ev["close"]).frame_type == 2
    assert rst[0] == b"" and parse(rst[1]).stream_id == 2          # one RST: the second late frame names no source
    data, rs, msgs = batch([[F(1, 2, data=b"next batch")]])
    messages, events, rst = o.process(data, rs, msgs)
    assert events == {} and parse(rst[0]).frame_type == 1


def test_feedback_only_moves_forward():
    o = S.StreamOracle()
    o.open(1)
    data, rs, msgs = batch([[S.feedback_frame(1, 0, 100), S.feedback_frame(1, 0, 100), S.feedback_frame(1, 0, 40)]])
    _, events, _ = o.process(data, rs, msgs)
    assert events[1]["remote_consumed"] == 100 and events[1]["flags"] == S.EV_MOVED
    data, rs, msgs = batch([[S.feedback_frame(1, 0, 99)]])
    _, events, _ = o.process(data, rs, msgs)
    assert events[1]["remote_consumed"] == 100 and events[1]["flags"] == 0


def test_empty_messages_write_no_feedback_and_false_continuation_completes():
    o = S.StreamOracle()
    o.open(1, remote=2, connected=True, need_feedback=True)
    data, rs, msgs = batch([[F(1, data=b""), F(1, cont=True, data=b""), F(1, cont=False, data=b"")]])
    messages, events, _ = o.process(data, rs, msgs)
    assert [(n, b) for _, n, b in messages[1]] == [(1, b""), (2, b"")] and events[1]["fb"] == b"" and events[1]["local_consumed"] == 0
    data, rs, msgs = batch([[F(1, cont=True, data=b"ab")], [F(1, cont=False, data=b"cd"), F(1, t=0, data=b"ignored")]])
    messages, events, _ = o.process(data, rs, msgs)
    assert [(n, b) for _, n, b in messages[1]] == [(2, b"abcd")] and parse(events[1]["fb"]).feedback.consumed_size == 4


def test_messages_straddle_batches_and_the_capacity_rule():
    o = S.StreamOracle(pending_bytes=16, out_bytes=64)
    o.open(1); o.open(2)
    data, rs, msgs = batch([[F(1, cont=True, data=b"0123456789"), F(2, cont=True, data=b"x" * 10)]])
    messages, events, _ = o.process(data, rs, msgs)
    assert messages[1] == [] and events[1]["pending_bytes"] == 10
    data, rs, msgs = batch([[F(1, data=b"ab"), F(2, cont=True, data=b"y" * 10)]])
    messages, events, _ = o.process(data, rs, msgs)
    assert [(n, b) for _, n, b in messages[1]] == [(2, b"0123456789ab")]
    assert events[2]["flags"] == S.EV_HANDED_OVER and events[2]["handover_msg"] == 1 and events[2]["pending_bytes"] == 10 and o.query(2)["handed_over"]
    data, rs, msgs = batch([[F(2, 5, data=b"per frame only")]])
    assert o.process(data, rs, msgs) == ({}, {}, {0: b""})


def test_set_connected_sends_the_first_feedback():
    o = S.StreamOracle()
    o.open(1)
    data, rs, msgs = batch([[F(1, data=b"hello")]])
    _, events, _ = o.process(data, rs, msgs)
    assert events[1]["fb"] == b""
    m = parse(o.set_connected(1, 44, True))
    assert (m.stream_id, m.source_stream_id, m.feedback.consumed_size) == (44, 1, 5)
    assert o.set_connected(1, 45, True) == b""
