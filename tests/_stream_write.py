"""Python oracle of b2_stream_write: the sending side of brpc's Stream, restated sequentially on top of _streams.StreamOracle (the
receiving side, whose outcomes stay as they are) and _oracle.pack_stream_frame.  Reference, function by function:
  StreamWrite                   src/brpc/stream.cpp:782-794   Socket::Address(stream_id) fails -> EINVAL: an id never opened, closed
                                                               locally, or closed by the peer (Close SetFailed's the fake socket, :710)
  AppendIfNotFull               :326-360   only when _cur_buf_size > 0 (max_buf_size > 0; fixed, as -socket_max_streams_unconsumed_bytes
                                           is 0): _produced >= _remote_consumed + _cur_buf_size -> 1 (EAGAIN), else _produced += length,
                                           checked BEFORE the add; then _fake_socket->Write, whose failure gives the length back (:349-353)
  Socket::Write                 socket.cpp:1609-1610  an empty IOBuf -> EINVAL
  CutMessageIntoFileDescriptor  stream.cpp:148-215  length > -stream_write_max_segment_size: cutn(seg) per frame, has_continuation =
                                           !data->empty(); else one frame with has_continuation = false (set_: always on the wire)
  PackStreamMessage             policy/streaming_rpc_protocol.cpp:42-58  "STRM", BE32 body size, BE32 meta size, StreamFrameMeta, payload
  SetRemoteConsumed             stream.cpp:362-401  was_full && !is_full wakes the StreamWait waiters (B2_STREAM_EV_WRITABLE)
Decisions of the device: a HANDED_OVER stream answers B2_STREAM_W_HANDED_OVER and a stream that is not connected answers
B2_STREAM_W_NOT_CONNECTED (brpc would queue the write in the fake socket until SetConnected); neither charges anything."""
import _streams as S

EAGAIN, EINVAL = 11, 22
NOT_CONNECTED, HANDED_OVER = -1, -2
EV_WRITABLE = 16
DEFAULT_SEGMENT = 512 << 20          # -stream_write_max_segment_size (stream.cpp:39)
HEAD_MAX = 38                        # 12 + the longest DATA meta: two 10-byte varints, frame_type, has_continuation


def _varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7f) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


def data_frame(remote, sid, cont, payload):
    """PackStreamMessage of a DATA frame, from the wire rules as _streams.feedback_frame is (_oracle.pack_stream_frame takes a negative
    source_stream_id for "absent", and a local StreamId may be any int64 here): fields 1-4 in number order, has_continuation always set"""
    meta = b"\x08" + _varint(remote) + b"\x10" + _varint(sid) + b"\x18\x03" + b"\x20" + (b"\x01" if cont else b"\x00")
    return b"STRM" + (len(meta) + len(payload)).to_bytes(4, "big") + len(meta).to_bytes(4, "big") + meta + payload


def cut_frames(remote, sid, payload, seg=0):
    """CutMessageIntoFileDescriptor + PackStreamMessage of one message: its frames."""
    seg = seg or DEFAULT_SEGMENT
    if len(payload) <= seg:
        return [data_frame(remote, sid, False, payload)]
    frames, data = [], payload
    while True:
        part, data = data[:seg], data[seg:]                     # data->cutn(&segment_buf, seg)
        frames.append(data_frame(remote, sid, len(data) > 0, part))
        if not data:
            return frames


def bound(length, seg=0):
    """what b2_stream_write asks of out_cap for one write: align16(len + ceil(len / seg) * 38), len 0 as one frame"""
    seg = seg or DEFAULT_SEGMENT
    n = max(1, -(-length // seg))
    return (length + n * HEAD_MAX + 15) & ~15


class WriteOracle(S.StreamOracle):
    def open(self, sid, remote=0, sock=0, connected=False, need_feedback=False, max_buf_size=0):
        super().open(sid, remote, sock, connected, need_feedback)
        s = self.streams[sid]
        s.max_buf, s.produced = max_buf_size, 0

    def full(self, s):
        return s.max_buf > 0 and s.produced >= s.remote_consumed + s.max_buf

    def write(self, sid, payload, seg=0):
        """one StreamWrite -> (status, frames, produced, host_socket_id)"""
        s = self.streams.get(sid)
        if s is None or s.closed:
            return EINVAL, [], 0, 0
        if s.handed_over:
            return HANDED_OVER, [], s.produced, s.sock
        if self.full(s):
            return EAGAIN, [], s.produced, s.sock
        if not payload:
            return EINVAL, [], s.produced, s.sock           # (_produced += 0, then -= 0)
        if not s.connected:
            return NOT_CONNECTED, [], s.produced, s.sock
        if s.max_buf > 0:
            s.produced += len(payload)
        return 0, cut_frames(s.remote, sid, payload, seg), s.produced, s.sock

    def write_many(self, writes, seg=0):
        """writes: [(sid, payload)] in array order -> (results [dict], out bytes) laid out as b2_stream_write lays them out: each
        admitted write's frames contiguous at a 16-aligned offset, in array order"""
        results, out = [], bytearray()
        for sid, payload in writes:
            st, frames, produced, sock = self.write(sid, payload, seg)
            body = b"".join(frames)
            results.append({"status": st, "n_frames": len(frames), "out_off": len(out), "out_len": len(body), "produced": produced,
                            "host_socket_id": sock, "frames": frames})
            out += body + b"\0" * ((-len(body)) % 16)
        return results, bytes(out)

    def process(self, data, rs, msgs):
        """the receiving side, plus B2_STREAM_EV_WRITABLE: during a batch produced is constant and remote_consumed only grows, so the
        FEEDBACK frames of the batch took the stream from full to not full exactly when it was full before and is not after"""
        before = {sid: s.remote_consumed for sid, s in self.streams.items()}
        messages, events, rst = super().process(data, rs, msgs)
        for sid, ev in events.items():
            s = self.streams[sid]
            mb = getattr(s, "max_buf", 0)
            if mb > 0 and s.produced >= before[sid] + mb and s.produced < s.remote_consumed + mb:
                ev["flags"] |= EV_WRITABLE
        return messages, events, rst
