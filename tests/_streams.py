"""Python oracle of the stream pass (b2_stream_*): the receiving side of brpc's Stream, restated sequentially and without capacities
(plus the one capacity rule the device adds), over _oracle.parse_stream_meta / pack_stream_frame.  Reference, function by function:
  ParseStreamingMessage  src/brpc/policy/streaming_rpc_protocol.cpp:99-129   Socket::Address(stream_id); unknown -> SendStreamRst (:139-149)
                                                                               unless FEEDBACK or no source_stream_id; a meta that fails
                                                                               to parse drops the frame (:101-104)
  Stream::OnReceived     src/brpc/stream.cpp:499-543    DATA -> _pending_buf, complete when has_continuation() is false; FEEDBACK ->
                                                        SetRemoteConsumed; RST -> Close(ECONNRESET); CLOSE -> Close(0); UNKNOWN ignored
  SetRemoteConsumed      :362-401   only moves forward (-socket_max_streams_unconsumed_bytes = 0: no _cur_buf_size bookkeeping)
  Stream::Consume        :582-651   _local_consumed += total length, SendFeedback when the peer asked for feedback
  SendFeedback           :653-662   {stream_id = remote, source_stream_id = id, FEEDBACK, feedback{consumed_size}}
  BeforeRecycle          :129-146   SendStreamClose of a connected stream: {stream_id = remote, source_stream_id = id, CLOSE}
  SetConnected           :270-307   a client-side stream sends its first FEEDBACK when it consumed bytes before
Decisions the reference leaves to scheduling, fixed here as the device fixes them: one Consume per stream per batch; a stream closed in a
batch still delivers what completed before the close and writes FEEDBACK before CLOSE; frames are taken in msgs[] order."""
import _oracle as O

RST, CLOSE, DATA, FEEDBACK = 1, 2, 3, 4
HAS_SOURCE, HAS_TYPE, HAS_CONT, HAS_FB, VAL_CONT = 2, 4, 8, 16, 256
ECONNRESET = 104
EV_MOVED, EV_RST, EV_CLOSE, EV_HANDED_OVER = 1, 2, 4, 8
MSG_STREAM_FRAME = 4


def feedback_frame(remote, sid, consumed):
    """pack_stream_frame has no feedback field: the FEEDBACK frame is built from the wire rules (field 5, Feedback{consumed_size = 1})."""
    def varint(v):
        v &= (1 << 64) - 1
        out = bytearray()
        while v >= 0x80:
            out.append((v & 0x7f) | 0x80); v >>= 7
        out.append(v)
        return bytes(out)
    fb = b"\x08" + varint(consumed)
    meta = b"\x08" + varint(remote) + b"\x10" + varint(sid) + b"\x18\x04" + b"\x2a" + varint(len(fb)) + fb
    n = len(meta).to_bytes(4, "big")
    return b"STRM" + n + n + meta


class Stream:
    def __init__(self, sid, remote, sock, connected, need_feedback):
        self.id, self.remote, self.sock, self.connected, self.need_feedback = sid, remote, sock, connected, need_feedback
        self.local_consumed = self.remote_consumed = 0
        self.pending, self.pending_frames = None, 0          # _pending_buf
        self.closed, self.error, self.handed_over = False, 0, False


class StreamOracle:
    def __init__(self, pending_bytes=None, out_bytes=None):
        self.streams = {}
        self.pending_bytes, self.out_bytes = pending_bytes, out_bytes

    def open(self, sid, remote=0, sock=0, connected=False, need_feedback=False):
        assert sid not in self.streams
        self.streams[sid] = Stream(sid, remote, sock, connected, need_feedback)

    def set_connected(self, sid, remote, need_feedback):
        s = self.streams[sid]
        if s.closed or s.connected:
            return b""
        s.remote, s.connected, s.need_feedback = remote, True, need_feedback
        return feedback_frame(remote, sid, s.local_consumed) if need_feedback and s.local_consumed > 0 else b""

    def close(self, sid):
        s = self.streams.pop(sid)
        return O.pack_stream_frame(s.remote, s.id, CLOSE) if s.connected and not s.closed else b""

    def process(self, data, rs, msgs):
        """data: the batch bytes; rs / msgs: the cut loop's run status and descriptors (the oracle's or the device's: they are equal).
        Returns (messages {sid: [(first_frame, n_frames, bytes)]}, events {sid: dict}, rst {run: bytes}).
        Streams do not interact, so the sequential walk over msgs[] is written as: who gets which frame, then each stream's frames in
        order (the capacity rule needs to see whether a message completes inside the batch), then the RST frames in msgs[] order."""
        data = bytes(data)
        frames, per_stream, wants_rst = {}, {}, set()
        for i, d in enumerate(msgs):
            if int(d["status"]) != MSG_STREAM_FRAME:
                continue             # (a meta that failed to parse is B2_MSG_BAD_STREAM_META: dropped, :101-104)
            fo, ms, bs = int(d["frame_off"]), int(d["meta_size"]), int(d["body_size"])
            ok, m = O.parse_stream_meta(data[fo + 12:fo + 12 + ms])
            assert ok
            ftype = m.frame_type if m.has & HAS_TYPE else 0
            frames[i] = (m, ftype, data[fo + 12 + ms:fo + 12 + bs], int(d["run_idx"]))
            s = self.streams.get(m.stream_id)
            if s is None or s.closed:
                wants_rst.add(i)
            elif not s.handed_over:      # (a handed-over stream is described per frame only)
                per_stream.setdefault(s.id, []).append(i)
        messages, events, out_used = {}, {}, 0
        for sid, idx in per_stream.items():
            s = self.streams[sid]
            done, flags, handover, consumed, k = [], 0, None, 0, 0
            while k < len(idx) and not s.closed and not s.handed_over:
                m, ftype, payload, _ = frames[idx[k]]
                if ftype == FEEDBACK:
                    c = m.consumed_size & ((1 << 64) - 1)
                    if c > s.remote_consumed:
                        s.remote_consumed = c; flags |= EV_MOVED
                    k += 1
                elif ftype in (RST, CLOSE):
                    s.closed, s.error = True, ECONNRESET if ftype == RST else 0
                    s.pending, s.pending_frames = None, 0
                    flags |= EV_RST if ftype == RST else EV_CLOSE
                    k += 1
                elif ftype == DATA:
                    # OnReceived frame by frame up to the end of the message, a close, or the end of the batch
                    parts, nfr, j, end = list(s.pending or []), s.pending_frames, k, None
                    while j < len(idx):
                        mj, fj, pj, _ = frames[idx[j]]
                        if fj in (RST, CLOSE):
                            break
                        if fj == FEEDBACK:
                            c = mj.consumed_size & ((1 << 64) - 1)
                            if c > s.remote_consumed:
                                s.remote_consumed = c; flags |= EV_MOVED
                        if fj == DATA:
                            parts.append(pj); nfr += 1
                            if not (mj.has & VAL_CONT):
                                end = j
                                break
                        j += 1
                    body = b"".join(parts)
                    if end is not None:
                        if nfr > 1 and self.out_bytes is not None:
                            need = (len(body) + 15) & ~15
                            if len(body) > self.out_bytes or out_used + need > self.out_bytes:
                                s.handed_over, handover = True, idx[k]
                                break
                            out_used += need
                        done.append((idx[k], nfr, body)); consumed += len(body)
                        s.pending, s.pending_frames = None, 0
                        k = end + 1
                    elif j < len(idx):
                        k = j                # the close drops the parts
                    else:
                        if self.pending_bytes is not None and len(body) > self.pending_bytes:
                            s.handed_over, handover = True, idx[k]
                            break
                        s.pending, s.pending_frames = parts, nfr
                        k = len(idx)
                else:
                    k += 1                   # FRAME_TYPE_UNKNOWN / absent / unknown enum value: ignored (:538-540)
            if s.closed:
                wants_rst.update(idx[k:])    # the id no longer resolves
            if s.handed_over:
                flags |= EV_HANDED_OVER
            s.local_consumed += consumed     # Consume, once
            messages[sid] = done
            events[sid] = {
                "flags": flags, "consumed": consumed, "local_consumed": s.local_consumed, "remote_consumed": s.remote_consumed,
                "n_msgs": len(done), "handover_msg": handover, "pending_bytes": sum(len(p) for p in s.pending) if s.pending else 0, "sock": s.sock,
                "fb": feedback_frame(s.remote, sid, s.local_consumed) if consumed > 0 and s.connected and s.need_feedback else b"",
                "close": O.pack_stream_frame(s.remote, sid, CLOSE) if s.closed and s.connected else b""}
        rst = {r: b"" for r in range(len(rs))}
        for i in sorted(wants_rst):
            m, ftype, _, run = frames[i]
            if (m.has & HAS_SOURCE) and ftype != FEEDBACK:
                rst[run] += O.pack_stream_frame(m.source_stream_id, -1, RST)
        return messages, events, rst

    def query(self, sid):
        s = self.streams[sid]
        return {"local_consumed": s.local_consumed, "remote_consumed": s.remote_consumed, "pending_bytes": sum(len(p) for p in s.pending) if s.pending else 0,
                "closed": s.closed, "handed_over": s.handed_over, "error_code": s.error}
