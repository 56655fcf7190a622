"""GPU: what a ring ticket overwrites on the device.  k_ring pulls every ticket's runs and bytes into the context's batch input (d_bytes,
d_meta) and serves it over the batch scratch, so b2_ring_submit ends what other calls left in those buffers:
  - the last h2 batch: b2_h2_pack_responses takes B2_H2_RESP_BODY_IN_INPUT bodies from it until a ring ticket comes between, and refuses
    them after;
  - the uploaded batch: b2_batch_execute runs it until a ring ticket comes between, and refuses it after."""
import random

import numpy as np
import pytest

import _h2serve as S
import _h2traffic as T
import _oracle as O
from _compare import assert_same
from _traffic import SEED, echo_frame, rnd62
from test_gpu_h2_serve import WINDOW, _ctx, call, prefix

pytestmark = pytest.mark.gpu
F_BODY_IN_INPUT = 16


def _err(fn, *a, **kw):
    from brpc_b200.abi import B2Error
    with pytest.raises(B2Error) as e:
        fn(*a, **kw)
    return e.value.code


def _replies(msgs, flags):
    """gRPC replies that echo each message's body, found at body_off = msg_off"""
    from brpc_b200.abi import H2_RESPONSE_DT
    r = np.zeros(len(msgs), H2_RESPONSE_DT)
    r["stream_id"] = msgs["stream_id"]; r["status_code"] = 200; r["flags"] = flags
    r["body_off"] = msgs["msg_off"]; r["body_len"] = msgs["msg_len"]
    return r


def test_a_ring_ticket_ends_the_last_h2_batch():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL
    rng = random.Random(SEED + 7)
    ctx, twin = _ctx(), _ctx()                  # the twin frames the same replies from host bytes
    for c in (ctx, twin):
        c.h2_conn_reset(0)
    enc = T.HpackEncoder(random.Random(1))
    msg = S.echo_request(b"zero-copy " * 50)

    def parse(sid, head=b""):
        """two calls to a host method on connection 0, parsed on both contexts"""
        data, runs = brpc_b200.make_runs([head + b"".join(call(enc, s, prefix(msg), path=b"/example.EchoService/Host") for s in (sid, sid + 2))])
        rs, msgs, _ = ctx.h2_process_batch(data, runs)
        assert msgs.tobytes() == twin.h2_process_batch(data, runs)[1].tobytes()
        assert len(msgs) == 2 and np.all(msgs["flags"] & F_BODY_IN_INPUT)
        return data, msgs

    # no ticket between: the bodies are read from the batch's input on the device
    data, msgs = parse(1, T.PREFACE + T.settings() + WINDOW)
    got = ctx.h2_pack_responses(None, _replies(msgs, 1 | 2))
    assert got == twin.h2_pack_responses(data, _replies(msgs, 1))
    assert all(msg in g for g in got)
    # a ring ticket between: it overwrote that input
    data, msgs = parse(5)
    frames = [echo_frame(rng, i, rnd62(rng, 256)) for i in range(8)]
    assert len(ctx.ring_wait(ctx.ring_submit(*brpc_b200.make_runs(frames)))[1]) == 8
    assert _err(ctx.h2_pack_responses, None, _replies(msgs, 1 | 2)) == B2_E_INVAL


def test_a_ring_ticket_ends_the_uploaded_batch():
    import brpc_b200
    from brpc_b200.abi import B2_E_INVAL
    rng = random.Random(SEED + 8)
    ctx = brpc_b200.Context(device=0, max_batch_bytes=8 << 20, max_msgs=1 << 14, max_runs=64)
    cfg = O.make_config()
    batch = [brpc_b200.make_runs([echo_frame(rng, i, rnd62(rng, 512)) for i in range(16)]) for _ in range(2)]
    # no ticket between: the uploaded batch runs
    ctx.upload(*batch[0])
    ctx.execute()
    assert_same(ctx.download(), O.process_batch(cfg, *batch[0]), "upload, execute")
    # a ring ticket between (of the same shape): it overwrote the uploaded runs and bytes
    ctx.upload(*batch[0])
    assert_same(ctx.ring_wait(ctx.ring_submit(*batch[1])), O.process_batch(cfg, *batch[1]), "the ticket")
    assert _err(ctx.execute) == B2_E_INVAL
    ctx.upload(*batch[0])
    ctx.execute()
    assert_same(ctx.download(), O.process_batch(cfg, *batch[0]), "uploaded again")
