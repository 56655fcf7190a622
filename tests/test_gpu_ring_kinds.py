"""GPU: a context's first ring call fixes which resident kernel it runs, its ring kind:
  - batch: k_ring (b2_ring_start / b2_ring_submit);
  - batch with the stream pass: k_ring after b2_stream_ring_enable;
  - h2 server: k_h2_ring after b2_h2_ring_enable;
  - h2 client: k_h2_client_ring after b2_h2_client_ring_enable.
One context of each kind, with h2 and a stream table configured wherever the kind allows it, so that a refusal comes from the kind rule
and not from a missing prerequisite.  Every ring call of the other kinds, and every enable a second time, returns B2_E_INVAL, both while a
ticket of the context's own kind is outstanding and after it was collected.  After the refusals a ticket of the own kind still equals the
same ticket on a fresh twin context, and b2_ring_start returns B2_OK on every kind and leaves the next ticket served."""
import random

import pytest

import _h2serve as S
import _h2traffic as T
import test_gpu_h2_client_ring as HC
import test_gpu_h2_ring as HR
import test_gpu_stream_ring as SR
from _compare import assert_same
from _h2client_cases import OK_HDRS, frame, grpc_body, trailers
from _traffic import SEED, echo_frame
from test_gpu_h2_serve import WINDOW, call, prefix
from test_gpu_streams import F

pytestmark = pytest.mark.gpu
H2_CAPS = (1 << 20, 64, 1 << 20, 1 << 20)
H2C_CAPS = (1 << 20, 64, 1 << 20, 16, 1 << 20)


class Batch:
    """k_ring; a stream table would take the context off the plain ring, so it gets h2 only"""
    own = ("ring_submit", "ring_wait")

    def __init__(self):
        import brpc_b200 as b2
        self.b2, self.rng = b2, random.Random(SEED + 70)
        self.ring, self.twin = (b2.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=64) for _ in range(2))
        self.ring.h2_configure(8)
        self.ring.ring_start()

    def submit(self):
        data, runs = self.b2.make_runs([echo_frame(self.rng, i) for i in range(8)])
        t = self.ring.ring_submit(data, runs)
        return t, lambda: assert_same(self.ring.ring_wait(t), self.twin.process_batch(data, runs), "batch ticket %d" % t)

    def close(self):
        self.ring.ring_stop(); self.ring.close(); self.twin.close()


class BatchStreams:
    """k_ring with the stream pass (the pair of test_gpu_stream_ring.py), and h2"""
    own = ("ring_submit", "ring_wait")

    def __init__(self):
        import brpc_b200 as b2
        self.p = SR.Pair(b2, 16, 4096, 1 << 16)
        self.ring = self.p.ring
        self.ring.h2_configure(8)
        self.p.open([(1, 101, 0, True, True)])
        self.k = 0

    def submit(self):
        self.k += 1
        t, data, runs = self.p.submit([F(1, 5, data=b"kinds %d" % self.k)])
        return t, lambda: self.p.wait(t, data, runs, "streams ticket %d" % t)

    def close(self):
        self.p.close()


class H2Server:
    """k_h2_ring (the pair of test_gpu_h2_ring.py), and a stream table"""
    own = ("h2_ring_submit", "h2_ring_wait")

    def __init__(self):
        self.p = HR.Pair(2)
        self.ring = self.p.ring
        self.ring.stream_configure(16, 4096)
        self.enc = [T.HpackEncoder(random.Random(k)) for k in range(2)]
        self.sid = 1

    def submit(self):
        head = T.PREFACE + T.settings() + WINDOW if self.sid == 1 else b""
        chunks = [head + call(self.enc[k], self.sid, prefix(S.echo_request(b"kinds %d" % self.sid))) for k in range(2)]
        self.sid += 2
        data, runs, want = self.p.twin_batch(chunks)
        t = self.ring.h2_ring_submit(data, runs)
        return t, lambda: HR._same(self.ring.h2_ring_wait(t), want, 2, self.p.region(2), "h2 ticket %d" % t)

    def close(self):
        self.ring.ring_stop(); self.ring.close(); self.p.twin.close()


class H2Client:
    """k_h2_client_ring (the pair of test_gpu_h2_client_ring.py), and a stream table"""
    own = ("h2_client_ring_submit", "h2_client_ring_wait")

    def __init__(self):
        self.p = HC.Pair(range(2))
        self.ring = self.p.ring
        self.ring.stream_configure(16, 4096)
        self.sid = 0

    def submit(self):
        # the server's answer to the previous ticket's calls (none before the first), then one more call per connection
        s = self.sid
        chunks = {k: frame(1, 4, s, OK_HDRS) + frame(0, 0, s, grpc_body(b"ok")) + frame(1, 5, s, trailers()) for k in range(2)} if s else {}
        self.sid = s + 2 if s else 1
        data, runs, reqs, want = self.p.twin_ticket(chunks, [HC._call(k, b"kinds") for k in range(2)])
        t = self.ring.h2_client_ring_submit(data, runs, reqs)
        return t, lambda: self.p.check(self.ring.h2_client_ring_wait(t), data, want, "client ticket %d" % t)

    def close(self):
        self.ring.ring_stop(); self.p.close()


def ring_calls(ctx, ticket):
    """every ring call of every kind, with arguments each kind would accept"""
    import brpc_b200 as b2
    data, runs = b2.make_runs([echo_frame(random.Random(1), 0)])
    h2_data, h2_runs = b2.make_runs([T.PREFACE + T.settings()])
    c_data, c_runs, c_reqs = HC.ticket({}, [HC._call(0)])
    return {
        "ring_submit": lambda: ctx.ring_submit(data, runs),
        "ring_wait": lambda: ctx.ring_wait(ticket),
        "stream_ring_enable": lambda: ctx.stream_ring_enable(1 << 16),
        "h2_ring_enable": lambda: ctx.h2_ring_enable(*H2_CAPS),
        "h2_ring_submit": lambda: ctx.h2_ring_submit(h2_data, h2_runs),
        "h2_ring_wait": lambda: ctx.h2_ring_wait(ticket),
        "h2_client_ring_enable": lambda: ctx.h2_client_ring_enable(*H2C_CAPS),
        "h2_client_ring_submit": lambda: ctx.h2_client_ring_submit(c_data, c_runs, c_reqs),
        "h2_client_ring_wait": lambda: ctx.h2_client_ring_wait(ticket),
    }


def refusals(kind, ticket):
    """the return code of every call that is not the kind's own submit / wait"""
    from brpc_b200.abi import B2Error
    got = {}
    for name, fn in ring_calls(kind.ring, ticket).items():
        if name in kind.own:
            continue
        try:
            fn()
            got[name] = 0
        except B2Error as e:
            got[name] = e.code
    return got


@pytest.mark.parametrize("make", [Batch, BatchStreams, H2Server, H2Client], ids=lambda k: k.__name__)
def test_the_first_ring_call_fixes_the_kind(make):
    from brpc_b200.abi import B2_E_INVAL
    kind = make()
    t, check = kind.submit()
    first = refusals(kind, t)                                       # the own ticket outstanding
    assert first == {name: B2_E_INVAL for name in first}, first
    assert len(first) == 7
    check()
    after = refusals(kind, t)                                       # ... and collected
    assert after == first, after
    t, check = kind.submit()                                        # the own kind still serves, as on the twin
    check()
    kind.ring.ring_start()                                          # B2_OK on every kind: the context's own kernel
    t, check = kind.submit()
    check()
    kind.ring.ring_stop()
    kind.ring.ring_start()                                          # a relaunch after a stop
    t, check = kind.submit()
    check()
    if make is Batch:
        # with a stream table now, the enable is refused by the kind rule, and the plain ring because it runs no stream pass
        kind.ring.stream_configure(16, 4096)
        calls = ring_calls(kind.ring, t)
        assert _code(calls["stream_ring_enable"]) == B2_E_INVAL and _code(calls["ring_submit"]) == B2_E_INVAL
    kind.close()


def _code(fn):
    from brpc_b200.abi import B2Error
    with pytest.raises(B2Error) as e:
        fn()
    return e.value.code
