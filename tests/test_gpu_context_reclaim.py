"""GPU: a Context that the cyclic garbage collector reclaims is destroyed at the next safe point (the next Context creation, close() or
exit), not inside the collection.  b2_ctx_destroy waits for the whole device: destroyed inside a collection that runs while another
context's resident ring kernel polls, it would block the collecting thread until that kernel idles out (B2_RING_IDLE_MS) and cost the
kernel a relaunch."""
import gc
import time

import pytest

pytestmark = pytest.mark.gpu


def _ctx():
    import brpc_b200
    return brpc_b200.Context(device=0, max_batch_bytes=1 << 20, max_msgs=1 << 12, max_runs=64, max_resp_bytes=1 << 20)


def test_a_context_the_collector_reclaims_is_destroyed_at_the_next_safe_point(monkeypatch):
    from brpc_b200 import abi
    monkeypatch.setenv("B2_RING_IDLE_MS", "3000")
    gc.collect()
    a = _ctx()
    a.ring_start()
    n0 = a.ring_launches()
    b = _ctx()
    b.cycle = b                                                      # reachable only through itself: only the collector frees it
    del b
    t0 = time.perf_counter()
    gc.collect()
    took = time.perf_counter() - t0
    assert len(abi._reclaimed) == 1 and took < 1.0, took
    a.ring_start()                                                   # still resident: nothing to relaunch
    assert a.ring_launches() == n0
    a.ring_stop()
    c = _ctx()                                                       # the next creation destroys what the collector reclaimed
    assert abi._reclaimed == []
    a.close(); c.close()
