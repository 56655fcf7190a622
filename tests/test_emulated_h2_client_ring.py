"""CPU: tests/test_gpu_h2_client_ring.py, unchanged, on the emulated library (see tests/test_emulated_library.py): k_h2_client_ring — the
client parse and the request pack of the batch calls as block phases over one CTA, the push into the slot, the refusals and retirements
around a ticket — equals the two batch calls ticket for ticket.  The lanes of a warp and the threads of the CTA are host threads that the
scheduler interleaves freely here, so a phase that relies on convergence or lacks a __syncthreads() shows as wrong bytes."""
from test_emulated_library import run_files


def test_h2_client_connections_on_the_ring_on_the_emulated_library():
    tail = run_files(["test_gpu_h2_client_ring.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
