"""CPU: tests/test_gpu_h2_ring_turns.py, unchanged, on the emulated library (see tests/test_emulated_library.py): a gRPC server's turn on
k_h2_ring — the serve passes, then the host replies packed as one more block phase, the push into the slot, the refusals and retirements
around a turn — equals b2_h2_serve_batch + b2_h2_pack_responses turn for turn.  The lanes of a warp and the threads of the CTA are host
threads that the scheduler interleaves freely here, so a phase that relies on convergence or lacks a __syncthreads() shows as wrong bytes."""
from test_emulated_library import run_files


def test_h2_server_turns_on_the_ring_on_the_emulated_library():
    tail = run_files(["test_gpu_h2_ring_turns.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
