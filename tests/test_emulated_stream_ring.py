"""CPU: tests/test_gpu_stream_ring.py, unchanged, on the emulated library (see tests/test_emulated_library.py): the stream pass inside
k_ring — stream_pass_block over one CTA, the slot's stream section, the park behind an overflowing ticket, the refusals while a ticket is
outstanding — equals the oracle and the batch path.  The lanes of a warp and the threads of the CTA are host threads that the scheduler
interleaves freely here, so a phase that relies on convergence or lacks a __syncthreads() shows as wrong bytes."""
from test_emulated_library import run_files


def test_stream_pass_on_the_ring_on_the_emulated_library():
    tail = run_files(["test_gpu_stream_ring.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
