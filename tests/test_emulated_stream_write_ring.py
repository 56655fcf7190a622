"""CPU: tests/test_gpu_stream_write_ring.py, unchanged, on the emulated library (see tests/test_emulated_library.py):
k_ring<RingBody::stream_writes> — the runs and the stream pass as a stream-ring ticket serves them, then stream_write_block (the seven
phases of b2_stream_write over the same CTA), the push of the results and frames into the slot, the overflow path that serves the
writes on the grid kernels before it releases the kernel, and the refusals around a ticket — equals the two batch calls ticket for
ticket.  The lanes of a warp and the threads of the CTA are host threads that the scheduler interleaves freely here, and device memory
starts as 0xa5 bytes, so a phase that lacks a __syncthreads() or reads scratch a ticket did not clear shows as wrong bytes."""
from test_emulated_library import run_files


def test_stream_producer_turns_on_the_ring_on_the_emulated_library():
    tail = run_files(["test_gpu_stream_write_ring.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
