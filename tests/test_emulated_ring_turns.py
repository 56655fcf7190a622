"""CPU: tests/test_gpu_ring_turns.py, unchanged, on the emulated library (see tests/test_emulated_library.py): a baidu_std server's turn on
k_ring<RingBody::replies> — the runs as k_ring serves them, then the host replies packed as b2_pack_responses packs them in a phase over the
same CTA, the push into the slot, the overflow fallback and the refusals around a turn — equals the two batch calls turn for turn.  The
lanes of a warp and the threads of the CTA are host threads that the scheduler interleaves freely here, and device memory starts as 0xa5
bytes, so a phase that reads scratch the runs' phase wrote, or lacks a __syncthreads(), shows as wrong bytes."""
from test_emulated_library import run_files


def test_baidu_std_server_turns_on_the_ring_on_the_emulated_library():
    tail = run_files(["test_gpu_ring_turns.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
