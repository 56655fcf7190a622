"""CPU: tests/test_gpu_ring_device_state.py, unchanged, on the emulated library (see tests/test_emulated_library.py): a ring ticket ends
the last h2 batch's zero-copy sources and the uploaded batch, because k_ring overwrites the device buffers both live in."""
from test_emulated_library import run_files


def test_ring_device_state_on_the_emulated_library():
    tail = run_files(["test_gpu_ring_device_state.py"], 900)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
