"""CPU: tests/test_gpu_ring_kinds.py, unchanged, on the emulated library (see tests/test_emulated_library.py): the ring kind a context's
first ring call fixes, every cross-kind and repeated-enable call refused, and the own kind's tickets served as on a twin context."""
from test_emulated_library import run_files


def test_ring_kinds_on_the_emulated_library():
    tail = run_files(["test_gpu_ring_kinds.py"], 3000)
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail
