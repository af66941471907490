"""The index algebra of the row sweep's split with one read per mirror pair (tools/proto_r2c_sweep_order.py,
paired_split) against numpy.fft.rfft on the CPU: every bin of both rows of each pair emitted exactly once, the
self-paired rows 0 and P/2, own reads in half buffer A and mirror reads in B, whole 64-byte store pieces, and the
order of the per-group partial sums."""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import proto_r2c_sweep_order as proto  # noqa: E402


def test_paired_split_index_algebra():
    assert proto.main_paired_split(3) == 0
