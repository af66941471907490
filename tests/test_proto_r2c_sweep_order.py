"""The index algebra of the sweep-order R2C route (tools/proto_r2c_sweep_order.py) against numpy on the CPU."""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import proto_r2c_sweep_order as proto  # noqa: E402


def test_sweep_order_index_algebra():
    assert proto.main(["proto", "5", "6"]) == 0
