"""The reference's position-fix types (gypsum/world_model.py:71-94) and the conversion from a device fix record
(_native.FIX_DTYPE, TrackerBank.position_fixes)."""
from __future__ import annotations

from dataclasses import dataclass

from gypsum_b200 import _native


@dataclass
class EcefCoordinates:
    x: float
    y: float
    z: float

    def __hash__(self):
        return hash(self.x) + hash(self.y) + hash(self.z)

    def __str__(self):
        return f'({self.x=:.2f}, {self.y=:.2f}, {self.z=:.2f})'

    @classmethod
    def zero(cls) -> "EcefCoordinates":
        return cls(x=0, y=0, z=0)


@dataclass
class ReceiverSolution:
    clock_bias: float
    receiver_pos: EcefCoordinates


def solution_from_fix(record) -> ReceiverSolution:
    """The ReceiverSolution attempt_position_fix returns, from a FIX_DTYPE record of status 1 (FIX_SOLVED)."""
    if int(record["status"]) != _native.FIX_SOLVED:
        raise ValueError(f"fix record has status {int(record['status'])}, not {_native.FIX_SOLVED} (solved)")
    return ReceiverSolution(clock_bias=float(record["clock_bias"]),
                            receiver_pos=EcefCoordinates(float(record["x"]), float(record["y"]), float(record["z"])))
