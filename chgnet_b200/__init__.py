"""chgnet_b200 — H100-native hot path for CHGNet (forward + force/stress backward)."""
from __future__ import annotations

from typing import Literal

PredTask = Literal["e", "ef", "em", "efs", "efsm"]

from chgnet_b200.graph import CrystalGraph  # noqa: E402

__all__ = ["PredTask", "CrystalGraph", "CHGNet"]


def __getattr__(name: str):
    if name == "CHGNet":
        from chgnet_b200.model import CHGNet

        return CHGNet
    raise AttributeError(name)
