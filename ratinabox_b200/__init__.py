"""ratinabox_b200 -- H100-native batched step engine behind RatInABox's
Environment / Agent / Neurons API (hot path only; see DESIGN.md).

    from ratinabox_b200 import Environment, Agent, PlaceCells, GridCells, BoundaryVectorCells

Importing the package does not need a GPU; constructing an Agent does, and there
is no CPU fallback (the CUDA library must load).
"""
verbose = False

from .Environment import Environment          # noqa: E402
from .Agent import Agent                      # noqa: E402
from .Neurons import (Neurons, PlaceCells, GridCells, BoundaryVectorCells, FieldOfViewBVCs,   # noqa: E402
                      ObjectVectorCells, FieldOfViewOVCs, FeedForwardLayer, RandomSpatialNeurons,
                      HeadDirectionCells, VelocityCells, SpeedCell, AgentVectorCells, FieldOfViewAVCs)

__all__ = ["Environment", "Agent", "Neurons", "PlaceCells", "GridCells", "BoundaryVectorCells", "FieldOfViewBVCs",
           "ObjectVectorCells", "FieldOfViewOVCs", "FeedForwardLayer", "RandomSpatialNeurons", "HeadDirectionCells",
           "VelocityCells", "SpeedCell", "AgentVectorCells", "FieldOfViewAVCs"]
