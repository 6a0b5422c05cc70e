from .TaskEnvironment import SpatialGoalEnvironment  # noqa: F401
from .ValueNeuron import ValueNeuron  # noqa: F401
from .SuccessorFeatures import SuccessorFeatures  # noqa: F401
from .PhasePrecessingPlaceCells import PhasePrecessingPlaceCells  # noqa: F401
from .SubAgent import (SubAgent, ThetaSequenceAgent, DumbAgent, ReplayAgent, ShiftAgent,  # noqa: F401
                       UnrelatedAgent)
from .PlaneWaveNeurons import PlaneWaveNeurons  # noqa: F401
from .NeuralNetworkNeurons import NeuralNetworkNeurons, MultiLayerPerceptron  # noqa: F401
