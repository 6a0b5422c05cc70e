"""ratinabox.contribs.SuccessorFeatures (contribs/SuccessorFeatures.py:12-49) on the device: a ValueNeuron whose reward
is the firing rate of a feature population."""
from .ValueNeuron import ValueNeuron


class SuccessorFeatures(ValueNeuron):
    """ratinabox.contribs.SuccessorFeatures: ``n = features.n`` successor features learned by TD with the features'
    rates as the reward.  ``update_weights()`` reads the features' current rates on the device, so a batched learning
    loop needs no host synchronisation.  The batch semantics are ValueNeuron's (per-agent traces, derivatives and TD
    errors; one weight matrix learned from the mean over agents).  Like the reference, ``update()`` does not update the
    features or the input layers."""
    default_params = {                                              # contribs/SuccessorFeatures.py:27-29
        "features": None,
    }

    def __init__(self, Agent, params={}):
        params = dict(params)
        if params.get("features") is None:                          # :33-36
            raise Exception(
                "The input parameter dictionary must contain features to calculate the successor features for. params['features'] = ... This can be any RatInABox Neurons class (e.g. PlaceCells, BoundaryVectorCells, GridCells etc...or more complex things)."
            )
        params["n"] = params["features"].n
        super().__init__(Agent, params)

    def update_weights(self):
        super().update_weights(self.params["features"])
