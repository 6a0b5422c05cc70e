"""Float64 restatement of AgentVectorCells.get_state (ratinabox/Neurons.py:2204-2320): ObjectVectorCells.get_state
(riab_oracle.ovc_get_state) with the partner Agent's position as the single object and every cell tuned to its type.
``partner`` is one (2,) position for every row, or (N_pos, 2) with one partner per row (the batched pairing)."""
import numpy as np

import riab_oracle as O


def avc_get_state(env, partner, tuning, pos, rng, wall_geometry="line_of_sight", head_direction=None, min_fr=0.0,
                  max_fr=1.0):
    """(N_cells, N_pos).  ``tuning`` = (tuning_distances, tuning_angles, sigma_distances, sigma_angles); ``partner`` None
    gives the reference's zeros (:2231-2232, one column per position here); ``head_direction`` (2,) or (N_pos, 2) makes
    the cells egocentric."""
    td, ta, sd, sa = (np.asarray(x, dtype=float) for x in tuning)
    pos = np.asarray(pos, dtype=float).reshape(-1, 2)
    if partner is None:
        return np.zeros((len(td), len(pos)))
    partner = np.asarray(partner, dtype=float)
    one = lambda obj, p, hd: O.ovc_get_state(env, obj.reshape(1, 2), [0], td, ta, sd, sa, np.zeros(len(td), dtype=int), p,
                                             rng, wall_geometry, head_direction=hd, min_fr=min_fr, max_fr=max_fr)
    if partner.ndim == 1:
        return one(partner, pos, head_direction)
    hd = None if head_direction is None else np.broadcast_to(np.asarray(head_direction, dtype=float).reshape(-1, 2), pos.shape)
    return np.concatenate([one(partner[a], pos[a], None if hd is None else hd[a]) for a in range(len(pos))], axis=1)
