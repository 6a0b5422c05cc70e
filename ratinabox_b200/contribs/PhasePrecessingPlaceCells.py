"""ratinabox.contribs.PhasePrecessingPlaceCells (contribs/PhasePrecessingPlaceCells.py:10-119) on the device: place cells
whose rate at the agent is modulated by a von Mises in theta phase that precesses as the agent crosses the field (George et
al. 2023, "Rapid learning of predictive maps with STDP and theta phase precession")."""
import copy
import ctypes as C

import numpy as np

from .. import _lib
from ..Neurons import PlaceCells


class PhasePrecessingPlaceCells(PlaceCells):
    """ratinabox.contribs.PhasePrecessingPlaceCells: ``get_state()`` at the agents is the PlaceCells rate times
    ``theta_modulation_factors()``, evaluated in the step kernel (riab_pppc_rates / RIAB_CELLS_PPPC) from each agent's
    position, ``Agent.velocity`` and ``Agent.t``.  Elsewhere (``"all"``, ``pos=``) the rates are the unmodulated PlaceCells
    rates, with the reference's message.  As in the reference the factor reads ``sigma`` (set once from ``kappa``), and
    ``theta_freq``, ``precess_fraction``, ``place_cell_widths`` and ``place_cell_centres`` on every call; the rates are not
    bounded by ``max_fr``."""
    default_params = {                                              # contribs/PhasePrecessingPlaceCells.py:33-42
        "n": 10,
        "min_fr": 0,
        "max_fr": 1,
        "theta_freq": 10,
        "kappa": 1,
        "precess_fraction": 0.5,
        "description": "gaussian_threshold",
        "name": "PhasePrecessingPlaceCell",
    }
    _cells_kind = _lib.CELLS_PPPC

    def __init__(self, Agent, params={}):
        p = copy.deepcopy(__class__.default_params)                 # :52-55
        p.update(params)
        super().__init__(Agent, p)
        self.sigma = np.sqrt(1 / self.kappa)                         # :56
        assert self.description in [                                # :58-63
            "gaussian",
            "diff_of_gaussians",
            "gaussian_threshold",
            "top_hat",
        ]

    def _signature(self):
        return super()._signature() + (float(self.theta_freq), float(self.sigma), float(self.precess_fraction))

    def _pack(self):
        c = _lib.PppcCells()
        c.place = super()._pack()
        c.theta_freq, c.sigma, c.precess_fraction = float(self.theta_freq), float(self.sigma), float(self.precess_fraction)
        return c

    def _cells(self):
        """The packed struct at the Agent's current clock (riab_run: the first step's; the library advances it)."""
        c = super()._cells()
        c.t = float(self.Agent.t)
        return c

    def get_state(self, evaluate_at="agent", **kwargs):
        """The PlaceCells rates, times the theta modulation factors at the agents (:66-92)."""
        firingrate = super().get_state(evaluate_at, **kwargs)
        if evaluate_at != "agent":
            print(
                "Since you are not evaluating hte firing rate using the current state of the agent no phase precession modulation has been applied (since this requires a velocity). Ignore this if you are plotting receptive field. "
            )
        return firingrate

    def _kernel_inputs(self, evaluate_at, n_pos, kwargs):
        return {"velocity": self.Agent._s["velocity"]} if evaluate_at == "agent" else {}

    def _rates_from_positions(self, pos_dev, n_pos, out, velocity=None):
        ag = self.Agent
        cells = self._cells()
        if velocity is None:                                        # away from the agents: the PlaceCells rates
            _lib.check(self._lib.riab_place_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()), C.byref(cells.place),
                                                  out.data_ptr(), out.stride(0), ag._stream()))
            return
        _lib.check(self._lib.riab_pppc_rates(pos_dev.data_ptr(), velocity.data_ptr(), n_pos, C.byref(ag._env_struct()),
                                             C.byref(cells), out.data_ptr(), out.stride(0), ag._stream()))

    def theta_modulation_factors(self):
        """(n, n_agents) float64 factors (n_agents = 1: (n, 1)), the reference's expression (:94-119) evaluated with torch
        in float64 on the device from the agents' current state (np.i0 gives the normalisation)."""
        torch = self._torch
        s = self._agent_state()
        pos, vel = s["pos"], s["velocity"]
        direction = vel / (1e-8 + torch.linalg.norm(vel, dim=1, keepdim=True))
        theta_phase = self.theta_freq * (self.Agent.t % (1 / self.theta_freq)) * 2 * np.pi
        sigma = np.array(self.place_cell_widths, dtype=np.float64).copy()
        if self.description == "gaussian":
            sigma *= 2
        centres = torch.as_tensor(np.asarray(self.place_cell_centres, dtype=np.float64).reshape(-1, 2), device=self.device)
        vectors_to_cells = pos[:, None, :] - centres[None, :, :]                  # get_vectors_between(pos, centres)
        sigmas_to_cell_midline = (vectors_to_cells * direction[:, None, :]).sum(-1) / torch.as_tensor(sigma, device=self.device)
        prefered_theta_phase = np.pi - sigmas_to_cell_midline * self.precess_fraction * np.pi
        phase_diff = prefered_theta_phase - theta_phase
        kappa = 1 / (self.sigma ** 2)                                             # utils.von_mises (utils.py:452-456)
        norm = np.exp(kappa) / (2 * np.pi * np.i0(kappa))
        norm = norm / np.exp(kappa)
        v = torch.exp(kappa * torch.cos(phase_diff)) * norm
        return (v * 2 * np.pi).T.contiguous().cpu().numpy()
