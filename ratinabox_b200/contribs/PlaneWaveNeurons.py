"""ratinabox.contribs.PlaneWaveNeurons (contribs/PlaneWaveNeurons.py:10-91) on the device: neurons whose rate is a plane
wave over the environment, with a random orientation, wavelength and offset per cell -- the building block of grid-cell
models (a grid cell is three of them at 60 degrees)."""
import copy
import ctypes as C

import numpy as np

from .. import _lib
from ..Neurons import Neurons, _f64p


class PlaneWaveNeurons(Neurons):
    """ratinabox.contribs.PlaneWaveNeurons: ``rate_i = 0.5 (cos phi_i + 1) (max_fr - min_fr) + min_fr`` with
    ``phi_i = (2 pi / wavescales[i]) ((phase_offsets[i] - pos) . w[i])``, evaluated in the step kernel (riab_pwn_rates /
    RIAB_CELLS_PWN).  As in the reference, ``w``, ``phase_offsets`` and ``wavescales`` may be overwritten after
    construction (``w`` is used as stored, not renormalised), and ``min_fr`` / ``max_fr`` are read at every call; edits are
    re-packed before the next use.  ``wavescale`` matters only at construction.  A lone PlaneWaveNeurons population takes
    ``Agent.run``'s whole-run launch like PlaceCells and GridCells."""
    default_params = {                                              # contribs/PlaneWaveNeurons.py:25-31
        "n": 10,
        "wavescale": 0.2,
        "min_fr": 0,
        "max_fr": 1,
        "name": "PlaneWaveNeurons",
    }
    _cells_kind = _lib.CELLS_PWN
    _phase_form = -1              # riab_pwn_pack's phase_form: -1 lets the pack choose, 0 / 1 force radians / turns

    def __init__(self, Agent, params={}):
        p = copy.deepcopy(__class__.default_params)                 # :41-44
        p.update(params)
        super().__init__(Agent, p)
        assert self.Agent.Environment.dimensionality == "2D", "PlaneWaveNeurons only available in 2D"   # :47-49
        if self.Agent.Environment.boundary_conditions == "periodic":                                  # :51-54
            print("PlaneWaveNeurons not optimized for periodic environments, you may notice some discontinuities")
        self.phase_offsets = np.random.uniform(0, self.wavescale, size=(self.n, 2))                  # :56-59
        self.w = np.random.normal(size=(self.n, 2))
        self.w = self.w / np.expand_dims(np.linalg.norm(self.w, axis=1), axis=1)
        self.wavescales = np.random.rayleigh(scale=self.wavescale, size=self.n)

    def _signature(self):
        return (np.ascontiguousarray(self.phase_offsets, dtype=np.float64).tobytes(),
                np.ascontiguousarray(self.w, dtype=np.float64).tobytes(),
                np.ascontiguousarray(self.wavescales, dtype=np.float64).tobytes(),
                tuple(np.asarray(self.Agent.Environment.extent, dtype=np.float64).tolist()), float(self.min_fr),
                float(self.max_fr), int(self._phase_form))

    def _pack(self):
        env = self.Agent.Environment
        ph = np.ascontiguousarray(self.phase_offsets, dtype=np.float64).reshape(-1, 2)
        w = np.ascontiguousarray(self.w, dtype=np.float64).reshape(-1, 2)
        lam = np.ascontiguousarray(self.wavescales, dtype=np.float64).reshape(-1)
        self.n = lam.shape[0]
        assert ph.shape[0] == self.n and w.shape[0] == self.n, "phase_offsets, w and wavescales need one row per cell"
        c = _lib.PwnCells()
        host = np.zeros(self._lib.riab_pwn_pack_floats(self.n), dtype=np.float32)
        ext = np.ascontiguousarray(env.extent, dtype=np.float64)
        _lib.check(self._lib.riab_pwn_pack(_f64p(ph), _f64p(w), _f64p(lam), self.n, _f64p(ext), int(self._phase_form),
                                           C.byref(c), host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        c.n_cells = self.n
        c.min_fr, c.max_fr = float(self.min_fr), float(self.max_fr)
        c.packed_dev = self._packed.data_ptr()
        return c

    def _rates_from_positions(self, pos_dev, n_pos, out):
        ag = self.Agent
        _lib.check(self._lib.riab_pwn_rates(pos_dev.data_ptr(), n_pos, C.byref(ag._env_struct()), C.byref(self._cells()),
                                            out.data_ptr(), out.stride(0), ag._stream()))
