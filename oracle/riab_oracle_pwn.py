"""Float64 restatement of PlaneWaveNeurons (ratinabox/contribs/PlaneWaveNeurons.py:10-91): the reference's draws
(:56-59) and get_state (:63-91), with utils.get_vectors_between (utils.py:203-215), in the reference's operation order."""
import numpy as np

DEFAULTS = {"n": 10, "wavescale": 0.2, "min_fr": 0, "max_fr": 1, "name": "PlaneWaveNeurons"}      # :25-31
PERIODIC_MESSAGE = "PlaneWaveNeurons not optimized for periodic environments, you may notice some discontinuities"   # :52-54


def draw(n, wavescale):
    """(phase_offsets (n,2), w (n,2), wavescales (n,)) from NumPy's global RNG, in the reference's order (:56-59)."""
    phase_offsets = np.random.uniform(0, wavescale, size=(n, 2))
    w = np.random.normal(size=(n, 2))
    w = w / np.expand_dims(np.linalg.norm(w, axis=1), axis=1)
    wavescales = np.random.rayleigh(scale=wavescale, size=n)
    return phase_offsets, w, wavescales


def get_state(pos, phase_offsets, w, wavescales, min_fr, max_fr):
    """(n, n_pos) rates at pos (n_pos, 2) (:76-91)."""
    pos = np.array(pos)
    pos = pos.reshape(-1, pos.shape[-1])
    po = np.asarray(phase_offsets)
    vecs = np.repeat(po.reshape(-1, 1, 2), pos.shape[0], axis=1) - np.repeat(pos.reshape(1, -1, 2), po.shape[0], axis=0)
    wt = np.tile(np.expand_dims(np.asarray(w), axis=1), reps=(1, pos.shape[0], 1))
    lam = np.tile(np.expand_dims(np.asarray(wavescales), axis=1), reps=(1, pos.shape[0]))
    phi_1 = ((2 * np.pi) / lam) * (vecs * wt).sum(axis=-1)
    firingrate = 0.5 * ((np.cos(phi_1)) + 1)
    return firingrate * (max_fr - min_fr) + min_fr
