"""Float64 NumPy restatement of the reference's FeedForwardLayer (ratinabox/Neurons.py:2654-2847) and of the premade
activations of utils.activate (ratinabox/utils.py:919-1026).  The GPU tests compare the CUDA layer against it; it is
pinned to the live reference by tests/golden/ffl.npz (oracle/gen_ffl_golden.py)."""
import numpy as np


def activate(x, name, deriv=False, args=None):
    """utils.activate(x, activation=name, deriv, other_args=args) for the premade set (utils.py:919-1026)."""
    args = dict(args or {})
    assert name in ("linear", "sigmoid", "relu", "tanh", "retanh", "softmax")
    x = np.asarray(x, dtype=np.float64)
    if name == "linear":                                            # utils.py:955-959
        return np.ones(x.shape) if deriv else x
    if name == "sigmoid":                                           # utils.py:961-979
        a = {"max_fr": 1, "min_fr": 0, "mid_x": 1, "width_x": 2}
        a.update(args)
        max_fr, min_fr, width_x, mid_x = a["max_fr"], a["min_fr"], a["width_x"], a["mid_x"]
        beta = np.log((1 - 0.05) / 0.05) / (0.5 * width_x)
        f = ((max_fr - min_fr) / (1 + np.exp(-beta * (x - mid_x)))) + min_fr
        if not deriv:
            return f
        return beta * (f - min_fr) * (1 - (f - min_fr) / (max_fr - min_fr))
    a = {"gain": 1, "threshold": 0}
    a.update(args)
    g, th = a["gain"], a["threshold"]
    if name == "relu":                                              # utils.py:981-989
        return g * ((x - th) > 0) if deriv else g * np.maximum(0, x - th)
    if name == "tanh":                                              # utils.py:991-999: the derivative ignores the threshold
        return g * (1 - np.tanh(x) ** 2) if deriv else g * np.tanh(x - th)
    if name == "retanh":                                            # utils.py:1001-1015
        return g * (1 - np.tanh(x) ** 2) * ((x - th) > 0) if deriv else g * np.maximum(0, np.tanh(x - th))
    # "softmax" is a softplus (utils.py:1017-1026)
    return g / (1 + np.exp(-(x - th))) if deriv else g * np.log(1 + np.exp(x - th))


def activation_lipschitz(name, args=None):
    """An upper bound of |phi'| (and of |phi''| for the derivatives' error budget) of the premade activations."""
    args = dict(args or {})
    if name == "linear":
        return 1.0
    if name == "sigmoid":
        a = {"max_fr": 1, "min_fr": 0, "mid_x": 1, "width_x": 2}
        a.update(args)
        beta = np.log((1 - 0.05) / 0.05) / (0.5 * a["width_x"])
        return abs(beta) * abs(a["max_fr"] - a["min_fr"]) * 0.25 + abs(beta) ** 2 * abs(a["max_fr"] - a["min_fr"]) * 0.1
    g = abs(dict({"gain": 1}, **args)["gain"])
    return g if name in ("relu", "softmax") else 2 * g     # tanh'' <= 0.77


def ffl_get_state(inputs, biases, name, args=None, deriv=False):
    """FeedForwardLayer.get_state (Neurons.py:2797-2847) once the inputs' rates are known: V = sum_l w_l @ I_l + b, in
    the reference's order (np.matmul per layer, accumulated into zeros, then the biases), then phi(V) or phi'(V).
    inputs: [(w (n, n_in), I (n_in,) or (n_in, n_pos)), ...]."""
    n = np.asarray(biases).shape[0]
    shape = (n,) if np.asarray(inputs[0][1]).ndim == 1 else (n, np.asarray(inputs[0][1]).shape[1]) if inputs else (n,)
    V = np.zeros(shape)
    for w, I in inputs:
        V += np.matmul(w, I)
    b = np.asarray(biases, dtype=np.float64)
    if b.shape != V.shape:
        b = b.reshape((-1, 1))
    V += b
    return activate(V, name, deriv, args)
