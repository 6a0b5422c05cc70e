"""Float64 NumPy restatement of the reference's ValueNeuron (contribs/ValueNeuron.py:10-113) and SuccessorFeatures
(contribs/SuccessorFeatures.py:12-49) learning rules, batched over agents.  Every expression repeats the reference's
operation order, so with one agent it reproduces the reference bit for bit (tests/golden/td.npz, written by
oracle/gen_td_golden.py); with A agents update_weights applies the mean over agents of every agent's reference update.
The layer's rates themselves come from riab_oracle_ffl (or are replayed from a recording)."""
import numpy as np


def td_derivative(fr, fr_last, dt):
    """firingrate_deriv (:66-71): (firingrate - firingrate_last) / dt, rows = agents."""
    return (np.asarray(fr, dtype=np.float64) - np.asarray(fr_last, dtype=np.float64)) / dt


def td_trace(e, I, dt, tau_e):
    """One eligibility-trace step (:72-81): dt I + (1 - dt / tau_e) e, I the input layer's firingrate after the update."""
    return dt * np.asarray(I, dtype=np.float64) + (1 - dt / tau_e) * np.asarray(e, dtype=np.float64)


def td_error(reward, fr, deriv, tau):
    """td_error (:92-94): reward + dV/dt - V / tau."""
    return reward + deriv - fr / tau


def td_learn(W, traces, reward, fr, deriv, prime, dt, tau, eta, L2):
    """update_weights (:83-104) over A agents (rows of fr, deriv, prime, traces[l]; reward broadcasts to (A, n)).
    W: list of (n, n_in_l) float64 weights, updated in place.  Returns td_error (A, n).
    dW_l = dt eta (sum_a outer(td_a phi'_a, e_{a,l}) / A) - eta dt L2 W_l; with A = 1 the sum is the reference's outer."""
    fr = np.atleast_2d(np.asarray(fr, dtype=np.float64))
    A = fr.shape[0]
    td = td_error(np.broadcast_to(np.asarray(reward, dtype=np.float64), fr.shape), fr,
                  np.atleast_2d(deriv), tau)
    g = td * np.atleast_2d(prime)
    for l, w in enumerate(W):
        e = np.atleast_2d(np.asarray(traces[l], dtype=np.float64))
        S = np.outer(g[0], e[0]) if A == 1 else g.T @ e
        dw = dt * eta * (S / A) - eta * dt * L2 * w
        w += dw
    return td


def td_learn_bound(traces, reward, fr, deriv, prime, tau):
    """|g| |e| averaged over agents: the scale of one learning step's contraction, (n, n_in) per input."""
    fr = np.atleast_2d(np.asarray(fr, dtype=np.float64))
    td = td_error(np.broadcast_to(np.asarray(reward, dtype=np.float64), fr.shape), fr, np.atleast_2d(deriv), tau)
    g = np.abs(td * np.atleast_2d(prime))
    return [g.T @ np.abs(np.atleast_2d(e)) / fr.shape[0] for e in traces]
