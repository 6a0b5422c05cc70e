"""Float64 per-agent TD learner: a batch of A independent ValueNeurons (ValueNeuron(per_agent_weights=True)).  Row a of
every array is the reference's single-agent ValueNeuron (contribs/ValueNeuron.py:10-113) driven by agent a's inputs and
reward, so each row runs riab_oracle_td's functions with one agent, and with A = 1 this is riab_oracle_td itself.
Weights are (A, n, n_in) per input."""
import numpy as np

import riab_oracle_ffl as F
import riab_oracle_td as T


def td_rates_pa(W, inputs, biases, act, act_args=None, deriv=False):
    """The layer's rates (or phi') per agent: W list of (A, n, n_in_l), inputs list of (A, n_in_l) rows -> (A, n)."""
    A = W[0].shape[0] if W else np.asarray(inputs[0]).shape[0]
    return np.stack([F.ffl_get_state([(w[a], np.asarray(I, dtype=np.float64)[a]) for w, I in zip(W, inputs)],
                                     biases, act, act_args, deriv=deriv) for a in range(A)])


def td_learn_pa(W, traces, reward, fr, deriv, prime, dt, tau, eta, L2):
    """update_weights for every agent, each its own reference update.  W: list of (A, n, n_in_l) float64, updated in
    place; traces[l] (A, n_in_l); reward broadcasts to (A, n).  Returns td_error (A, n)."""
    fr = np.atleast_2d(np.asarray(fr, dtype=np.float64))
    A = fr.shape[0]
    reward = np.broadcast_to(np.asarray(reward, dtype=np.float64), fr.shape)
    deriv, prime = np.atleast_2d(deriv), np.atleast_2d(prime)
    td = np.empty_like(fr)
    for a in range(A):
        Wa = [w[a] for w in W]                          # views: T.td_learn's `w += dw` writes agent a's block
        td[a] = T.td_learn(Wa, [np.atleast_2d(e)[a] for e in traces], reward[a], fr[a], deriv[a], prime[a],
                           dt, tau, eta, L2)[0]
    return td


def td_apply_pa(W, traces, td, prime, dt, eta, L2):
    """The weight step of td_learn_pa from a given td_error (A, n): W[a] += (dt eta) outer(td_a phi'_a, e_a) -
    (eta dt L2) W[a], elementwise in the reference's order."""
    g = np.atleast_2d(np.asarray(td, dtype=np.float64)) * np.atleast_2d(np.asarray(prime, dtype=np.float64))
    for w, e in zip(W, traces):
        e = np.atleast_2d(np.asarray(e, dtype=np.float64))
        dw = dt * eta * (g[:, :, None] * e[:, None, :]) - eta * dt * L2 * w
        w += dw
