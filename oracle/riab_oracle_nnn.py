"""Float64 NumPy restatement of the forward pass of the reference's NeuralNetworkNeurons (contribs/NeuralNetworkNeurons.py:
74-104) for a module that is a chain of Linear layers and elementwise activations, from a recorded ``state_dict``.  The
GPU tests compare the CUDA kernel against it; it is pinned to the live reference by tests/golden/nnn.npz
(oracle/gen_nnn_golden.py)."""
import numpy as np

ACTIVATIONS = {
    "identity": lambda x: x,
    "relu": lambda x: np.maximum(x, 0.0),
    "sigmoid": lambda x: 1.0 / (1.0 + np.exp(-x)),
    "tanh": np.tanh,
}


def chain_from_state_dict(state, acts):
    """[(W (out, in), b (out,) or None, activation name), ...] from a Sequential's state_dict (keys "<i>.weight" /
    "<i>.bias", with any prefix) and the activation after each Linear layer."""
    ws = sorted([k for k in state if k.endswith("weight")], key=lambda k: [int(p) if p.isdigit() else p for p in k.split(".")])
    assert len(ws) == len(acts), (ws, acts)
    out = []
    for k, a in zip(ws, acts):
        b = k[: -len("weight")] + "bias"
        out.append((np.asarray(state[k], dtype=np.float64), None if b not in state else np.asarray(state[b], dtype=np.float64), a))
    return out


def forward(X, chain):
    """The module on X (n_batch, n_in) in float64 -> (n_batch, n_out)."""
    h = np.asarray(X, dtype=np.float64)
    for W, b, a in chain:
        h = h @ W.T
        if b is not None:
            h = h + b
        h = ACTIVATIONS[a](h)
    return h


def get_state(inputs, chain):
    """NeuralNetworkNeurons.get_state: the inputs' rates (a list of (n_i, n_batch) arrays, the reference's get_state
    shape) concatenated and passed through the network -> (n_out, n_batch)."""
    return forward(np.concatenate(inputs).T, chain).T
