"""ratinabox.contribs.NeuralNetworkNeurons (contribs/NeuralNetworkNeurons.py:11-146) on the device: neurons whose rates are
a torch ``nn.Module`` applied to the concatenated firing rates of other populations of the same Agent, and the default
``MultiLayerPerceptron`` (a ReLU MLP with hidden layers [20, 20])."""
import copy
import ctypes as C
import warnings

import numpy as np
import torch
import torch.nn as nn

from .. import _lib
from ..Neurons import Neurons

_ACTIVATIONS = {nn.ReLU: "relu", nn.Sigmoid: "sigmoid", nn.Tanh: "tanh"}
# the reference's messages (contribs/NeuralNetworkNeurons.py:57-70)
DEFAULT_MLP_WARNING = ("No NeuralNetworkModule was provided so a default MLP with {n_in} inputs, {n} outputs and 2 hidden "
                       "ReLU layers of size 20 will be used. Alternatively provide one in the "
                       "params['NeuralNetworkModule']=<any-torch-nn.Module-with-a-.forward()-method> and don't set 'n'.")
BOTH_ERROR = ("You provided both 'n' and `NeuralNetworkModule` as parameters. These are mutually exclusive. Either provide "
              "'NeuralNetworkModule' and no 'n' (the output size of the NeuralNetworkModule will be used as the number of "
              "neurons in this layer) or 'n' and no 'NeuralNetworkModule (a default MLP will be initialised)")
NEITHER_ERROR = ("You provided neither a 'NeuralNetworkModule' nor 'n' as parameters. Either provide 'NeuralNetworkModule' "
                 "and no 'n' (the output size of the NeuralNetworkModule will be used as the number of neurons in this "
                 "layer) or 'n' and no 'NeuralNetworkModule (a default MLP will be initialised)")
PROBE_ERROR = ("You provided inputs layers with a total of {n_in} neurons but the NeuralNetworkModule you provided does not "
               "accept inputs of size (1,{n_in}) so they are incompatible")


class MultiLayerPerceptron(nn.Module):
    """ratinabox.contribs.NeuralNetworkNeurons.MultiLayerPerceptron (:126-146): Linear layers of sizes
    ``[n_in] + n_hidden + [n_out]`` with a ReLU after every hidden layer.  Built like the reference's, on the CPU, so
    that the same ``torch.manual_seed`` gives the same initial weights bit for bit."""

    def __init__(self, n_in=20, n_out=1, n_hidden=[20, 20]):
        nn.Module.__init__(self)
        n = [n_in] + n_hidden + [n_out]
        layers = nn.ModuleList()
        for i in range(len(n) - 1):
            layers.append(nn.Linear(n[i], n[i + 1]))
            if i < len(n) - 2:
                layers.append(nn.ReLU())
        self.net = nn.Sequential(*layers)

    def forward(self, X):
        return self.net(X)


def _linear_chain(module):
    """``([(nn.Linear, activation name), ...], None)`` when ``module`` is a chain of Linear layers and elementwise
    activations the fused kernel runs, else ``(None, reason)``."""
    mods = []

    def flatten(m):
        if m._forward_hooks or m._forward_pre_hooks:
            return False
        if type(m) is MultiLayerPerceptron:
            return flatten(m.net)
        if type(m) is nn.Sequential:
            return all(flatten(c) for c in m)
        mods.append(m)
        return True

    if not flatten(module):
        return None, "a module with forward hooks"
    chain = []
    for m in mods:
        if type(m) is nn.Identity:
            continue
        if type(m) is nn.Linear:
            if m.weight.dtype != torch.float32:
                return None, f"a Linear layer with {m.weight.dtype} weights"
            chain.append([m, "identity"])
        elif type(m) in _ACTIVATIONS and chain and chain[-1][1] == "identity":
            chain[-1][1] = _ACTIVATIONS[type(m)]
        elif type(m) in _ACTIVATIONS:
            return None, f"{type(m).__name__} " + ("before the first Linear layer" if not chain else "after another activation")
        else:
            return None, f"{type(m).__name__} is not a Linear layer or one of ReLU, Sigmoid, Tanh and Identity"
    if not chain:
        return None, "no Linear layer"
    if len(chain) > _lib.NNN_MAX_LAYERS:
        return None, f"{len(chain)} Linear layers (the kernel runs at most {_lib.NNN_MAX_LAYERS})"
    wide = [lin.out_features for lin, _ in chain[:-1] if lin.out_features > _lib.NNN_MAX_HIDDEN]
    if wide:
        return None, f"a hidden layer of width {wide[0]} (the kernel runs at most {_lib.NNN_MAX_HIDDEN})"
    return chain, None


class _FusedForward(torch.autograd.Function):
    """The fused kernel's rates as a node of the module's graph: the forward returns them, the backward re-runs the module
    in torch on the saved input rows and returns ``torch.autograd.grad`` of that (exact gradients of the torch forward)."""

    @staticmethod
    def forward(ctx, rates, X, module, *params):
        ctx.module = module
        ctx.save_for_backward(X, *params)
        return rates.clone()

    @staticmethod
    def backward(ctx, grad):
        X, *params = ctx.saved_tensors
        want = [p for p, need in zip(params, ctx.needs_input_grad[3:]) if need]
        with torch.enable_grad():
            out = ctx.module(X.detach())
            g = iter(torch.autograd.grad(out, want, grad, allow_unused=True))
        return (None, None, None) + tuple(next(g) if need else None for need in ctx.needs_input_grad[3:])


class NeuralNetworkNeurons(Neurons):
    """ratinabox.contribs.NeuralNetworkNeurons: ``firingrate = NeuralNetworkModule(concatenated input rates)``.

    The input layers must belong to this Agent; like a FeedForwardLayer's, an input registered before this population
    gives this step's rates, one registered after it the previous step's.  The module is moved to the Agent's device
    with ``.to()``, which modifies it in place, and its parameters must be float32.

    A module that is ``MultiLayerPerceptron`` or an ``nn.Sequential`` (nested or not) of ``nn.Linear`` layers and the
    elementwise ``ReLU``, ``Sigmoid``, ``Tanh`` and ``Identity`` runs as one fused kernel (``fused`` is True) within the
    limits of include/riab_b200.h (at most 8 Linear layers, hidden widths of at most 256, at most 4 input layers);
    ``Agent.run`` accepts it.  Any other module runs itself in torch on the gathered input rows (``fused`` is False), and
    ``Agent.run`` refuses it.  ``update()`` sets ``firingrate_torch``, the ``(n_agents, n)`` device tensor attached to the
    module's parameters (batch first, as in the reference), through which a loss can be back-propagated.  Weight edits
    (``opt.step()``, or assignments under ``torch.no_grad()``) are seen by the parameters' version counters and re-packed
    before the next evaluation; writes through ``.data`` bypass those counters and are not seen."""
    default_params = {                                              # contribs/NeuralNetworkNeurons.py:32-36
        "n": None,
        "input_layers": [],
        "NeuralNetworkModule": None,
        "name": "NeuralNetworkNeurons",
    }
    _cells_kind = _lib.CELLS_NNN

    def __init__(self, Agent, params={}):
        p = copy.deepcopy(__class__.default_params)                 # :38-43
        p.update(params)
        super().__init__(Agent, p)
        assert isinstance(self.input_layers, list), "param['input_layers'] must be a list of Neurons."
        assert len(self.input_layers) > 0, ("No input layers have been provided. Hand them in in the params dictionary "
                                            "params['input_layers']=[list,of,inputs]")
        for layer in self.input_layers:
            if layer.Agent is not self.Agent:
                raise ValueError("a NeuralNetworkNeurons' input layers must belong to its own Agent")
        self.n_in = sum([layer.n for layer in self.input_layers])
        if self.n is not None and self.NeuralNetworkModule is not None:                               # :59-63
            raise ValueError(BOTH_ERROR)
        if self.n is None and self.NeuralNetworkModule is None:
            raise ValueError(NEITHER_ERROR)
        if self.NeuralNetworkModule is None:                                                          # :55-57
            self.NeuralNetworkModule = MultiLayerPerceptron(n_in=self.n_in, n_out=self.n, n_hidden=[20, 20])
            warnings.warn(DEFAULT_MLP_WARNING.format(n_in=self.n_in, n=self.n))
        module = self.NeuralNetworkModule
        first = next(module.parameters(), None)
        try:                                                                                          # :66-70
            with torch.no_grad():
                y = module(torch.zeros(1, self.n_in, device=first.device if first is not None else "cpu"))
        except Exception:
            raise ValueError(PROBE_ERROR.format(n_in=self.n_in))
        if self.n is None:
            self.n = int(y.shape[1])
        bad = [name for name, t in list(module.named_parameters()) if t.dtype != torch.float32]
        if bad:
            raise TypeError(f"the NeuralNetworkModule's parameters must be float32 ({bad[0]} is not)")
        module.to(self.device)
        self._fused = False
        self._fused_reason = None
        self._n_packs = 0
        self._generic_rows = None
        self.firingrate_torch = None

    # ------------------------------------------------------------------ packing
    def _signature(self):
        m = self.NeuralNetworkModule
        return (id(m), tuple(id(layer) for layer in self.input_layers),
                tuple((t.data_ptr(), t._version) for t in m.parameters()))

    def _pack(self):
        self._n_packs += 1
        chain, reason = _linear_chain(self.NeuralNetworkModule)
        if chain is not None and len(self.input_layers) > _lib.FFL_MAX_INPUTS:
            chain, reason = None, f"{len(self.input_layers)} input layers (the kernel reads at most {_lib.FFL_MAX_INPUTS})"
        self._fused, self._fused_reason = chain is not None, reason
        c = _lib.NnnCells()
        if chain is None:
            c.n_cells, c.n_layers, c.n_inputs = self.n, 0, 1
            c.inputs[0].n_in = self.n
            return c
        c.n_layers, c.n_inputs = len(chain), len(self.input_layers)
        c.widths[0] = self.n_in
        blocks = []
        for l, (lin, act) in enumerate(chain):
            c.widths[l + 1], c.act[l] = lin.out_features, _lib.NNN_ACTIVATIONS[act]
            blocks.append(lin.weight.detach().reshape(-1))
            blocks.append(lin.bias.detach() if lin.bias is not None else torch.zeros(lin.out_features, device=self.device))
        params = torch.cat([b.to(device="cpu", dtype=torch.float64) for b in blocks]).numpy()
        for i, layer in enumerate(self.input_layers):
            c.inputs[i].n_in = layer.n
        host = np.zeros(self._lib.riab_nnn_pack_floats(C.byref(c)), dtype=np.float32)
        _lib.check(self._lib.riab_nnn_pack(params.ctypes.data_as(_lib.c_double_p), C.byref(c),
                                           host.ctypes.data_as(_lib.c_float_p)))
        self._packed = self._upload(host)
        c.packed_dev = self._packed.data_ptr()
        return c

    @property
    def fused(self):
        """Whether the module runs as the fused kernel (read-only; re-evaluated when the module or its weights change)."""
        self._cells()
        return self._fused

    # ------------------------------------------------------------------ input rows
    def _lag(self, layer):
        return 0 if layer._population_id < self._population_id else 1

    def _input_rows(self):
        """The rows each input gives now (its last row, None before its first update), bound like a FeedForwardLayer's."""
        out = []
        for layer in self.input_layers:
            if self._lag(layer):
                layer._ring_min = 2           # read one step late: its previous row must survive its next update
            out.append(None if layer._last_slot is None else layer._hist[layer._last_slot])
        return out

    def _gather(self, rows, n_pos):
        """(n_pos, n_in) float32: the input rows concatenated in list order (zeros for an input not yet updated)."""
        return torch.cat([r[:, : layer.n] if r is not None else
                          torch.zeros((n_pos, layer.n), dtype=torch.float32, device=self.device)
                          for layer, r in zip(self.input_layers, rows)], dim=1)

    def _cells(self):
        c = super()._cells()
        if not self._fused:
            g = self._generic_rows
            c.inputs[0].rows_dev, c.inputs[0].ld = (g.data_ptr() if g is not None else None), self.n
            return c
        for i, (layer, r) in enumerate(zip(self.input_layers, self._input_rows())):
            meta = c.inputs[i]
            meta.population, meta.lag = layer._population_id, self._lag(layer)
            meta.rows_dev, meta.ld = (r.data_ptr() if r is not None else None), layer._ld()
        return c

    def _reserve_history(self, n_more):
        self._input_rows()                    # Agent.run reserves every ring before binding rows: set the ring minimums
        super()._reserve_history(n_more)

    def _check_run(self):
        self._cells()
        if not self._fused:
            raise NotImplementedError(f"Agent.run runs a NeuralNetworkNeurons module only as the fused kernel, which does "
                                      f"not take this one ({self._fused_reason}): step with update() instead")

    def _cells_for_run(self):
        """Agent.run: the rows read one step late before the run's first step are snapshots (the run may overwrite the
        ring slot they sit in before this population reads them)."""
        c = self._cells()
        self._run_keep = []
        for i, layer in enumerate(self.input_layers):
            if c.inputs[i].lag == 1 and layer._last_slot is not None:
                snap = layer._hist[layer._last_slot].clone()
                self._run_keep.append(snap)
                c.inputs[i].rows_dev = snap.data_ptr()
        return c

    def _attached(self, rates, rows, n_pos):
        """firingrate_torch: ``rates`` (n_pos, n) as the module's output on the gathered ``rows``, attached to its
        parameters (the rows are gathered only when there is a graph to attach to)."""
        params = list(self.NeuralNetworkModule.parameters())
        if torch.is_grad_enabled() and any(p.requires_grad for p in params):
            return _FusedForward.apply(rates, self._gather(rows, n_pos), self.NeuralNetworkModule, *params)
        return rates.clone()

    def _fused_rates(self, c, rows, n_pos):
        """The fused kernel on `rows` (one per input, (n_pos, ld) float32 or None) -> (n_pos, ld) float32, no noise."""
        fc = _lib.NnnCells.from_buffer_copy(c)
        for i, r in enumerate(rows):
            fc.inputs[i].rows_dev = r.data_ptr() if r is not None else None
            fc.inputs[i].ld = r.stride(0) if r is not None else self.input_layers[i]._ld()
        out = torch.empty((n_pos, self._ld()), dtype=torch.float32, device=self.device)
        ro = _lib.RatesOut()
        ro.rates_row, ro.ld = out.data_ptr(), self._ld()
        _lib.check(self._lib.riab_nnn_rates(C.byref(fc), n_pos, None, None, C.byref(ro), self.Agent._stream()))
        return out

    # ------------------------------------------------------------------ update / get_state
    def update(self, **kwargs):
        """NeuralNetworkNeurons.update (:107-109): the module on the inputs' current rows, OU noise and spikes into this
        population's ring row, and ``firingrate_torch`` set."""
        self._cells()
        rows = self._input_rows()
        A = self.Agent.n_agents
        if not self._fused:
            Y = self.NeuralNetworkModule(self._gather(rows, A))
            self._generic_rows = Y.detach().to(torch.float32).contiguous()
            super().update(**kwargs)
            self.firingrate_torch = Y
            return
        super().update(**kwargs)
        if self.noise_std != 0:               # the ring row holds the rates plus noise: firingrate_torch is the module's
            rates = self._fused_rates(self._cells(), rows, A)[:, : self.n]
        else:
            rates = self._hist[self._last_slot][:, : self.n]
        self.firingrate_torch = self._attached(rates, rows, A)

    def get_state(self, evaluate_at="last", save_torch=False, **kwargs):
        """NeuralNetworkNeurons.get_state (:74-104): "last" reads the inputs' current rows; anything else evaluates the
        inputs with ``get_state(evaluate_at, **kwargs)`` on the device first.  Returns (n, n_pos) float64 (the reference's
        shape), or with ``return_tensor=True`` the (n_pos, n) float32 device tensor.  ``save_torch=True`` sets
        ``firingrate_torch`` from this evaluation."""
        return_tensor = kwargs.pop("return_tensor", False)
        kwargs.pop("max_recurrence", None)
        c = self._cells()
        if evaluate_at == "last":
            self.Agent._flush_pending()
            rows, n_pos = self._input_rows(), self.Agent.n_agents
        else:
            rows = []
            for layer in self.input_layers:
                I = layer.get_state(evaluate_at, return_tensor=True, **kwargs)
                if I.dtype != torch.float32 or I.stride(1) != 1 or I.stride(0) % 4 or I.data_ptr() % 16:
                    J = torch.zeros((I.shape[0], (I.shape[1] + 3) // 4 * 4), dtype=torch.float32, device=self.device)
                    J[:, : I.shape[1]] = I
                    I = J
                rows.append(I)
            n_pos = int(rows[0].shape[0])
        if self._fused:
            rates = self._fused_rates(c, rows, n_pos)[:, : self.n]
            if save_torch:
                self.firingrate_torch = self._attached(rates, rows, n_pos)
        else:
            with torch.set_grad_enabled(torch.is_grad_enabled() and save_torch):
                Y = self.NeuralNetworkModule(self._gather(rows, n_pos))
            if save_torch:
                self.firingrate_torch = Y
            rates = Y.detach()
        if return_tensor:
            return rates
        return rates.T.contiguous().cpu().numpy().astype(np.float64)
