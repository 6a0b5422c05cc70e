"""ratinabox.contribs.ValueNeuron (contribs/ValueNeuron.py:10-113) on the device: TD learning of a value function on a
FeedForwardLayer, with per-agent eligibility traces and one weight matrix shared by the batch, or with
``per_agent_weights`` one independent learner per agent."""
import ctypes as C

import numpy as np

from .. import _lib
from ..Neurons import FeedForwardLayer, Neurons, _FflInput, _f64p


class _TdInput(_FflInput):
    """One entry of ``ValueNeuron.inputs``.  ``"w"`` is a host copy of the layer's float64 device master, made when read;
    in-place edits of it and assignments are uploaded before the master is next used.  ``"eligibility_trace"`` is a
    host copy of the device trace, ``(n_in,)`` for one agent, else ``(n_agents, n_in)``; like the reference, only the
    inputs present at construction have one."""

    def __init__(self, owner, name, entry):
        dict.__init__(self, entry)
        self._owner, self._name = owner, name

    def __getitem__(self, k):
        if k == "w":
            return self._owner._w_read(self._name, dict.__getitem__(self, "w"))
        if k == "eligibility_trace":
            dict.__getitem__(self, k)                   # KeyError for an input added after construction
            return self._owner._trace_read(self._name)
        return _FflInput.__getitem__(self, k)

    def __setitem__(self, k, v):
        if k == "w":
            self._owner._w_assign(self._name, v)
        elif k == "eligibility_trace":
            self._owner._trace_assign(self._name, v)
        dict.__setitem__(self, k, v)


class _BatchLearning:
    """The batch engine's ValueNeuron param, collected with the defaults like every class's ``default_params`` but kept
    apart from ``ValueNeuron.default_params``, which stay the reference's.

    ``per_agent_weights``: False (default) -- one weight matrix per input shared by the batch, learned from the mean of
    the agents' updates; True -- every agent is an independent learner with its own weights (see ValueNeuron)."""
    default_params = {"per_agent_weights": False}


class ValueNeuron(FeedForwardLayer, _BatchLearning):
    """ratinabox.contribs.ValueNeuron: ``n`` value functions V = phi(sum_l w_l . I_l + b) learned by continuous TD,

        update():          firingrate_deriv = (firingrate - firingrate_last) / dt,  e_l <- dt I_l + (1 - dt / tau_e) e_l
        update_weights(r): td_error = r + firingrate_deriv - firingrate / tau
                           w_l += dt eta outer(td_error * firingrate_prime, e_l) - eta dt L2 w_l

    With ``n_agents == 1`` this is the reference class.  With a batch of agents:

    * ``firingrate``, ``firingrate_deriv``, ``td_error`` (each ``(n_agents, n)``) and the eligibility traces
      (``inputs[name]["eligibility_trace"]``, ``(n_agents, n_in)``) are per agent and independent across agents;
    * the weights are the layer's single ``(n, n_in)`` matrices, and ``update_weights`` applies the MEAN over agents
      of every agent's reference update, ``dw = dt eta / A sum_a outer(td_a phi'_a, e_a) - eta dt L2 w``;
    * ``reward`` may be a scalar, ``(n,)`` (every agent), ``(n_agents, n)``, ``(n_agents,)`` when ``n == 1``, a torch
      tensor of those shapes on the device (read there, no host copy), or a population of the same Agent with ``n``
      cells, whose current rates are read on the device -- a learning loop without host synchronisation;
    * ``reset(agents=None)`` also takes an index array or a boolean mask and resets only those agents.

    The weights are kept in float64 on the device (the L2 decay moves a weight by ~5e-8 of itself per step at the
    demo's values, under float32's half ulp) and re-split into the layer's error-compensated TF32 operands after each
    learning step.  ``Agent.run`` runs ``update()`` (rates, derivative, traces) but never ``update_weights``.

    With ``params["per_agent_weights"] = True`` agent ``a`` of the batch IS the reference's single-agent ValueNeuron
    driven by its own inputs and reward:

    * every input's weights are ``(n_agents, n, n_in)`` float64 on the device (``8 n_agents sum n n_in`` bytes, checked
      against the free device memory before anything is allocated: ``MemoryError``).  Construction draws the reference's
      ``(n, n_in)`` weights and gives every agent a copy; ``inputs[name]["w"]`` reads ``(n_agents, n, n_in)`` (``(n,
      n_in)`` for one agent) and takes ``(n, n_in)`` (every agent) or ``(n_agents, n, n_in)``;
    * the rates contract each agent's own weights with its inputs in float64 (csrc/riab_td.cuh, k_td_forward_pa);
    * ``update_weights`` applies each agent's own reference update, nothing averaged, with the same reward forms;
    * ``get_state(evaluate_at="all" | None, pos=...)`` gives ``(n_agents, n, n_pos)`` (``(n, n_pos)`` for one agent), and
      ``agents=[...]`` picks the learners evaluated: ``(len(agents), n, n_pos)``.  At "last" / "agent" each agent's
      row uses its own weights, ``(n, n_agents)`` as for shared weights, and firingrate_prime is not refreshed."""
    default_params = {                                              # contribs/ValueNeuron.py:36-43
        "tau": 2,
        "tau_e": None,
        "eta": 0.001,
        "L2": 0.001,
        "activation_function": {"activation": "relu"},
        "n": 1,
    }
    _cells_kind = _lib.CELLS_TD

    def __init__(self, Agent, params={}):
        self._master = {}           # name -> (n, n_in) float64 device master
        self._w_pack = {}           # name -> W_hi | W_lo device block (riab_ffl_pack layout)
        self._w_shadow = {}         # name -> [host array handed out, snapshot at hand-out or None after an assignment]
        self._trace = {}            # name -> (A, ld_in) float32 device trace
        self._fr_prev = self._deriv = self._td = None
        self._scratch = None
        self._reward_keep = None
        self._pa = bool(dict(params).get("per_agent_weights", False))
        if self._pa:
            n = int(dict(params).get("n", ValueNeuron.default_params["n"]))
            self._check_memory(Agent, 8 * Agent.n_agents * n * sum(l.n for l in dict(params).get("input_layers", [])))
        super().__init__(Agent, params)
        if self.tau_e is None:                                      # :50-51
            self.tau_e = self.tau / 4
        for e in self.inputs.values():
            dict.__setitem__(e, "eligibility_trace", None)          # :52-53: the inputs present now get a trace

    def add_input(self, input_layer, w=None, w_init_scale=1, recurrent=False, **kwargs):
        if self._pa and input_layer.name not in getattr(self, "inputs", {}):
            others = sum(e["layer"].n for e in getattr(self, "inputs", {}).values())
            self._check_memory(self.Agent, 8 * self.Agent.n_agents * self.n * (others + input_layer.n))
        super().add_input(input_layer, w=w, w_init_scale=w_init_scale, recurrent=recurrent, **kwargs)
        name = input_layer.name
        for d in (self._master, self._w_pack, self._w_shadow, self._trace):
            d.pop(name, None)
        self.inputs[name] = _TdInput(self, name, self.inputs[name])

    @staticmethod
    def _check_memory(Agent, need):
        """Refuse per-agent weights that would not fit in the device's free memory, before allocating them."""
        import torch
        if need <= 0 or Agent.device.type != "cuda":
            return
        free, _ = torch.cuda.mem_get_info(Agent.device)
        if need > free:
            raise MemoryError(f"per-agent weights need {need} bytes ({need / 1e9:.1f} GB) of device memory for "
                              f"{Agent.n_agents} agents; {free} bytes are free")

    # ------------------------------------------------------------------ weights
    def _signature(self):
        # the weights live on the device: only the structure and the biases are compared per step
        sig = [self.n, repr(self.activation_function), np.ascontiguousarray(self.biases, dtype=np.float64).tobytes()]
        for name, e in self.inputs.items():
            sig += [name, id(e["layer"]), e["layer"].n, id(e)]
        return tuple(sig)

    def _pack(self):
        act, prm = self._activation()
        c = _lib.TdCells()
        f = c.ffl
        f.n_cells, f.activation = self.n, act
        for i in range(4):
            f.act[i] = prm[i]
        b = np.ascontiguousarray(self.biases, dtype=np.float64).reshape(-1)
        assert b.shape[0] == self.n, f"biases must have shape ({self.n},)"
        self._bias_dev = self._upload(b.astype(np.float32))
        f.bias_dev = self._bias_dev.data_ptr()
        for i, (name, e) in enumerate(self.inputs.items()):
            n_in = e["layer"].n
            if self._pa:
                if name not in self._master:
                    self._master[name] = self._upload(self._w_full(name, dict.__getitem__(e, "w")))
                f.inputs[i].n_in, f.inputs[i].k_pad = n_in, (n_in + 31) // 32 * 32
                f.inputs[i].w_dev = None                            # the per-agent contraction reads the masters
                continue
            if name not in self._master:
                w = np.ascontiguousarray(dict.__getitem__(e, "w"), dtype=np.float64)
                assert w.shape == (self.n, n_in), f"inputs[{name!r}]['w'] must have shape ({self.n}, {n_in})"
                self._master[name] = self._upload(w)
                self._w_pack[name] = self._upload(self._split(w, f.inputs[i]))
            else:
                self._split(np.zeros((self.n, n_in)), f.inputs[i])     # fills n_in / k_pad; the block is kept
            f.inputs[i].w_dev = self._w_pack[name].data_ptr()
        f.n_inputs = len(self.inputs)
        return c

    def _w_full(self, name, w):
        """Per-agent weights: ``w`` ((n, n_in), every agent, or (n_agents, n, n_in)) as a C-contiguous (n_agents, n,
        n_in) float64 array."""
        A, n_in = self.Agent.n_agents, self.inputs[name]["n"]
        w = np.asarray(w, dtype=np.float64)
        if w.shape not in ((self.n, n_in), (A, self.n, n_in)):
            raise ValueError(f"inputs[{name!r}]['w'] must have shape ({self.n}, {n_in}) or ({A}, {self.n}, {n_in}), "
                             f"not {w.shape}")
        return np.array(np.broadcast_to(w, (A, self.n, n_in)), order="C")            # an own, writable copy

    def _split(self, w, meta):
        host = np.zeros(self._lib.riab_ffl_pack_floats(self.n, w.shape[1]), dtype=np.float32)
        _lib.check(self._lib.riab_ffl_pack(_f64p(np.ascontiguousarray(w, dtype=np.float64)), self.n, w.shape[1],
                                           C.byref(meta), host.ctypes.data_as(_lib.c_float_p)))
        return host

    def _w_read(self, name, initial):
        if name not in self._master and self._pa:
            self._cells()                                   # per-agent weights: (A, n, n_in) from the first read on
        if name not in self._master:
            return initial                                  # not on the device yet: the array add_input stored
        sh = self._w_shadow.get(name)
        if sh is None:
            host = self._master[name].cpu().numpy()
            if self._pa and self.Agent.n_agents == 1:
                host = host[0]                                      # the squeeze rule: (n, n_in) for one agent
            sh = self._w_shadow[name] = [host, host.copy()]
        return sh[0]

    def _w_assign(self, name, v):
        if name in self._master:
            sh = self._w_shadow.get(name)
            if sh is None or sh[0] is not v:
                self._w_shadow[name] = [v, None]
            else:
                sh[1] = None                                # `w *= 0.1` re-assigns the array it edited in place

    def _sync_weights(self):
        """Upload the weights the user edited in place or assigned since they were read (Agent._sync_user_writes)."""
        for name, sh in list(self._w_shadow.items()):
            if name not in self._master:
                continue
            host, snap = sh
            if snap is not None and np.array_equal(host, snap, equal_nan=True):
                continue
            if self._pa:
                self._master[name].copy_(self._torch.as_tensor(self._w_full(name, host)))
                sh[1] = np.array(host, dtype=np.float64, copy=True)
                if np.shape(host) != self._master[name].shape[self.Agent.n_agents == 1:]:
                    del self._w_shadow[name]                        # broadcast: the next read copies the masters
                continue
            w = np.ascontiguousarray(host, dtype=np.float64)
            assert w.shape == tuple(self._master[name].shape), \
                f"inputs[{name!r}]['w'] must have shape {tuple(self._master[name].shape)}"
            self._master[name].copy_(self._torch.as_tensor(w))
            meta = _lib.FflInput()
            self._w_pack[name].copy_(self._torch.as_tensor(self._split(w, meta)))
            sh[1] = np.array(host, dtype=np.float64, copy=True)

    # ------------------------------------------------------------------- state
    def _state_rows(self):
        A, ld, torch = self.Agent.n_agents, self._ld(), self._torch
        if self._fr_prev is None:
            self._fr_prev, self._deriv, self._td = (torch.zeros((A, ld), dtype=torch.float32, device=self.device)
                                                    for _ in range(3))

    def _cells(self):
        self._sync_weights()
        c = super()._cells()
        self._state_rows()
        c.fr_prev_dev, c.deriv_dev, c.td_error_dev, c.ld = (self._fr_prev.data_ptr(), self._deriv.data_ptr(),
                                                            self._td.data_ptr(), self._ld())
        c.self_input = -1
        for i, (name, e) in enumerate(self.inputs.items()):
            n_in = e["layer"].n
            ld_in = (n_in + 3) // 4 * 4
            if name not in self._trace and dict.__contains__(e, "eligibility_trace"):
                self._trace[name] = self._torch.zeros((self.Agent.n_agents, ld_in), dtype=self._torch.float32,
                                                      device=self.device)
            c.trace_dev[i] = self._trace[name].data_ptr() if name in self._trace else None
            c.trace_ld[i] = ld_in
            c.w_master_dev[i] = self._master[name].data_ptr()
            if e["layer"] is self:
                c.self_input = i
        self._bind_self(c)
        c.per_agent_weights = int(self._pa)
        c.dt, c.tau, c.tau_e = float(self.Agent.dt), float(self.tau), float(self.tau_e)
        c.eta, c.L2 = float(self.eta), float(self.L2)
        return c

    def _bind_self(self, c):
        """The self-recurrent input reads ``firingrate_last`` (zeros before the first update and after reset)."""
        if c.self_input >= 0:
            c.inputs[c.self_input].rows_dev, c.inputs[c.self_input].ld = self._fr_prev.data_ptr(), self._ld()

    def _layer_struct(self, c):
        return c.ffl

    def _row_buffers(self):
        out = super()._row_buffers()
        self._bind_self(self._cstruct)
        return out

    def _cells_for_run(self):
        self._check_update()
        c = super()._cells_for_run()
        self._bind_self(c)
        return c

    def _host(self, t, n):
        if t is None:
            return np.zeros(n) if self.Agent.n_agents == 1 else np.zeros((self.Agent.n_agents, n))
        r = t[:, :n].cpu().numpy().astype(np.float64)
        return r[0] if self.Agent.n_agents == 1 else r

    @property
    def firingrate(self):
        """The rates of the last update (zeros before it and after ``reset``)."""
        return self._host(self._fr_prev, self.n)

    @property
    def firingrate_deriv(self):
        return self._host(self._deriv, self.n)

    @property
    def td_error(self):
        return self._host(self._td, self.n)

    def _trace_read(self, name):
        self._cells()
        return self._host(self._trace[name], self.inputs[name]["n"])

    def _trace_assign(self, name, v):
        self._cells()
        n_in = self.inputs[name]["n"]
        if name not in self._trace:
            self._trace[name] = self._torch.zeros((self.Agent.n_agents, (n_in + 3) // 4 * 4), dtype=self._torch.float32,
                                                  device=self.device)
        v = np.broadcast_to(np.asarray(v, dtype=np.float64), (self.Agent.n_agents, n_in))
        self._trace[name][:, :n_in].copy_(self._torch.as_tensor(np.ascontiguousarray(v, dtype=np.float32)))

    # --------------------------------------------------------------- get_state
    def get_state(self, evaluate_at="last", max_recurrence=None, **kwargs):
        """FeedForwardLayer.get_state; with per-agent weights see the class docstring (``agents=`` picks the learners
        evaluated at "all" / ``pos``)."""
        if not self._pa:
            return super().get_state(evaluate_at, max_recurrence=max_recurrence, **kwargs)
        torch, A, n = self._torch, self.Agent.n_agents, self.n
        return_tensor = kwargs.pop("return_tensor", False)
        agents = kwargs.pop("agents", None)
        c = self._cells()
        tc = _lib.TdCells.from_buffer_copy(c)
        tc.ffl.prime_dev = None
        per_row = evaluate_at in ("last", "agent")            # the points are the agents: row a uses agent a's weights
        if per_row and agents is not None:
            raise ValueError(f"agents= selects learners for get_state at positions, not at {evaluate_at!r}")
        if evaluate_at == "last":
            self.Agent._flush_pending()
            n_pos = A
        else:
            if max_recurrence != 0 and any(e["layer"] is self for e in self.inputs.values()):
                raise NotImplementedError("get_state away from the agents' rows of a per-agent ValueNeuron that is its "
                                          "own input: pass max_recurrence=0")
            n_pos, keep = self._input_rows(tc.ffl, evaluate_at, max_recurrence, kwargs)
        sel = None
        if per_row:
            n_rows, w_row, in_row = n_pos, None, None
        else:
            sel = np.arange(A) if agents is None else np.asarray(agents, dtype=np.int64).reshape(-1)
            if sel.size and (sel.min() < -A or sel.max() >= A):
                raise IndexError(f"agent index out of range for {A} agents")
            sel = np.where(sel < 0, sel + A, sel)
            n_rows = sel.size * n_pos
            w_row = torch.as_tensor(sel, device=self.device).repeat_interleave(n_pos)
            in_row = torch.arange(n_pos, device=self.device, dtype=torch.int64).repeat(sel.size)
        out = torch.empty((n_rows, self._ld()), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.riab_td_rates_pa(C.byref(tc), n_rows, None if w_row is None else w_row.data_ptr(),
                                              None if in_row is None else in_row.data_ptr(), out.data_ptr(),
                                              self._ld(), self.Agent._stream()))
        if per_row:
            r = self._result(out, return_tensor)
            return r[:, 0] if (evaluate_at == "last" and n_pos == 1 and not return_tensor) else r
        rows = out[:, :n].reshape(sel.size, n_pos, n)                      # (agents, n_pos, n)
        if agents is None and A == 1:
            rows = rows[0]
            return rows if return_tensor else rows.T.contiguous().cpu().numpy().astype(np.float64)
        return rows if return_tensor else rows.transpose(1, 2).contiguous().cpu().numpy().astype(np.float64)

    # ------------------------------------------------------------------ update
    def _check_update(self):
        if self.tau_e == 0:                        # the reference reads input_layer.firingrate of a dict (:75-76)
            raise AttributeError("'dict' object has no attribute 'firingrate'")
        for e in self.inputs.values():
            if not dict.__contains__(e, "eligibility_trace"):
                raise KeyError("eligibility_trace")

    def update(self):
        """ValueNeuron.update (:56-81): the layer's rates (noise and the NaN-position guard included), then the rate
        derivative and every input's eligibility trace, on the device."""
        self._check_update()
        super().update()

    def _reward_operand(self, reward):
        """(riab_td_reward_mode, device pointer, tensors to keep alive) of update_weights' reward."""
        torch, A, n, ld = self._torch, self.Agent.n_agents, self.n, self._ld()
        if isinstance(reward, Neurons):
            if reward.Agent is not self.Agent or reward.n != n:
                raise ValueError(f"a reward population must belong to this Agent and have n={n} cells, "
                                 f"not n={reward.n}")
            if reward._last_slot is None:                           # never updated: its firingrate is zeros
                z = torch.zeros(n, dtype=torch.float64, device=self.device)
                return _lib.TD_REWARD_SHARED, z.data_ptr(), z
            return _lib.TD_REWARD_ROWS, reward._hist.data_ptr() + reward._last_slot * A * ld * 4, None
        if isinstance(reward, torch.Tensor) and reward.device.type == "cuda":
            t = reward.to(device=self.device)
            if t.dim() <= 1 and t.numel() == n and (t.dim() == 0 or A == 1 or n > 1 or t.numel() != A):
                t = t.to(torch.float64).reshape(n).contiguous()
                return _lib.TD_REWARD_SHARED, t.data_ptr(), t
            rows = None
            if t.dim() == 2 and tuple(t.shape) == (A, n):
                rows = t
            elif n == 1 and t.dim() == 1 and t.numel() == A:
                rows = t.reshape(A, 1)
            if rows is not None:
                if rows.dtype == torch.float32 and rows.is_contiguous() and n == ld and rows.data_ptr() % 16 == 0:
                    return _lib.TD_REWARD_ROWS, rows.data_ptr(), rows
                buf = torch.zeros((A, ld), dtype=torch.float32, device=self.device)
                buf[:, :n] = rows
                return _lib.TD_REWARD_ROWS, buf.data_ptr(), buf
            size = t.numel()
        else:
            if isinstance(reward, torch.Tensor):
                reward = reward.detach().cpu().numpy()
            r = np.array(reward, dtype=np.float64)
            if r.size == n and (r.ndim <= 1 or A == 1):
                t = self._upload(r.reshape(n))
                return _lib.TD_REWARD_SHARED, t.data_ptr(), t
            if A > 1 and (r.shape == (A, n) or (n == 1 and r.shape == (A,))):
                buf = np.zeros((A, ld), dtype=np.float32)
                buf[:, :n] = r.reshape(A, n)
                t = self._upload(buf)
                return _lib.TD_REWARD_ROWS, t.data_ptr(), t
            size = r.size
        assert size == n, print(                                    # :86-89, the reference's assert ..., print(...)
            f"Must send same number of reward signals as value neurons (n={self.n}), you sent {size}"
        )
        raise ValueError(f"reward of {size} values fits neither (n,) = ({n},) nor (n_agents, n) = ({A}, {n})")

    def update_weights(self, reward):
        """ValueNeuron.update_weights (:83-104) for every agent, the weight change averaged over the agents."""
        A = self.Agent.n_agents
        mode, ptr, keep = self._reward_operand(reward)
        c = self._cells()
        need = self._lib.riab_td_scratch_bytes(C.byref(c), A)
        if need < 0:
            _lib.check(-1)
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = self._torch.empty(max(int(need), 16), dtype=self._torch.uint8, device=self.device)
        _lib.check(self._lib.riab_td_learn(C.byref(c), A, ptr, mode, c.td_error_dev, self._scratch.data_ptr(),
                                           self.Agent._stream()))
        self._reward_keep = keep
        self._w_shadow.clear()          # the masters moved: the next read of inputs[name]["w"] copies them again

    def reset(self, agents=None):
        """ValueNeuron.reset (:106-113): zero the traces, firingrate (the next update's firingrate_last),
        firingrate_deriv and td_error -- of every agent, or of ``agents`` (indices or a boolean mask)."""
        torch, A = self._torch, self.Agent.n_agents
        c = self._cells()
        mask = None
        if agents is not None:
            sel = np.asarray(agents)
            m = np.zeros(A, dtype=np.uint8)
            if sel.dtype == bool:
                if sel.shape != (A,):
                    raise ValueError(f"a boolean agent mask must have shape ({A},), not {sel.shape}")
                m[sel] = 1
            else:
                idx = sel.astype(np.int64).reshape(-1)
                if idx.size and (idx.min() < -A or idx.max() >= A):
                    raise IndexError(f"agent index out of range for {A} agents")
                m[idx] = 1
            mask = torch.as_tensor(m, device=self.device)
        _lib.check(self._lib.riab_td_reset(C.byref(c), A, mask.data_ptr() if mask is not None else None,
                                           self.Agent._stream()))
        self._reward_keep = mask
