"""ctypes binding of libriab_b200.so (C ABI in include/riab_b200.h).

There is no CPU fallback: if the library cannot be loaded (or built in-tree with
nvcc) importing this module raises, and every entry point raises on a non-zero
status with the library's own message."""
import ctypes as C
import os

from . import _build

c_double_p = C.POINTER(C.c_double)
c_float_p = C.POINTER(C.c_float)


class RiabError(RuntimeError):
    pass


class Env(C.Structure):
    _fields_ = [("walls_dev", C.c_void_p), ("n_walls", C.c_int32), ("n_boundary_walls", C.c_int32),
                ("extent", C.c_double * 4), ("boundary_mode", C.c_int32), ("n_hole_walls", C.c_int32), ("scale", C.c_double),
                ("hole_wall0", C.c_int32), ("reserved", C.c_int32)]


class Agents(C.Structure):
    _fields_ = [("n_agents", C.c_int64), ("id_offset", C.c_int64), ("pos", C.c_void_p), ("velocity", C.c_void_p),
                ("rotational_velocity", C.c_void_p), ("measured_velocity", C.c_void_p),
                ("measured_rotational_velocity", C.c_void_p), ("head_direction", C.c_void_p),
                ("distance_travelled", C.c_void_p), ("distance_to_closest_wall", C.c_void_p)]


class MotionParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "dt", "speed_coherence_time_kw", "speed_mean_kw", "speed_mean", "speed_std", "speed_coherence_time",
        "rotational_velocity_coherence_time_kw", "rotational_velocity_std_kw", "rotational_velocity_drift_kw",
        "head_direction_smoothing_timescale", "thigmotaxis_kw", "wall_repel_distance_kw", "wall_repel_strength_kw",
        "drift_to_random_strength_ratio")]


class StepIO(C.Structure):
    _fields_ = [("drift_velocity", C.c_void_p), ("xi", C.c_void_p), ("seed", C.c_uint64), ("step", C.c_uint64),
                ("collision_mask", C.c_void_p), ("first_hit", C.c_void_p), ("n_iters", C.c_void_p),
                ("history_row", C.c_void_p), ("pos_mirror", C.c_void_p)]


class Trajectory(C.Structure):
    _fields_ = [("times_dev", C.c_void_p), ("y_dev", C.c_void_p), ("M_dev", C.c_void_p), ("T", C.c_int64),
                ("n_traj", C.c_int64), ("t_max", C.c_double)]


class MotionSource(C.Structure):
    _fields_ = [("kind", C.c_int32), ("forced_broadcast", C.c_int32), ("t", C.c_double), ("traj", Trajectory),
                ("forced_dev", C.c_void_p)]


MOTION_RANDOM, MOTION_IMPORTED, MOTION_FORCED = 0, 1, 2      # riab_motion_kind


class ThetaSeq(C.Structure):
    _fields_ = [("n_agents", C.c_int64), ("id_offset", C.c_int64), ("lead_pos", C.c_void_p), ("lead_velocity", C.c_void_p),
                ("lead_rotational_velocity", C.c_void_p), ("lead_distance", C.c_void_p), ("ring", C.c_void_p),
                ("ring_rows", C.c_int64), ("ring_head", C.c_int64), ("window", C.c_int64), ("fwd", Agents),
                ("fwd_pair", C.c_void_p), ("fwd_stop", C.c_void_p), ("fwd_steps", C.c_void_p), ("xi_forward", C.c_void_p),
                ("xi_steps", C.c_int64), ("seed", C.c_uint64), ("rollout", C.c_uint64), ("phase", C.c_int32),
                ("reserved", C.c_int32), ("d_half", C.c_double), ("offset", C.c_double), ("forward_distance", C.c_double),
                ("out_pos", C.c_void_p)]


THETA_NONE, THETA_BEHIND, THETA_AHEAD_FIRST, THETA_AHEAD = 0, 1, 2, 3   # riab_theta_phase


class SubAgentStep(C.Structure):
    _fields_ = [("n_agents", C.c_int64), ("id_offset", C.c_int64), ("kind", C.c_int32), ("reserved", C.c_int32),
                ("seed", C.c_uint64), ("step", C.c_uint64), ("lead_pos", C.c_void_p), ("lead_head_direction", C.c_void_p),
                ("dt", C.c_double), ("shift_m", C.c_double), ("displacement", C.c_void_p),
                ("displacement_velocity", C.c_void_p), ("ou_theta", C.c_double), ("ou_sigma", C.c_double),
                ("acceleration_scale", C.c_double), ("xi_displacement", C.c_void_p), ("resample_pos", C.c_void_p),
                ("t", C.c_double), ("p_start", C.c_double), ("mean_speed", C.c_double), ("mean_duration", C.c_double),
                ("replaying", C.c_void_p), ("replay_state", C.c_void_p), ("replay_count", C.c_void_p), ("sham", Agents),
                ("replay_draws", C.c_void_p), ("xi_replay", C.c_void_p), ("xi_steps", C.c_int64), ("out_pos", C.c_void_p)]


SUBAGENT_SHIFT, SUBAGENT_DUMB, SUBAGENT_REPLAY = 0, 1, 2       # riab_subagent_kind
REPLAY_FIELDS = 9                                            # RIAB_REPLAY_FIELDS


class PlaceCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("description", C.c_int32), ("wall_geometry", C.c_int32),
                ("n_inner_walls", C.c_int32), ("min_fr", C.c_float), ("max_fr", C.c_float),
                ("top_hat_width", C.c_double), ("packed_dev", C.c_void_p), ("centres_dev", C.c_void_p),
                ("eps", C.c_float * 8), ("ep_valid", C.c_int32), ("n_pad", C.c_int32),
                ("k_uniform", C.c_float), ("r2_max", C.c_float)]


class GridCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("description", C.c_int32), ("width_ratio", C.c_double),
                ("min_fr", C.c_float), ("max_fr", C.c_float), ("packed_dev", C.c_void_p), ("n_pad", C.c_int32),
                ("phase_turns", C.c_int32)]


class BvcCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("n_test_angles", C.c_int32), ("min_fr", C.c_float), ("max_fr", C.c_float),
                ("packed_dev", C.c_void_p), ("test_dirs_dev", C.c_void_p), ("n_pad", C.c_int32),
                ("egocentric", C.c_int32)]


MAX_OBJECTS = 9


class OvcCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("n_objects", C.c_int32), ("objects", C.c_double * (2 * MAX_OBJECTS)),
                ("object_types", C.c_int32 * MAX_OBJECTS), ("walls_occlude", C.c_int32), ("egocentric", C.c_int32),
                ("min_fr", C.c_float), ("max_fr", C.c_float), ("packed_dev", C.c_void_p), ("n_pad", C.c_int32),
                ("reserved", C.c_int32)]


FFL_MAX_INPUTS = 4


class FflInput(C.Structure):
    _fields_ = [("w_dev", C.c_void_p), ("n_in", C.c_int32), ("k_pad", C.c_int32), ("rows_dev", C.c_void_p),
                ("ld", C.c_int64), ("population", C.c_int32), ("lag", C.c_int32)]


class FflCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("activation", C.c_int32), ("act", C.c_float * 4), ("bias_dev", C.c_void_p),
                ("prime_dev", C.c_void_p), ("n_inputs", C.c_int32), ("reserved", C.c_int32),
                ("inputs", FflInput * FFL_MAX_INPUTS)]


class TdCells(C.Structure):
    _fields_ = [("ffl", FflCells), ("fr_prev_dev", C.c_void_p), ("deriv_dev", C.c_void_p), ("td_error_dev", C.c_void_p),
                ("ld", C.c_int64), ("trace_dev", C.c_void_p * FFL_MAX_INPUTS), ("trace_ld", C.c_int64 * FFL_MAX_INPUTS),
                ("w_master_dev", C.c_void_p * FFL_MAX_INPUTS), ("dt", C.c_double), ("tau", C.c_double),
                ("tau_e", C.c_double), ("eta", C.c_double), ("L2", C.c_double), ("self_input", C.c_int32),
                ("per_agent_weights", C.c_int32)]
    # FeedForwardLayer's host code reaches the embedded layer's fields through these (they share the struct's memory)
    inputs = property(lambda self: self.ffl.inputs)
    prime_dev = property(lambda self: self.ffl.prime_dev, lambda self, v: setattr(self.ffl, "prime_dev", v))


TdCells.reserved = TdCells.per_agent_weights      # the header's union keeps the field's former name


TD_REWARD_SHARED, TD_REWARD_ROWS = 0, 1                       # riab_td_reward_mode


class RsnCells(C.Structure):
    _fields_ = [("points", PlaceCells), ("targets_dev", C.c_void_p), ("n_cells", C.c_int32), ("n_points", C.c_int32),
                ("k_pad", C.c_int32), ("min_fr", C.c_float), ("max_fr", C.c_float), ("reserved", C.c_int32)]


class KinCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("variant", C.c_int32), ("use_velocity", C.c_int32), ("reserved0", C.c_int32),
                ("min_fr", C.c_float), ("max_fr", C.c_float), ("inv_one_sigma_speed", C.c_double), ("packed_dev", C.c_void_p),
                ("n_pad", C.c_int32), ("reserved1", C.c_int32)]


class AvcCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("walls_occlude", C.c_int32), ("egocentric", C.c_int32), ("partner_is_self", C.c_int32),
                ("min_fr", C.c_float), ("max_fr", C.c_float), ("packed_dev", C.c_void_p), ("other_pos_dev", C.c_void_p),
                ("n_other", C.c_int64), ("n_pad", C.c_int32), ("reserved", C.c_int32)]


class PppcCells(C.Structure):
    _fields_ = [("place", PlaceCells), ("theta_freq", C.c_double), ("sigma", C.c_double), ("precess_fraction", C.c_double),
                ("t", C.c_double)]


class PwnCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("n_pad", C.c_int32), ("min_fr", C.c_float), ("max_fr", C.c_float),
                ("packed_dev", C.c_void_p), ("phase_turns", C.c_int32), ("reserved", C.c_int32)]


NNN_MAX_LAYERS, NNN_MAX_HIDDEN = 8, 256
NNN_ACTIVATIONS = {"identity": 0, "relu": 1, "sigmoid": 2, "tanh": 3}   # riab_nnn_activation


class NnnCells(C.Structure):
    _fields_ = [("n_cells", C.c_int32), ("n_layers", C.c_int32), ("n_inputs", C.c_int32),
                ("widths", C.c_int32 * (NNN_MAX_LAYERS + 1)), ("act", C.c_int32 * NNN_MAX_LAYERS),
                ("packed_dev", C.c_void_p), ("inputs", FflInput * FFL_MAX_INPUTS)]


class HistoryView(C.Structure):
    _fields_ = [("agent_ring", C.c_void_p), ("agent_ring_rows", C.c_int32), ("agent_row0", C.c_int32),
                ("rates_ring", C.c_void_p), ("rates_ring_rows", C.c_int32), ("rates_row0", C.c_int32),
                ("n_steps", C.c_int64), ("n_agents", C.c_int64), ("ld", C.c_int64), ("n_cells", C.c_int32),
                ("reserved", C.c_int32)]


class NeuronNoise(C.Structure):
    _fields_ = [("noise_std", C.c_float), ("noise_coherence_time", C.c_float), ("dt", C.c_double),
                ("seed", C.c_uint64), ("step", C.c_uint64), ("id_offset", C.c_int64), ("population_id", C.c_int32)]


class RatesOut(C.Structure):
    _fields_ = [("rates_row", C.c_void_p), ("ld", C.c_int64), ("spikes_row", C.c_void_p),
                ("noise_state", C.c_void_p), ("bvc_scratch", C.c_void_p)]


class Population(C.Structure):
    _fields_ = [("kind", C.c_int32), ("cells", C.c_void_p), ("noise", NeuronNoise), ("out", RatesOut),
                ("rates_ring", C.c_void_p), ("spikes_ring", C.c_void_p), ("ring_rows", C.c_int32),
                ("ring_next", C.c_int32)]


class AgentHistory(C.Structure):
    _fields_ = [("ring", C.c_void_p), ("ring_rows", C.c_int32), ("ring_next", C.c_int32)]


PC_DESCRIPTIONS = {"gaussian": 0, "gaussian_threshold": 1, "diff_of_gaussians": 2, "top_hat": 3, "one_hot": 4}
WALL_GEOMETRIES = {"euclidean": 0, "line_of_sight": 1, "geodesic": 2}
GC_DESCRIPTIONS = {"rectified_cosines": 0, "shifted_cosines": 1}
(CELLS_PLACE, CELLS_GRID, CELLS_BVC, CELLS_OVC, CELLS_FFL, CELLS_RSN, CELLS_KIN, CELLS_AVC, CELLS_TD, CELLS_PPPC,
 CELLS_PWN, CELLS_NNN) = range(12)
KIN_HEAD_DIRECTION, KIN_VELOCITY, KIN_SPEED = 0, 1, 2                # riab_kin_variant
PLACE_MAX_WI = 8                                              # inner walls of the line-of-sight / geodesic kernels
ACTIVATIONS = {"linear": 0, "sigmoid": 1, "relu": 2, "tanh": 3, "retanh": 4, "softmax": 5}   # riab_activation
MAX_REC_ITERS = 4
MAX_WALLS = 1024                                              # RIAB_MAX_WALLS: walls of the motion and BVC kernels
MAX_STEP_WALLS = 64                                           # RIAB_MAX_STEP_WALLS: walls of the rate kernels that read them

# name -> (restype, argtypes); every symbol include/riab_b200.h declares
SYMBOLS = {
    "riab_abi_version": (C.c_int, []),
    "riab_last_error": (C.c_char_p, []),
    "riab_launch_count": (C.c_int64, []),
    "riab_stream_synchronize": (C.c_int, [C.c_void_p]),
    # (view, edges_x f64, n, edges_y f64, n, sum f64 or NULL, count u64, stream): device pointers
    "riab_history_rate_maps": (C.c_int, [C.POINTER(HistoryView), C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_void_p, C.c_void_p, C.c_void_p]),
    "riab_agent_update": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO), C.c_void_p]),
    "riab_trajectory_build": (C.c_int, [C.POINTER(Trajectory), c_double_p, C.c_void_p]),
    "riab_agent_update_src": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO),
                                        C.POINTER(MotionSource), C.c_void_p]),
    "riab_theta_seq_step": (C.c_int, [C.POINTER(ThetaSeq), C.POINTER(Env), C.POINTER(MotionParams), C.c_void_p]),
    "riab_subagent_step": (C.c_int, [C.POINTER(SubAgentStep), C.POINTER(Env), C.POINTER(MotionParams), C.c_void_p]),
    "riab_place_pack_floats": (C.c_int64, [C.c_int32, C.c_int32]),
    "riab_place_pack": (C.c_int, [c_double_p, c_double_p, C.c_int32, c_double_p, C.c_int32, C.c_int32, c_double_p,
                                  C.c_int32, C.POINTER(PlaceCells), c_float_p]),
    "riab_place_rates": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(PlaceCells), C.c_void_p, C.c_int64, C.c_void_p]),
    "riab_grid_pack_floats": (C.c_int64, [C.c_int32]),
    "riab_grid_pack": (C.c_int, [c_double_p, c_double_p, c_double_p, C.c_int32, c_double_p, C.POINTER(GridCells), c_float_p]),
    "riab_grid_rates": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(GridCells), C.c_void_p, C.c_int64, C.c_void_p]),
    "riab_bvc_pack_floats": (C.c_int64, [C.c_int32, C.c_int32]),
    "riab_bvc_scratch_floats": (C.c_int64, [C.c_int64, C.c_int32]),
    "riab_bvc_pack": (C.c_int, [c_double_p, c_double_p, c_double_p, c_double_p, C.c_int32, c_double_p, C.c_int32,
                                C.POINTER(BvcCells), c_float_p]),
    "riab_bvc_rates": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(BvcCells), C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "riab_ovc_pack_floats": (C.c_int64, [C.c_int32]),
    "riab_ovc_pack": (C.c_int, [c_double_p, c_double_p, c_double_p, c_double_p, C.POINTER(C.c_int32), C.c_int32,
                                C.POINTER(OvcCells), c_float_p]),
    "riab_ovc_rates": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(OvcCells), C.c_void_p, C.c_void_p,
                                 C.c_int64, C.c_void_p]),
    "riab_ffl_pack_floats": (C.c_int64, [C.c_int32, C.c_int32]),
    "riab_ffl_pack": (C.c_int, [c_double_p, C.c_int32, C.c_int32, C.POINTER(FflInput), c_float_p]),
    "riab_ffl_rates": (C.c_int, [C.POINTER(FflCells), C.c_int64, C.c_void_p, C.POINTER(NeuronNoise), C.POINTER(RatesOut),
                                 C.c_void_p]),
    "riab_td_splits": (C.c_int64, [C.c_int32, C.c_int32, C.c_int64]),
    "riab_td_scratch_bytes": (C.c_int64, [C.POINTER(TdCells), C.c_int64]),
    "riab_td_learn": (C.c_int, [C.POINTER(TdCells), C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "riab_td_reset": (C.c_int, [C.POINTER(TdCells), C.c_int64, C.c_void_p, C.c_void_p]),
    "riab_td_rates_pa": (C.c_int, [C.POINTER(TdCells), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                   C.c_void_p]),
    "riab_rsn_pack_floats": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "riab_rsn_pack": (C.c_int, [c_double_p, C.c_int32, c_double_p, C.c_int32, C.c_double, c_double_p, C.c_int32, C.c_int32,
                                c_double_p, C.c_int32, C.POINTER(RsnCells), c_float_p, c_double_p]),
    "riab_rsn_rates": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(RsnCells), C.c_void_p, C.c_int64, C.c_void_p]),
    "riab_kin_pack_floats": (C.c_int64, [C.c_int32]),
    "riab_kin_pack": (C.c_int, [c_double_p, c_double_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_double,
                                C.POINTER(KinCells), c_float_p]),
    "riab_kin_rates": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.POINTER(KinCells), C.c_void_p, C.c_int64,
                                 C.c_void_p]),
    "riab_avc_pack_floats": (C.c_int64, [C.c_int32]),
    "riab_avc_pack": (C.c_int, [c_double_p, c_double_p, c_double_p, c_double_p, C.c_int32, C.POINTER(AvcCells), c_float_p]),
    "riab_avc_rates": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.POINTER(Env), C.POINTER(AvcCells),
                                 C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "riab_pppc_rates": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(PppcCells), C.c_void_p,
                                  C.c_int64, C.c_void_p]),
    "riab_pwn_pack_floats": (C.c_int64, [C.c_int32]),
    "riab_pwn_pack": (C.c_int, [c_double_p, c_double_p, c_double_p, C.c_int32, c_double_p, C.c_int32, C.POINTER(PwnCells),
                                c_float_p]),
    "riab_pwn_rates": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(Env), C.POINTER(PwnCells), C.c_void_p, C.c_int64, C.c_void_p]),
    "riab_nnn_pack_floats": (C.c_int64, [C.POINTER(NnnCells)]),
    "riab_nnn_pack": (C.c_int, [c_double_p, C.POINTER(NnnCells), c_float_p]),
    "riab_nnn_rates": (C.c_int, [C.POINTER(NnnCells), C.c_int64, C.c_void_p, C.POINTER(NeuronNoise), C.POINTER(RatesOut),
                                 C.c_void_p]),
    "riab_step_fused": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO),
                                  C.c_int32, C.c_void_p, C.POINTER(NeuronNoise), C.POINTER(RatesOut), C.c_void_p]),
    "riab_neurons_update": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.c_int32, C.c_void_p, C.POINTER(NeuronNoise),
                                      C.POINTER(RatesOut), C.c_void_p]),
    "riab_run": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO),
                           C.POINTER(Population), C.c_int32, C.POINTER(AgentHistory), C.c_int64, C.c_void_p]),
    "riab_run_src": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO),
                               C.POINTER(MotionSource), C.POINTER(Population), C.c_int32, C.POINTER(AgentHistory), C.c_int64,
                               C.c_void_p]),
    "riab_agent_update_host": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO),
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "riab_positions_wait": (C.c_int, []),
    "riab_positions_fence": (C.c_int, [C.c_void_p]),
    "riab_step_fused_host": (C.c_int, [C.POINTER(Agents), C.POINTER(Env), C.POINTER(MotionParams), C.POINTER(StepIO),
                                       C.c_int32, C.c_void_p, C.POINTER(NeuronNoise), C.POINTER(RatesOut),
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None


def lib_path():
    return _build.LIB


def load():
    """Load (building in-tree first if needed).  Raises if that is impossible."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if not os.path.exists(path):
        if not _have_nvcc():
            raise ImportError(f"{path} is missing and nvcc is not available to build it: "
                              "ratinabox_b200 has no CPU fallback")
        _build.build()
    elif os.path.isdir(_build.CSRC) and _build.needs_build():
        # sources newer than the library (or file times scrambled by a copy): rebuilding takes minutes, so it is only
        # done on request (__graft_entry__.build(), `python ratinabox_b200/_build.py`, RIAB_AUTO_REBUILD=1)
        if os.environ.get("RIAB_AUTO_REBUILD") == "1" and _have_nvcc():
            _build.build()
        else:
            import warnings
            warnings.warn(f"{path} is older than its CUDA sources; run __graft_entry__.build() to rebuild")
    lib = C.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)      # AttributeError if the symbol is not exported
        fn.restype, fn.argtypes = res, args
    if lib.riab_abi_version() != 3:
        raise ImportError("libriab_b200.so ABI version mismatch")
    _lib = lib
    return lib


def _have_nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return os.path.exists(nvcc)


def check(rc):
    if rc != 0:
        raise RiabError(f"libriab_b200 status {rc}: {load().riab_last_error().decode()}")
