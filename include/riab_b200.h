/* riab_b200.h -- C ABI of the H100-native batched step engine for RatInABox's
 * per-step hot path (Agent.update + Neurons.update for PlaceCells, GridCells,
 * BoundaryVectorCells).
 *
 * The reference (RatInABox v1.15.3) is pure Python: it has no FFI.  Its
 * extension boundary is two overridable methods,
 *     Agent.update(dt, drift_velocity, drift_to_random_strength_ratio, **kw)   ratinabox/Agent.py:160
 *     Neurons.update(**kw) -> get_state(evaluate_at, **kw)                     ratinabox/Neurons.py:145,173
 * and that is what this library sits behind.  Each entry point below names the
 * reference function it replaces.  The Python host mirror (ratinabox_b200/)
 * binds these symbols with ctypes; INTEGRATION.md shows the stub a reference
 * maintainer would add.
 *
 * Conventions
 *   - plain C: pointers, sizes, POD structs; no torch / C++ types.
 *   - "dev" pointers are CUDA device pointers owned by the caller (the Python
 *     host allocates them with torch); "host" pointers are ordinary memory.
 *   - every launch goes to the CUDA stream passed as `stream` (a cudaStream_t
 *     cast to void*; NULL = legacy default stream).  No host sync inside.
 *   - return value: 0 on success, negative riab_status otherwise;
 *     riab_last_error() gives the message (thread local).
 *   - agent state is float64 (the reference's dtype, Agent.py:197-198); firing
 *     rates / history rows are float32.
 */
#ifndef RIAB_B200_H
#define RIAB_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RIAB_ABI_VERSION 3

typedef enum {
  RIAB_OK = 0,
  RIAB_ERR_INVALID = -1,   /* bad argument (the reference would assert / raise ValueError) */
  RIAB_ERR_CUDA = -2,      /* CUDA runtime error */
  RIAB_ERR_UNSUPPORTED = -3 /* outside the supported path (see DESIGN.md "out of scope") */
} riab_status;

int riab_abi_version(void);
const char* riab_last_error(void);

/* RIAB_BOUNDARY_SOLID_BOX: strict 4-compare in-environment test and clamp (Environment.py:793-806, :880-889).
 * RIAB_BOUNDARY_PERIODIC_BOX: no boundary walls are built (:130-144); positions wrap (:877-879), displacement /
 *   distance vectors take the short way round (:670-675).
 * RIAB_BOUNDARY_POLYGON: polygon boundary and / or holes, solid.  In the environment <=> strictly inside the boundary
 *   polygon and not strictly inside a hole (:807-817, shapely `contains`), decided by an even-odd ray cast over the
 *   boundary / hole walls; a position outside after the bounce loop is re-drawn uniformly inside (:892-893, the
 *   reference draws from np.random there; here a Philox stream keyed by seed / step / agent). */
typedef enum { RIAB_BOUNDARY_SOLID_BOX = 0, RIAB_BOUNDARY_PERIODIC_BOX = 1, RIAB_BOUNDARY_POLYGON = 2 } riab_boundary_mode;

/* ---------------------------------------------------------------- Environment
 * walls: (n_walls,2,2) float64, boundary walls first (Environment.py:137-144),
 * then user walls (add_wall, :330-342), then the walls of the holes (:147-160).  2D: rectangular box (solid or
 * periodic), or a polygon boundary and / or holes (solid).
 *
 * Wall count: every entry point accepts up to RIAB_MAX_WALLS walls for what reads no walls or reads them in the motion
 * and BVC ray kernels (the stepped motion, SubAgents, ThetaSequenceAgent, BVCs, and the populations below that ignore
 * walls).  Rates that read walls keep RIAB_MAX_STEP_WALLS: line_of_sight / geodesic PlaceCells, PhasePrecessingPlaceCells
 * and RandomSpatialNeurons (and so the SpatialGoalEnvironment goal test), ObjectVectorCells / AgentVectorCells with
 * walls_occlude.  Above RIAB_MAX_STEP_WALLS, riab_step_fused and riab_run run the stand-alone motion kernel and then
 * each population (no fused, skewed or whole-run launch). */
#define RIAB_MAX_WALLS 1024
#define RIAB_MAX_STEP_WALLS 64        /* walls the rate kernels (k_step, k_place_onehot, k_rsn) stage */
typedef struct {
  const double* walls_dev;     /* device, n_walls*4 doubles */
  int32_t n_walls;
  int32_t n_boundary_walls;    /* the first n_boundary_walls walls are the closed boundary polygon (4 for the box) */
  double extent[4];            /* left,right,bottom,top  (Environment.py:171-173) */
  int32_t boundary_mode;       /* riab_boundary_mode */
  int32_t n_hole_walls;        /* RIAB_BOUNDARY_POLYGON: walls [hole_wall0, hole_wall0 + n_hole_walls) are the edges of the holes */
  double scale;                /* Environment.scale: the wrap threshold is scale/2 on both axes (:671) */
  int32_t hole_wall0;
  int32_t reserved;
} riab_env;

/* ---------------------------------------------------------------------- Agent
 * Structure-of-arrays batched state; every pointer is a device array with
 * n_agents rows.  Mirrors the attributes Agent.update mutates (Agent.py:193-201,
 * SURVEY 8(b)). */
typedef struct {
  int64_t n_agents;
  int64_t id_offset;             /* global id of row 0 (multi-GPU shards; keys the Philox stream) */
  double* pos;                   /* (A,2)  Agent.pos */
  double* velocity;              /* (A,2)  Agent.velocity */
  double* rotational_velocity;   /* (A)    Agent.rotational_velocity */
  double* measured_velocity;     /* (A,2)  Agent.measured_velocity */
  double* measured_rotational_velocity; /* (A) */
  double* head_direction;        /* (A,2) */
  double* distance_travelled;    /* (A) */
  double* distance_to_closest_wall; /* (A) */
} riab_agents;

/* Scalar parameters of one Agent.update call.  `*_kw` are the values after the
 * per-call kwargs override (Agent.py:280-285, :353-355); the others are the
 * attributes the reference reads directly. */
typedef struct {
  double dt;
  double speed_coherence_time_kw;               /* Agent.py:283 */
  double speed_mean_kw;                         /* Agent.py:284: Rayleigh sigma of the speed process */
  double speed_mean;                            /* attribute: wall repulsion (:370) and bounce speed (:439) */
  double speed_std;                             /* attribute: ==0 -> constant speed (:310) */
  double speed_coherence_time;                  /* attribute: drift update (:340) */
  double rotational_velocity_coherence_time_kw; /* :281 */
  double rotational_velocity_std_kw;            /* :280 */
  double rotational_velocity_drift_kw;          /* :282 */
  double head_direction_smoothing_timescale;    /* attribute (:489) */
  double thigmotaxis_kw;                        /* :355 */
  double wall_repel_distance_kw;                /* :354 */
  double wall_repel_strength_kw;                /* :353 */
  double drift_to_random_strength_ratio;        /* Agent.update arg */
} riab_motion_params;

/* Optional per-step inputs / parity taps (device pointers, may be NULL).  drift_velocity and pos_mirror may
 * also point to page-locked HOST memory (unified addressing): the motion step then reads the commands and posts the
 * new positions over the bus itself, without separate copies (1 MB each way at 65 536 agents). */
typedef struct {
  const double* drift_velocity;   /* (A,2) Agent.update(drift_velocity=...), Agent.py:324-341 */
  const double* xi;               /* (A,2) injected standard normals for the two OU draws
                                     (oracle mode A); NULL -> Philox4x32-10(seed, step, agent id) */
  uint64_t seed;
  uint64_t step;                  /* step counter (Philox counter word) */
  uint8_t* collision_mask;        /* (A, RIAB_MAX_REC_ITERS, n_walls) per-iteration wall_collisions
                                     of Environment.check_wall_collisions (Environment.py:820-841) */
  int32_t* first_hit;             /* (A, RIAB_MAX_REC_ITERS) lowest colliding wall index or -1 (Agent.py:437) */
  int32_t* n_iters;               /* (A) number of collision-loop iterations executed */
  float* history_row;             /* (A,8) float32: pos.xy, vel.xy (measured), head_direction.xy,
                                     rot_vel, distance_travelled -- Agent.save_to_history, Agent.py:509-521 */
  double* pos_mirror;             /* (A,2) second copy of the new positions (e.g. a pinned host buffer) or NULL */
} riab_step_io;

#define RIAB_MAX_REC_ITERS 4
#define RIAB_MAX_BOUNCE_ITERS 32

/* Agent.update (Agent.py:160-242, random-motion branch) for n_agents agents; up to RIAB_MAX_WALLS walls. */
int riab_agent_update(const riab_agents* agents, const riab_env* env,
                      const riab_motion_params* prm, const riab_step_io* io, void* stream);

/* ---------------------------------------------------- imported / forced motion
 * Agent.update's other two branches (Agent.py:202-242): the position of a step comes from an imported trajectory
 * (Agent.import_trajectory, :543-659: `pos = pos_interp(t % max(t_interp))`, pos_interp the not-a-knot cubic spline of
 * scipy's interp1d(kind="cubic")) or from a forced_next_position; then measured velocity / rotational velocity with
 * overwrite_velocity=True (:444-472), head direction, distance travelled (+0 when pos or prev_pos holds a NaN) and the
 * history row.  The random-motion parameters and drift_velocity are ignored, distance_to_closest_wall is not updated.
 *
 * A trajectory: times shared by every agent, positions either shared (n_traj = 1) or one per agent (n_traj = n_agents),
 * stored sample-major so that the agents' samples of one time are contiguous.  M holds the spline's second
 * derivatives, written by riab_trajectory_build. */
typedef struct {
  const double* times_dev;  /* (T) f64, times[0] == 0, strictly increasing (import_trajectory shifts and sorts) */
  const double* y_dev;      /* (T, n_traj, 2) f64 positions */
  double* M_dev;            /* (T, n_traj, 2) f64 second derivatives of the spline */
  int64_t T;                /* >= 4 (interp1d's minimum for kind="cubic") */
  int64_t n_traj;           /* 1 (shared) or n_agents */
  double t_max;             /* times[T-1] = max(t_interp) */
} riab_trajectory;

/* Solve the not-a-knot spline system of every (trajectory, axis) column (one thread per column) into tr->M_dev.
 * times_host: the same T times as tr->times_dev; the elimination factors, which depend on the times only, are
 * computed on the host in float64. */
int riab_trajectory_build(const riab_trajectory* tr, const double* times_host, void* stream);

typedef enum { RIAB_MOTION_RANDOM = 0, RIAB_MOTION_IMPORTED = 1, RIAB_MOTION_FORCED = 2 } riab_motion_kind;
typedef struct {
  int32_t kind;                 /* riab_motion_kind */
  int32_t forced_broadcast;     /* RIAB_MOTION_FORCED: 1 = forced_dev is one (2) position for every agent */
  double t;                     /* Agent.t of the (first) step, after its `t += dt`; later steps of a run add dt */
  riab_trajectory traj;         /* RIAB_MOTION_IMPORTED */
  const double* forced_dev;     /* RIAB_MOTION_FORCED: (A,2) or (2) f64, device or page-locked host memory */
} riab_motion_source;

/* Agent.update with a motion source; src == NULL or RIAB_MOTION_RANDOM is riab_agent_update.  io: seed / step (the
 * zero-displacement draw), history_row, pos_mirror; drift_velocity, xi and the collision taps are ignored. */
int riab_agent_update_src(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                          const riab_step_io* io, const riab_motion_source* src, void* stream);

/* ------------------------------------------------------ ThetaSequenceAgent
 * contribs/SubAgent.py:182-356: the position of a theta sweep over a lead Agent's batch at one lead step, written to
 * out_pos; the ThetaSequenceAgent then moves there with riab_agent_update_src (RIAB_MOTION_FORCED).  The host computes
 * the theta phase from the lead's clock (:266-267), so `phase` is the same for every agent:
 *   RIAB_THETA_NONE        before the look-behind or after the look-ahead (:270-271, :337-338): NaN
 *   RIAB_THETA_BEHIND      :274-300: interp1d over rows [idx-3, idx+3) of the window of the lead's recent rows, idx the
 *                          first arg-min of |distance - target|; the lead's position while its distance is < d_half.
 *                          Where the reference raises (idx < 3, or target outside those rows) the two window rows that
 *                          bracket the target are interpolated; a target before the window gives NaN.
 *   RIAB_THETA_AHEAD_FIRST :305-327: the forward agent starts from the lead's pos / velocity / rotational velocity /
 *                          distance (its measured velocity and head direction carry over); stop = distance + forward_distance
 *   RIAB_THETA_AHEAD       :328-334: the forward agent advances (at least one step per rollout) while its distance is
 *                          below both the query and the stop; the position interpolates its last two samples.  A query
 *                          past the stop or behind the kept pair gives NaN.
 * target / query = lead distance + offset (-distance_back / +distance_ahead, host float64).  Any position farther than
 * d_half from the lead's (periodic boundaries wrap) becomes NaN (:341-343).  The lead's (x, y, distance) row is appended
 * to the ring at ring_head on every call (:259-264). */
typedef enum { RIAB_THETA_NONE = 0, RIAB_THETA_BEHIND = 1, RIAB_THETA_AHEAD_FIRST = 2, RIAB_THETA_AHEAD = 3 } riab_theta_phase;
typedef struct {
  int64_t n_agents;
  int64_t id_offset;                      /* global id of row 0 (keys the forward rollouts' Philox stream) */
  const double* lead_pos;                 /* (A,2) device: the lead Agent's state after its update */
  const double* lead_velocity;            /* (A,2) */
  const double* lead_rotational_velocity; /* (A) */
  const double* lead_distance;            /* (A) distance_travelled */
  double* ring;                           /* (3, ring_rows, A) f64: lead x, y, distance of the recent lead steps */
  int64_t ring_rows;
  int64_t ring_head;                      /* slot of this step's row */
  int64_t window;                         /* 1 <= window <= ring_rows rows end at ring_head (RIAB_THETA_BEHIND) */
  riab_agents fwd;                        /* forward agent state (id_offset ignored) */
  double* fwd_pair;                       /* (A,3) distance, x, y of the forward agent's previous rollout sample */
  double* fwd_stop;                       /* (A) stop distance of the current rollout */
  int64_t* fwd_steps;                     /* (A) rollout steps taken */
  const double* xi_forward;               /* (A, xi_steps, 2) injected standard normals of rollout steps 0.. or NULL; */
  int64_t xi_steps;                       /*   steps >= xi_steps draw Philox4x32-10(seed, rollout, step, agent id) */
  uint64_t seed;
  uint64_t rollout;                       /* rollout counter (Philox sub-index) */
  int32_t phase;                          /* riab_theta_phase */
  int32_t reserved;
  double d_half;
  double offset;
  double forward_distance;                /* d_half + 100 average_measured_speed (theta_frac / 2) T_theta */
  double* out_pos;                        /* (A,2) device */
} riab_theta_seq;
/* fwd_prm: the forward agent's motion parameters, dt = lead dt * v_sequence / average_measured_speed. */
int riab_theta_seq_step(const riab_theta_seq* ts, const riab_env* env, const riab_motion_params* fwd_prm, void* stream);

/* ------------------------------------------------- DumbAgent, ShiftAgent, ReplayAgent
 * contribs/SubAgent.py:118-179, :358-431, :466-478: the position of one SubAgent per lead agent at one lead step,
 * written to out_pos; the SubAgent then moves there with riab_agent_update_src (RIAB_MOTION_FORCED).  float64, in the
 * reference's operation order.
 *   RIAB_SUBAGENT_SHIFT  lead pos + lead head direction * shift_m (no boundary condition, :476)
 *   RIAB_SUBAGENT_DUMB   :151-179: OU + spring on displacement_velocity, displacement cut back to 0.95 of the nearest
 *                        strict wall crossing of [lead pos, lead pos + displacement], boundary conditions (a polygon or
 *                        hole re-draws a random position), displacement re-measured through the boundary
 *   RIAB_SUBAGENT_REPLAY :380-426: not replaying: one uniform, u > p_start tracks the lead, else a replay starts at a
 *                        random position of the sham agent; replaying with t < end: the sham's rollout interpolated by
 *                        its distance at replay_speed (t - start), the rollout stepped lazily with motion_step
 *                        (sham_prm) while its distance is below the query and the stop; else back to the lead.
 * Draws: Philox4x32-10 keyed by global agent id; DUMB: stream 6 (sub 0 the two normals, sub 1 + k the k-th re-draw),
 * step = `step`; REPLAY: stream 7 (sub 0: u, speed; sub 1: duration, direction; sub 2 + k: the k-th start position),
 * step = `step`; rollouts: stream 8, sub = the agent's replay index, step = rollout step. */
typedef enum { RIAB_SUBAGENT_SHIFT = 0, RIAB_SUBAGENT_DUMB = 1, RIAB_SUBAGENT_REPLAY = 2 } riab_subagent_kind;
#define RIAB_REPLAY_FIELDS 9          /* replay_state columns: speed, duration, start, end, stop, start distance,
                                         previous rollout sample's distance, x, y */
typedef struct {
  int64_t n_agents;
  int64_t id_offset;                  /* global id of row 0 */
  int32_t kind;                       /* riab_subagent_kind */
  int32_t reserved;
  uint64_t seed;
  uint64_t step;                      /* this SubAgent's update count (Philox step word) */
  const double* lead_pos;             /* (A,2) device: the lead Agent's state after its update */
  const double* lead_head_direction;  /* (A,2) SHIFT */
  double dt;                          /* LeadAgent.dt */
  double shift_m;                     /* SHIFT */
  /* DUMB */
  double* displacement;               /* (A,2) in / out */
  double* displacement_velocity;      /* (A,2) in / out */
  double ou_theta, ou_sigma;          /* 1 / tau_v, sqrt(2 sigma^2 / (tau_v dt)) (utils.py:364-366) */
  double acceleration_scale;
  const double* xi_displacement;      /* (A,2) injected standard normals or NULL */
  const double* resample_pos;         /* (A,2) injected re-drawn positions or NULL */
  /* REPLAY */
  double t;                           /* the ReplayAgent's t before the step (:399) */
  double p_start;                     /* replay_freq * dt */
  double mean_speed, mean_duration;
  uint8_t* replaying;                 /* (A) in / out: is_undergoing_replay */
  double* replay_state;               /* (A, RIAB_REPLAY_FIELDS) */
  int64_t* replay_count;              /* (A,2): replays started, rollout steps of the current one */
  riab_agents sham;                   /* the sham rollout agent's state (n_agents, id_offset ignored) */
  const double* replay_draws;         /* (A,6) injected u, speed, duration (before the clamp), x0, y0, direction or NULL */
  const double* xi_replay;            /* (A, xi_steps, 2) injected standard normals of rollout steps 0.. or NULL */
  int64_t xi_steps;
  double* out_pos;                    /* (A,2) device */
} riab_subagent;
/* sham_prm: the sham agent's motion parameters (REPLAY; may be NULL otherwise). */
int riab_subagent_step(const riab_subagent* sa, const riab_env* env, const riab_motion_params* sham_prm, void* stream);

/* ----------------------------------------------------------------- PlaceCells */
typedef enum { RIAB_PC_GAUSSIAN = 0, RIAB_PC_GAUSSIAN_THRESHOLD = 1, RIAB_PC_DIFF_OF_GAUSSIANS = 2,
               RIAB_PC_TOP_HAT = 3, RIAB_PC_ONE_HOT = 4 } riab_pc_description;   /* Neurons.py:959-976 */
typedef enum { RIAB_GEOM_EUCLIDEAN = 0, RIAB_GEOM_LINE_OF_SIGHT = 1, RIAB_GEOM_GEODESIC = 2 } riab_wall_geometry; /* Environment.py:707-774 */

typedef struct {
  int32_t n_cells;
  int32_t description;     /* riab_pc_description */
  int32_t wall_geometry;   /* riab_wall_geometry */
  int32_t n_inner_walls;   /* walls[4:] used by line_of_sight / geodesic */
  float min_fr, max_fr;    /* Neurons.py:978-980 */
  double top_hat_width;    /* the scalar `widths` param (Neurons.py:975-976) */
  const float* packed_dev; /* device block written by riab_place_pack (size riab_place_pack_floats) */
  const double* centres_dev; /* (N,2) float64 centres, used by the exact fall-back of the wall predicates */
  /* filled by riab_place_pack: */
  float eps[8];            /* relative uncertainty band of the float32 line-of-sight predicate, per inner wall */
  int32_t ep_valid;        /* geodesic: bit k set iff end k of walls[4] lies strictly inside the box (Environment.py:748) */
  int32_t n_pad;           /* n_cells rounded up to a multiple of 4 */
  float k_uniform;         /* log2(e)/(2 w^2) when every cell has the same width w, else 0 */
  float r2_max;            /* max squared distance of a centre or box corner from the box centre */
} riab_place_cells;

/* Host-side packing of PlaceCells parameters (place_cell_centres (N,2) f64,
 * place_cell_widths (N) f64, walls (W,2,2) f64) into the float32 block the
 * kernels read.  Returns number of floats written / needed. */
int64_t riab_place_pack_floats(int32_t n_cells, int32_t n_inner_walls);
int riab_place_pack(const double* centres_host, const double* widths_host, int32_t n_cells,
                    const double* walls_host, int32_t n_walls, int32_t n_boundary_walls,
                    const double* extent, int32_t wall_geometry, riab_place_cells* meta_out, float* out_host);

/* PlaceCells.get_state(evaluate_at=None, pos=P) (Neurons.py:936-981):
 * pos_dev (n_pos,2) f64 -> out_dev (n_pos, ld_out) f32, row = position, col = cell
 * (the transposed, coalesced view of the reference's (n_cells,n_pos)). */
int riab_place_rates(const double* pos_dev, int64_t n_pos, const riab_env* env,
                     const riab_place_cells* pc, float* out_dev, int64_t ld_out, void* stream);

/* ------------------------------------------------------------------ GridCells */
typedef enum { RIAB_GC_RECTIFIED_COSINES = 0, RIAB_GC_SHIFTED_COSINES = 1 } riab_gc_description; /* Neurons.py:1203-1218 */
typedef struct {
  int32_t n_cells;
  int32_t description;
  double width_ratio;      /* Neurons.py:1064 */
  float min_fr, max_fr;
  const float* packed_dev; /* riab_grid_pack output */
  int32_t n_pad;           /* filled by riab_grid_pack */
  int32_t phase_turns;     /* filled by riab_grid_pack: 1 = the block holds wave vectors and phases in turns, for the
                              compensated phase of large |k| r_max (riab_grid.cuh); 0 = radians */
} riab_grid_cells;
int64_t riab_grid_pack_floats(int32_t n_cells);
int riab_grid_pack(const double* gridscales_host, const double* phase_offsets_host /* (N,2) */,
                   const double* w_host /* (N,3,2) */, int32_t n_cells, const double* extent,
                   riab_grid_cells* meta_out, float* out_host);
/* GridCells.get_state (2D), Neurons.py:1172-1236 */
int riab_grid_rates(const double* pos_dev, int64_t n_pos, const riab_env* env,
                    const riab_grid_cells* gc, float* out_dev, int64_t ld_out, void* stream);

/* -------------------------------------------------------- BoundaryVectorCells */
typedef struct {
  int32_t n_cells;
  int32_t n_test_angles;   /* T = int(360/dtheta), Neurons.py:1588 */
  float min_fr, max_fr;
  const float* packed_dev;       /* riab_bvc_pack output (per-cell tuning + von Mises table tiles) */
  const double* test_dirs_dev;   /* (T,2) f64 test_directions (Neurons.py:1584-1596, duplicated-0 quirk kept) */
  int32_t n_pad;                 /* filled by riab_bvc_pack: n_cells rounded up to the cell tile (64) */
  int32_t egocentric;            /* reference_frame == "egocentric" (Neurons.py:1693-1708, FieldOfViewBVCs :1847-1887):
                                    test angles are measured from utils.get_angle(head_direction) */
} riab_bvc_cells;
int64_t riab_bvc_pack_floats(int32_t n_cells, int32_t n_test_angles);
int riab_bvc_pack(const double* tuning_distances, const double* tuning_angles, const double* sigma_distances,
                  const double* sigma_angles, int32_t n_cells, const double* test_angles, int32_t n_test_angles,
                  riab_bvc_cells* meta_out, float* out_host);
/* Packed block (float32 unless noted), Np = n_cells rounded up to 64:  s[Np] | m[Np] | 1/norm[Np] (cell order) |
 * von Mises weights, peak 1, [Np/64][T][64] in SLOT order | egocentric extras 3 Np + 2 T | int32 perm[Np] (slot -> cell:
 * the cells sorted by tuning angle) | int32 (th0, len)[Np/32]: the angular window of each 32 slots outside which every
 * weight is < 2^-30 and the integrand terms are skipped (their sum is < T 2^-30 / norm of the peak rate). */
/* BoundaryVectorCells.get_state (allocentric), Neurons.py:1617-1778.
 * scratch_dev: riab_bvc_scratch_floats(n_pos, T) float32 workspace holding dist_to_first_wall in
 * [agent tile of 32][T][32] order; first_wall_dev optional (n_pos,T) int32 (argmax wall id, Neurons.py:1677-1679). */
int64_t riab_bvc_scratch_floats(int64_t n_pos, int32_t n_test_angles);
int riab_bvc_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_bvc_cells* bvc,
                   float* scratch_dev, int32_t* first_wall_dev, const double* head_direction_dev /* (n_pos,2) f64 for
                   egocentric cells; NULL = [1,0] (the reference's default, Neurons.py:1703) */,
                   float* out_dev, int64_t ld_out, void* stream);

/* --------------------------------------------------------- ObjectVectorCells
 * Neurons.py:1892-2113.  Objects live in the Environment (Environment.add_object, Environment.py:366-395): up to
 * RIAB_MAX_OBJECTS positions with an integer type each.  Cell i fires for the objects whose type equals
 * tuning_types[i]: sum of gaussian(distance) * von_mises(bearing), both with peak 1 (Neurons.py:2090-2104); with
 * walls_occlude the distance is the `line_of_sight` one (1000 behind an inner wall, Environment.py:710-730);
 * egocentric cells measure bearings from the head direction (Neurons.py:2030-2047). */
#define RIAB_MAX_OBJECTS 9
typedef struct {
  int32_t n_cells;
  int32_t n_objects;
  double objects[2 * RIAB_MAX_OBJECTS];     /* Environment.objects["objects"], (n_objects,2) */
  int32_t object_types[RIAB_MAX_OBJECTS];   /* Environment.objects["object_types"] */
  int32_t walls_occlude;                    /* 1: wall_geometry "line_of_sight", 0: "euclidean" (Neurons.py:1937-1940) */
  int32_t egocentric;                       /* reference_frame == "egocentric" */
  float min_fr, max_fr;
  const float* packed_dev;                  /* device block written by riab_ovc_pack (riab_ovc_pack_floats floats) */
  int32_t n_pad;                            /* filled by riab_ovc_pack */
  int32_t reserved;
} riab_ovc_cells;
int64_t riab_ovc_pack_floats(int32_t n_cells);
/* tuning_angles / sigma_angles in radians (VectorCells attributes), tuning_types (n_cells) int32 */
int riab_ovc_pack(const double* tuning_distances, const double* tuning_angles, const double* sigma_distances,
                  const double* sigma_angles, const int32_t* tuning_types, int32_t n_cells, riab_ovc_cells* meta_out,
                  float* out_host);
/* ObjectVectorCells.get_state at given positions; head_direction_dev (n_pos,2) for egocentric cells, NULL = [1,0]. */
int riab_ovc_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_ovc_cells* ovc,
                   const double* head_direction_dev, float* out_dev, int64_t ld_out, void* stream);

/* ----------------------------------------------------------- FeedForwardLayer
 * Neurons.py:2654-2847: firingrate = phi(sum_l W_l . I_l + biases), W_l the (n, n_in) weights of input layer l
 * (add_input, :2758-2795) and I_l its firing rates, over a batch of rows (agents or positions).  The activations are
 * the premade set of utils.activate (utils.py:919-1026); bespoke callables stay on the host side and are refused there. */
#define RIAB_FFL_MAX_INPUTS 4
typedef enum { RIAB_ACT_LINEAR = 0, RIAB_ACT_SIGMOID = 1, RIAB_ACT_RELU = 2, RIAB_ACT_TANH = 3, RIAB_ACT_RETANH = 4,
               RIAB_ACT_SOFTPLUS = 5 /* utils.activate's "softmax": gain * log(1 + exp(x - threshold)), utils.py:1017-1026 */
} riab_activation;
typedef struct {
  const float* w_dev;      /* riab_ffl_pack block of inputs[name]["w"] (Neurons.py:2781-2786): W_hi | W_lo */
  int32_t n_in;            /* input_layer.n (:2779) */
  int32_t k_pad;           /* filled by riab_ffl_pack: n_in rounded up to 32 */
  const float* rows_dev;   /* the input's firing rates, (n_rows, ld) f32 (Neurons.py:2819 / :2822); NULL = zeros (the
                              input has not been updated yet, Neurons.py:120).  riab_run: the row before its first step */
  int64_t ld;              /* row stride of rows_dev in floats, a multiple of 4 */
  int32_t population;      /* riab_run: index of the input in `pops` */
  int32_t lag;             /* riab_run: 0 = this step's row (input registered before the layer), 1 = the previous one
                              (registered at or after it, recurrence included): the reference's update order */
} riab_ffl_input;
typedef struct {
  int32_t n_cells;                  /* n */
  int32_t activation;               /* riab_activation */
  float act[4];                     /* sigmoid: max_fr, min_fr, mid_x, beta = log(19) / (width_x / 2)  (utils.py:961-979);
                                       relu / tanh / retanh / softplus: gain, threshold (utils.py:981-1026) */
  const float* bias_dev;            /* (n) f32 biases (Neurons.py:2749-2750, :2829-2832) */
  float* prime_dev;                 /* (n_rows, ld) f32 firingrate_prime = phi'(V) (Neurons.py:2839-2845) or NULL */
  int32_t n_inputs;
  int32_t reserved;
  riab_ffl_input inputs[RIAB_FFL_MAX_INPUTS];
} riab_ffl_cells;
/* Host-side packing of one float64 weight matrix w (n_cells, n_in), row-major, into the error-compensated float32
 * operand block: W_hi = tf32(w) then W_lo = tf32(float32(w) - W_hi), each (n_pad, k_pad) row-major with n_pad = n
 * rounded up to 8 and k_pad = n_in rounded up to 32, pads zero.  Fills meta->n_in / k_pad. */
int64_t riab_ffl_pack_floats(int32_t n_cells, int32_t n_in);
int riab_ffl_pack(const double* w_host, int32_t n_cells, int32_t n_in, riab_ffl_input* meta_out, float* out_host);

/* ------------------------------------------------------- Neurons.update extras
 * OU noise (Neurons.py:153-160) and spikes (Neurons.py:681-684) for a block of
 * rates already written to rates_dev.  noise_dev (A,N) f32 state (NULL when
 * noise_std == 0); spikes (A, 4*ceil(N/128)) uint32 words (layout: riab_rates_out.spikes_row), NULL to skip. */
typedef struct {
  float noise_std, noise_coherence_time;
  double dt;                /* the Agent's dt: the thinned spike stream's tables and the OU constants use it in float64 */
  uint64_t seed, step;
  int64_t id_offset;
  int32_t population_id;    /* distinguishes the Philox streams of populations of one Agent */
} riab_neuron_noise;

/* --------------------------------------------------------------- fused step
 * One launch = Agent.update for every agent + Neurons.update of ONE population
 * (motion -> rates [-> noise] [-> spikes] -> history row).  `cells_kind` selects
 * which of pc / gc / bvc / ovc is read. */
typedef enum { RIAB_CELLS_PLACE = 0, RIAB_CELLS_GRID = 1, RIAB_CELLS_BVC = 2, RIAB_CELLS_OVC = 3,
               RIAB_CELLS_FFL = 4, RIAB_CELLS_RSN = 5, RIAB_CELLS_KIN = 6, RIAB_CELLS_AVC = 7,
               RIAB_CELLS_TD = 8 /* riab_td_cells: a FeedForwardLayer learning by TD (ValueNeuron, SuccessorFeatures) */,
               RIAB_CELLS_PPPC = 9 /* riab_pppc_cells: PhasePrecessingPlaceCells */,
               RIAB_CELLS_PWN = 10 /* riab_pwn_cells: PlaneWaveNeurons */,
               RIAB_CELLS_NNN = 11 /* riab_nnn_cells: NeuralNetworkNeurons */
} riab_cells_kind;
typedef struct {
  float* rates_row;        /* (A, ld) f32: firing rates of this step (doubles as the history row) */
  int64_t ld;
  uint32_t* spikes_row;    /* (A, 4*ceil(N/128)) uint32 words, 16-byte aligned, or NULL.  Bit L of word 4B+i =
                            * spike of cell 128B + 4L + i (a warp's ballot of its lanes' i-th cell). */
  float* noise_state;      /* (A, ld) f32 OU noise state or NULL (noise_std == 0) */
  float* bvc_scratch;      /* (A, T) f32, BVC only */
} riab_rates_out;

/* Above RIAB_MAX_STEP_WALLS walls the motion kernel runs first, then the population's rate kernel. */
int riab_step_fused(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                    const riab_step_io* io, int32_t cells_kind, const void* cells /* riab_place_cells* etc. */,
                    const riab_neuron_noise* noise, const riab_rates_out* out, void* stream);

/* Neurons.update (Neurons.py:145-171) alone, for the agents' CURRENT positions
 * (agents->pos): rates [-> noise] [-> spikes].  Used for the 2nd, 3rd ... population
 * of an Agent after riab_step_fused / riab_agent_update moved it. */
int riab_neurons_update(const riab_agents* agents, const riab_env* env, int32_t cells_kind, const void* cells,
                        const riab_neuron_noise* noise, const riab_rates_out* out, void* stream);

/* FeedForwardLayer.get_state over n_rows input rows (ffl->inputs[i].rows_dev) -> out->rates_row (n_rows, ld) and
 * ffl->prime_dev, then OU noise and spikes like every population (noise NULL: rates only).  pos_dev (n_rows, 2) f64 or
 * NULL: rows whose x is NaN get zeros (+ noise) and keep their prime (Neurons.update, Neurons.py:163-164).  With
 * RIAB_CELLS_FFL, riab_neurons_update / riab_step_fused call this for the agents' rows and positions. */
int riab_ffl_rates(const riab_ffl_cells* ffl, int64_t n_rows, const double* pos_dev, const riab_neuron_noise* noise,
                   const riab_rates_out* out, void* stream);

/* ------------------------------------------------------- RandomSpatialNeurons
 * Neurons.py:2865-2954: rate[a, i] = sum_j k(pos_a, X_j) targets[j, i] / sum_j k(pos_a, X_j), k = exp(-d^2 / 2 l^2) with
 * the population's wall_geometry distance d.  k(pos, X) is a PlaceCells row (centres X, widths l, gaussian, [0, 1]);
 * the contraction with the targets is the FeedForwardLayer GEMM with its A operand generated in registers. */
typedef struct {
  riab_place_cells points;   /* the sample points: riab_place_pack block of X in the packed K order (riab_rsn_pack);
                                packed_dev / centres_dev (k_pad,2 f64, riab_rsn_pack's centres_out) set by the caller */
  const float* targets_dev;  /* T_hi | T_lo: riab_ffl_pack of targets.T, (n_pad8, k_pad) each */
  int32_t n_cells;           /* n */
  int32_t n_points;          /* |X| */
  int32_t k_pad;             /* filled by riab_rsn_pack: |X| rounded up to 32 */
  float min_fr, max_fr;      /* the targets' range (validation only: the targets are already scaled) */
  int32_t reserved;
} riab_rsn_cells;
/* Floats of the packed block: the sample-point block (riab_place_pack_floats(k_pad, n_inner_walls)) followed by the
 * targets block (riab_ffl_pack_floats(n_cells, n_points)); the targets block starts 16-byte aligned. */
int64_t riab_rsn_pack_floats(int32_t n_cells, int32_t n_points, int32_t n_inner_walls);
/* X (n_points,2) f64, targets (n_points, n_cells) f64 row-major, lengthscale l.  Packed position p of K stage s (32 points)
 * holds sample point s*32 + rsn_k(p % 32) so that a consumer thread's 8 fragment columns are 2 runs of 4 packed points;
 * positions past n_points repeat point 0 and are masked in the kernel.  centres_out: (k_pad,2) f64 in packed order. */
int riab_rsn_pack(const double* X_host, int32_t n_points, const double* targets_host, int32_t n_cells, double lengthscale,
                  const double* walls_host, int32_t n_walls, int32_t n_boundary_walls, const double* extent,
                  int32_t wall_geometry, riab_rsn_cells* meta_out, float* out_host, double* centres_out);
/* RandomSpatialNeurons.get_state(evaluate_at=None, pos=P): pos_dev (n_pos,2) f64 -> out_dev (n_pos, ld_out) f32; rows
 * whose x is NaN get zeros.  With RIAB_CELLS_RSN, riab_neurons_update / riab_step_fused / riab_run run the same kernel. */
int riab_rsn_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_rsn_cells* rsn, float* out_dev,
                   int64_t ld_out, void* stream);

/* ------------------------------------------- kinematic cells (RIAB_CELLS_KIN)
 * HeadDirectionCells (Neurons.py:2357-2485), VelocityCells (:2534-2583) and SpeedCell (:2586-2651): rates from the
 * agent's head direction, velocity or measured velocity, no position tuning.
 *   head direction: fr_i = von_mises(get_angle(d), mu_i, sigma_i, norm=1) (max_fr - min_fr) + min_fr      (:2466-2474)
 *                   d = head_direction, or velocity / |velocity| when use_velocity                        (:2428-2460)
 *   velocity:       the use_velocity head-direction rates times |velocity| inv_one_sigma_speed             (:2580-2582)
 *   speed:          |measured_velocity| inv_one_sigma_speed (max_fr - min_fr) + min_fr                     (:2641-2650)
 * utils.get_angle's 1e-6 eps (utils.py:258-260) is kept; a zero velocity gives NaN like the reference's 0/0. */
typedef enum { RIAB_KIN_HEAD_DIRECTION = 0, RIAB_KIN_VELOCITY = 1, RIAB_KIN_SPEED = 2 } riab_kin_variant;
typedef struct {
  int32_t n_cells;
  int32_t variant;               /* riab_kin_variant */
  int32_t use_velocity;          /* head direction: 1 = the normalised velocity replaces it (get_state(use_velocity=True));
                                    velocity cells: always 1 */
  int32_t reserved0;
  float min_fr, max_fr;
  double inv_one_sigma_speed;    /* 1 / (Agent.speed_mean + Agent.speed_std), taken at construction (:2567, :2625) */
  const float* packed_dev;       /* riab_kin_pack output */
  int32_t n_pad;                 /* filled by riab_kin_pack */
  int32_t reserved1;
} riab_kin_cells;
/* Floats of the packed block: cos(mu/2) | sin(mu/2) | k_q = sqrt(2 kappa log2(e)), kappa = 1/sigma^2 (utils.py:452), each
 * n_pad = n_cells rounded up to 128; pads and speed cells hold (1, 0, 0). */
int64_t riab_kin_pack_floats(int32_t n_cells);
/* preferred_angles / angular_tunings (n_cells) f64 radians (Neurons.py:2405-2409; NULL for RIAB_KIN_SPEED); computed in
 * float64, stored as float32.  Fills every field of cells_out but packed_dev. */
int riab_kin_pack(const double* preferred_angles, const double* angular_tunings, int32_t n_cells, int32_t variant,
                  int32_t use_velocity, float min_fr, float max_fr, double one_sigma_speed, riab_kin_cells* cells_out,
                  float* out_host);
/* get_state away from the agents' step: vec_dev (n_pos,2) f64 when vec_per_position, else one (2) vector for every row --
 * the head direction (use_velocity 0), the velocity (use_velocity 1) or, for speed cells, the velocity whose norm is the
 * speed -> out_dev (n_pos, ld_out) f32.  speed_scale: velocity cells' factor |Agent.velocity| / one_sigma_speed of every
 * row (Neurons.py:2581); a negative value takes each row's own |vec| inv_one_sigma_speed instead (vec = the agents'
 * velocities).  No noise, no NaN-position masking (get_state does neither). */
int riab_kin_rates(const double* vec_dev, int32_t vec_per_position, int64_t n_pos, double speed_scale,
                   const riab_kin_cells* cells, float* out_dev, int64_t ld_out, void* stream);

/* ------------------------------------------------ AgentVectorCells (RIAB_CELLS_AVC)
 * AgentVectorCells / FieldOfViewAVCs (Neurons.py:2151-2351): ObjectVectorCells whose single "object" is the position of
 * another Agent, with no type mask (:2242-2320):
 *   fr_i = gaussian(d; mu_d_i, sigma_d_i, norm=1) von_mises(bearing; mu_theta_i, sigma_theta_i, norm=1) (max_fr - min_fr) + min_fr
 *   d       = |pos - partner|, or 1000 when walls_occlude and an inner wall (walls[4:]) crosses the segment (:2235-2247)
 *   bearing = utils.get_angle(partner - pos) [- utils.get_angle(head_direction) when egocentric]        (:2248-2279)
 * The agents of a batch are paired row by row: row i sees partner row i, or partner row 0 when n_other == 1. */
typedef struct {
  int32_t n_cells;
  int32_t walls_occlude;         /* 1: wall_geometry "line_of_sight", 0: "euclidean" (:2189-2192) */
  int32_t egocentric;            /* reference_frame == "egocentric" */
  int32_t partner_is_self;       /* 1: the Agent is its own partner, each row reads its own (possibly just moved) position */
  float min_fr, max_fr;
  const float* packed_dev;       /* device block written by riab_avc_pack (riab_avc_pack_floats floats) */
  const double* other_pos_dev;   /* the partner's positions (n_other, 2) f64; NULL and partner_is_self == 0: no partner
                                    (tuning_type_agent is None), every rate is 0 (:2231-2232) */
  int64_t n_other;               /* 1 (every row sees row 0) or the number of rows */
  int32_t n_pad;                 /* filled by riab_avc_pack */
  int32_t reserved;
} riab_avc_cells;
/* Floats of the packed block: the riab_ovc_pack block without its type column, mu_d | s_d | cos(mu/2) | sin(mu/2) | k_q. */
int64_t riab_avc_pack_floats(int32_t n_cells);
/* tuning_angles / sigma_angles in radians (VectorCells attributes).  Fills n_cells and n_pad of meta_out. */
int riab_avc_pack(const double* tuning_distances, const double* tuning_angles, const double* sigma_distances,
                  const double* sigma_angles, int32_t n_cells, riab_avc_cells* meta_out, float* out_host);
/* AgentVectorCells.get_state at given positions: other_pos_dev (n_pos,2) f64 when other_per_position, else one (2)
 * partner position for every row (cells->other_pos_dev and partner_is_self are not read); head_direction_dev (n_pos,2)
 * for egocentric cells, NULL = [1,0] (:2263-2278).  No noise, no NaN-position masking. */
int riab_avc_rates(const double* pos_dev, int64_t n_pos, const double* other_pos_dev, int32_t other_per_position,
                   const riab_env* env, const riab_avc_cells* cells, const double* head_direction_dev, float* out_dev,
                   int64_t ld_out, void* stream);

/* ------------------------------------------------ TD learning (RIAB_CELLS_TD)
 * contribs/ValueNeuron.py:10-113 and contribs/SuccessorFeatures.py:12-49: a FeedForwardLayer whose update also keeps,
 * per agent row,
 *   deriv = (fr - fr_prev) / dt,  fr_prev <- fr                          (firingrate_deriv, ValueNeuron.py:66-71)
 *   e_l   <- dt I_l + (1 - dt / tau_e) e_l   for every input l           (eligibility traces, :72-81)
 * where I_l is the row the layer's contraction read (the layer's own new row for its self-recurrent input), and whose
 * learning step (update_weights, :83-104) applies the mean over the rows of every row's reference update:
 *   td   = reward + deriv - fr_prev / tau
 *   W_l += dt eta (sum_a outer(td_a * phi'_a, e_{a,l}) / n_rows) - eta dt L2 W_l
 * to float64 master weights, then rewrites the layer's W_hi | W_lo blocks (riab_ffl_pack of the new master, bit for
 * bit).  The contraction runs over the row (agent) axis in fixed-size chunks whose float64 partial tiles are summed in
 * a fixed order: no atomics, the same inputs give the same weights.
 *
 * Per-agent weights (per_agent_weights = 1): every row a is an independent learner with its own masters
 * w_master_dev[l] (A, n_cells, n_in) f64, and the layer's contraction reads them directly (k_td_forward_pa):
 *   V[a, j] = sum_l W_l[a, j, :] . I_l[a, :] + b_j   (float64 accumulation, then the layer's activation and phi')
 * update_weights applies each row's own reference update, nothing averaged:
 *   td   = reward + deriv - fr_prev / tau
 *   W_l[a] += (dt eta) outer(td_a phi'_a, e_{a,l}) - (eta dt L2) W_l[a]
 * elementwise in the reference's operation order (contribs/ValueNeuron.py:94-100), in non-contracting float64 from the
 * float32 td, phi' and traces.  There is no W_hi | W_lo block (ffl.inputs[l].w_dev is not read and may be NULL), no
 * scratch and no split of the agent axis. */
typedef struct {
  riab_ffl_cells ffl;                       /* the layer; ffl.inputs[l].w_dev is the W_hi | W_lo block the learning rewrites */
  float* fr_prev_dev;                       /* (A, ld) f32: firingrate of the last update (zeros before it and after reset) */
  float* deriv_dev;                         /* (A, ld) f32 firingrate_deriv */
  float* td_error_dev;                      /* (A, ld) f32 td_error (riab_td_reset zeroes it) */
  int64_t ld;                               /* row stride of the layer's rates, fr_prev, deriv and td_error (floats) */
  float* trace_dev[RIAB_FFL_MAX_INPUTS];    /* (A, trace_ld[l]) f32 eligibility trace of ffl.inputs[l] */
  int64_t trace_ld[RIAB_FFL_MAX_INPUTS];    /* multiple of 4, >= ffl.inputs[l].n_in */
  double* w_master_dev[RIAB_FFL_MAX_INPUTS];/* (n_cells, n_in) f64 row-major master weights of ffl.inputs[l];
                                               per_agent_weights: (A, n_cells, n_in), agent a's block at a n_cells n_in */
  double dt, tau, tau_e, eta, L2;           /* Agent.dt and the ValueNeuron params; tau_e > 0 */
  int32_t self_input;                       /* index of the input that is the layer itself (it reads fr_prev), or -1 */
  union {
    int32_t per_agent_weights;              /* 0: one weight matrix per input shared by the rows; 1: one per row (agent) */
    int32_t reserved;                       /* the field's former name */
  };
} riab_td_cells;
typedef enum { RIAB_TD_REWARD_SHARED = 0 /* (n_cells) f64, every row */, RIAB_TD_REWARD_ROWS = 1 /* (n_rows, ld) f32 */
} riab_td_reward_mode;
/* Number of agent chunks riab_td_learn splits the contraction of one input (n_in) into: float64 partial tiles of
 * n_cells x n_in each, summed in a fixed order.  Depends on the shapes only.  Shared weights only: the per-agent
 * update has no contraction over the agents. */
int64_t riab_td_splits(int32_t n_cells, int32_t n_in, int64_t n_rows);
/* Device scratch riab_td_learn needs for n_rows rows (bytes); 0 with per_agent_weights. */
int64_t riab_td_scratch_bytes(const riab_td_cells* cells, int64_t n_rows);
/* ValueNeuron.update_weights(reward) over n_rows rows: td -> td_error_out (n_rows, ld) f32, then every input's master
 * and W_hi | W_lo (shared weights), or each row's own masters (per_agent_weights, n_rows = the masters' A).  scratch:
 * riab_td_scratch_bytes device bytes, 16-byte aligned (may be NULL with per_agent_weights). */
int riab_td_learn(const riab_td_cells* cells, int64_t n_rows, const void* reward, int32_t reward_mode, float* td_error_out,
                  void* scratch, void* stream);
/* ValueNeuron.reset (:106-113): zero fr_prev, deriv, td_error and the traces of the rows whose mask byte is non-zero
 * (mask (A) uint8 device, NULL = every row). */
int riab_td_reset(const riab_td_cells* cells, int64_t n_rows, const uint8_t* mask, void* stream);
/* The per-agent layer's rates away from the agents' step (get_state at positions, for chosen agents): row r is
 *   out[r] = phi(sum_l W_l[weight_agent_of_row[r]] . I_l[input_row_of_row[r]] + b)
 * with I_l = cells->ffl.inputs[l].rows_dev (rows of ld ffl.inputs[l].ld; NULL = zeros).  A NULL map is the identity.
 * out_dev (n_rows, ld_out) f32; firingrate_prime, noise and spikes are not touched.  Needs per_agent_weights. */
int riab_td_rates_pa(const riab_td_cells* cells, int64_t n_rows, const int64_t* weight_agent_of_row_dev,
                     const int64_t* input_row_of_row_dev, float* out_dev, int64_t ld_out, void* stream);

/* ------------------------------------ PhasePrecessingPlaceCells (RIAB_CELLS_PPPC)
 * contribs/PhasePrecessingPlaceCells.py:66-119: at the agents, the PlaceCells rate of `place` times the theta modulation
 *   factor_i = von_mises(pi - s_i precess_fraction pi - phi, 0, sigma) 2 pi = exp(kappa cos x) / I0(kappa), kappa = 1/sigma^2
 *   phi = theta_freq (t % (1 / theta_freq)) 2 pi,  s_i = ((pos - c_i) . d) / sigma_i,  d = velocity / (1e-8 + |velocity|)
 *   sigma_i = the cell's width (riab_place_pack's widths), times 2 for "gaussian"
 * Rates are not bounded by max_fr (the factor peaks at exp(kappa) / I0(kappa)).  one_hot is refused. */
typedef struct {
  riab_place_cells place;        /* riab_place_pack of place_cell_centres / place_cell_widths; description != one_hot */
  double theta_freq;             /* Hz */
  double sigma;                  /* the von Mises spread sqrt(1 / kappa), as the reference stores it at construction */
  double precess_fraction;
  double t;                      /* Agent.t of the step (after its `t += dt`); riab_run: of the first step, the library
                                    advances it by `t += dt` per step */
} riab_pppc_cells;
/* PhasePrecessingPlaceCells.get_state(evaluate_at="agent"): pos_dev / velocity_dev (n_pos,2) f64, the agents' positions
 * and Agent.velocity -> out_dev (n_pos, ld_out) f32.  No noise, no NaN-position masking. */
int riab_pppc_rates(const double* pos_dev, const double* velocity_dev, int64_t n_pos, const riab_env* env,
                    const riab_pppc_cells* cells, float* out_dev, int64_t ld_out, void* stream);

/* ---------------------------------------------------- PlaneWaveNeurons (RIAB_CELLS_PWN)
 * contribs/PlaneWaveNeurons.py:63-91: phi_i = (2 pi / wavescale_i) ((phase_offset_i - pos) . w_i),
 *   rate_i = 0.5 (cos phi_i + 1) (max_fr - min_fr) + min_fr   (w as stored: not renormalised)
 * Rates lie between min_fr and max_fr; riab_run takes a lone PlaneWaveNeurons population as one launch like Place / Grid. */
typedef struct {
  int32_t n_cells;
  int32_t n_pad;           /* filled by riab_pwn_pack */
  float min_fr, max_fr;
  const float* packed_dev; /* riab_pwn_pack output, 16-byte aligned */
  int32_t phase_turns;     /* filled by riab_pwn_pack: 1 = wave vectors as float32 hi / lo pairs and phases in turns, for
                              the compensated phase of large |k| r_max (riab_pwn.cuh); 0 = radians */
  int32_t reserved;
} riab_pwn_cells;
int64_t riab_pwn_pack_floats(int32_t n_cells);
/* phase_offsets_host / w_host (N,2), wavescales_host (N) f64; extent the environment's.  phase_form: -1 chooses (turns when
 * max |2 pi w / wavescale| times the box's half-diagonal exceeds 40), 0 forces radians, 1 forces turns. */
int riab_pwn_pack(const double* phase_offsets_host, const double* w_host, const double* wavescales_host, int32_t n_cells,
                  const double* extent, int32_t phase_form, riab_pwn_cells* meta_out, float* out_host);
/* PlaneWaveNeurons.get_state at pos_dev (n_pos,2) f64 -> out_dev (n_pos, ld_out) f32 */
int riab_pwn_rates(const double* pos_dev, int64_t n_pos, const riab_env* env, const riab_pwn_cells* cells,
                   float* out_dev, int64_t ld_out, void* stream);

/* ------------------------------------------------ NeuralNetworkNeurons (RIAB_CELLS_NNN)
 * contribs/NeuralNetworkNeurons.py:74-104 for a module that is a chain of Linear layers and elementwise activations:
 *   h_0 = [I_0 | I_1 | ...] (the inputs' rates, concatenated in input order), h_l = act_l(W_l h_{l-1} + b_l), rates = h_L.
 * One launch per evaluation (riab_nnn.cuh, k_nnn): layer 1 is the FeedForwardLayer's error-compensated TF32 wgmma GEMM
 * over the gathered input rows; the hidden activations stay in shared memory and the later layers run in float32 FMA.
 * Limits of the fused kernel: 1..RIAB_NNN_MAX_LAYERS Linear layers, hidden widths (widths[1 .. n_layers-1]) of at most
 * RIAB_NNN_MAX_HIDDEN, at most RIAB_FFL_MAX_INPUTS input populations; the input count (widths[0]) and the output width
 * are unbounded.  Rows whose position x is NaN get zeros, then OU noise and spikes as for every population.  riab_run
 * treats the kind like a FeedForwardLayer (plain schedule, input rows by registration-order lag). */
#define RIAB_NNN_MAX_LAYERS 8
#define RIAB_NNN_MAX_HIDDEN 256
typedef enum { RIAB_NNN_IDENTITY = 0, RIAB_NNN_RELU = 1, RIAB_NNN_SIGMOID = 2 /* 1 / (1 + exp(-x)) */, RIAB_NNN_TANH = 3
} riab_nnn_activation;
typedef struct {
  int32_t n_cells;                            /* filled by riab_nnn_pack: widths[n_layers] */
  int32_t n_layers;                           /* Linear layers.  0: the rates were computed by the caller (a module the
                                                 kernel does not run) and sit in inputs[0].rows_dev (n_rows, ld, n_in =
                                                 n_cells): the library only masks NaN rows, adds noise and draws spikes */
  int32_t n_inputs;
  int32_t widths[RIAB_NNN_MAX_LAYERS + 1];    /* widths[0] = the sum of inputs[i].n_in, widths[l] = layer l's outputs */
  int32_t act[RIAB_NNN_MAX_LAYERS];           /* riab_nnn_activation applied after Linear layer l + 1 */
  const float* packed_dev;                    /* riab_nnn_pack block, 16-byte aligned */
  riab_ffl_input inputs[RIAB_FFL_MAX_INPUTS]; /* n_in, rows_dev, ld, population, lag as for a FeedForwardLayer; w_dev is
                                                 unused (layer 1's weights are in packed_dev) */
} riab_nnn_cells;
/* Floats of the packed block of `meta` (n_layers, widths, n_inputs, inputs[i].n_in set):
 *   for each input i, riab_ffl_pack of W_1's columns of that input (riab_ffl_pack_floats(widths[1], n_in_i) floats);
 *   b_1 (widths[1] rounded up to 8); then per layer l >= 2, W_l^T (widths[l-1], widths[l] rounded up to 8) and b_l. */
int64_t riab_nnn_pack_floats(const riab_nnn_cells* meta);
/* params_host: per Linear layer l = 1..n_layers, W_l (widths[l], widths[l-1]) f64 row-major then b_l (widths[l]) (zeros
 * for a Linear without bias).  meta in: n_layers, widths, act, n_inputs, inputs[i].n_in; out: n_cells, inputs[i].k_pad.
 * Refuses what the fused kernel does not run (the limits above). */
int riab_nnn_pack(const double* params_host, riab_nnn_cells* meta, float* out_host);
/* The network over n_rows input rows (cells->inputs[i].rows_dev) -> out->rates_row (n_rows, ld), then OU noise and spikes
 * (noise NULL: rates only); pos_dev (n_rows, 2) f64 or NULL: rows whose x is NaN get zeros.  With RIAB_CELLS_NNN,
 * riab_neurons_update / riab_step_fused call this for the agents' rows and positions. */
int riab_nnn_rates(const riab_nnn_cells* cells, int64_t n_rows, const double* pos_dev, const riab_neuron_noise* noise,
                   const riab_rates_out* out, void* stream);

/* ------------------------------------------------------------- multi-step run
 * `for _ in range(n_steps): Ag.update(); [Ns.update() for Ns in Ag.Neurons]`
 * (tests/test_advanced.py:21-23) without returning to the host between steps.
 * Population 0 is fused with the motion kernel, the others use riab_neurons_update; FeedForwardLayers
 * (RIAB_CELLS_FFL, RIAB_CELLS_TD with its trace pass, and RIAB_CELLS_NNN) run after every other population of the step, in index order,
 * reading ring rows (next + s - lag) of their inputs, and an Agent with one keeps this unskewed schedule.  A TD layer's
 * self-recurrent input reads its fr_prev.  riab_run never calls riab_td_learn.
 * History rows go to device rings: row (next + s) % rows for step s. */
typedef struct {
  int32_t kind;                 /* riab_cells_kind */
  const void* cells;            /* riab_place_cells* / riab_grid_cells* / riab_bvc_cells* / riab_ovc_cells* / riab_ffl_cells* /
                                   riab_rsn_cells* / riab_kin_cells* / riab_avc_cells* / riab_td_cells* / riab_pppc_cells* /
                                   riab_pwn_cells* / riab_nnn_cells* */
  riab_neuron_noise noise;      /* seed/step base; step is advanced per step */
  riab_rates_out out;           /* ld, noise_state, bvc_scratch; rates_row/spikes_row are set from the rings */
  float* rates_ring;            /* (rows, A, ld) f32 */
  uint32_t* spikes_ring;        /* (rows, A, 4*ceil(N/128)) or NULL */
  int32_t ring_rows;
  int32_t ring_next;            /* in: first row to write */
} riab_population;

typedef struct {
  float* ring;                  /* (rows, A, 8) f32 agent history rows, or NULL */
  int32_t ring_rows;
  int32_t ring_next;
} riab_agent_history;

/* Above RIAB_MAX_STEP_WALLS walls every step is the motion kernel, then each population (no whole-run or skewed launch). */
int riab_run(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm, const riab_step_io* io,
             const riab_population* pops, int32_t n_pops, const riab_agent_history* hist, int64_t n_steps,
             void* stream);

/* riab_run following a motion source (src == NULL or RIAB_MOTION_RANDOM: riab_run).  RIAB_MOTION_IMPORTED: step s
 * reads the trajectory at (t + dt + ... + dt) % t_max, the clock advanced by `t += dt` like Agent.update.  A single
 * Place / Grid / PlaneWave population runs as one launch where riab_run's would; otherwise every step is the motion kernel followed
 * by the populations' rates.  RIAB_MOTION_FORCED is refused: a forced position belongs to one step. */
int riab_run_src(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm, const riab_step_io* io,
                 const riab_motion_source* src, const riab_population* pops, int32_t n_pops,
                 const riab_agent_history* hist, int64_t n_steps, void* stream);

/* ------------------------------------------------------------ history analytics
 * utils.bin_data_for_histogramming (utils.py:544-589) over the device history rings, pooled over agents and steps:
 * count[ix, iy] = number of (step, agent) samples whose position falls into bin (ix, iy) -- np.histogram2d with the
 * explicit edges np.arange(extent[0], extent[1] + dx, dx) (right-most edge inclusive, outside samples dropped) --
 * and sum[(ix, iy), c] = the sum of cell c's rates over those samples.  rate map = sum / max(count, 1), laid out
 * `.T[::-1, :]` by the host like the reference (Neurons.py:483-490 plot_rate_map(method="history"),
 * Agent.py:956 plot_position_heatmap).  Counts are exact 64-bit integers and sums float64 (device atomics, so the
 * sums' last bits depend on the order the samples arrive in: about n * 2^-53 relative for n samples in a bin). */
typedef struct {
  const float* agent_ring;     /* (agent_ring_rows, A, 8) f32 history rows (pos.xy first), riab_agent_history.ring */
  int32_t agent_ring_rows;
  int32_t agent_row0;          /* ring row of the first step to use */
  const float* rates_ring;     /* (rates_ring_rows, A, ld) f32 or NULL (occupancy only) */
  int32_t rates_ring_rows;
  int32_t rates_row0;
  int64_t n_steps, n_agents, ld;
  int32_t n_cells;
  int32_t reserved;
} riab_history_view;
int riab_history_rate_maps(const riab_history_view* h, const double* edges_x_dev, int32_t n_edges_x,
                           const double* edges_y_dev, int32_t n_edges_y, double* sum_dev /* ((nx*ny), ld), zeroed here */,
                           uint64_t* count_dev /* (nx*ny), zeroed here */, void* stream);

/* Number of kernels launched by the library since load (bench.py "gpu_launches"). */
int64_t riab_launch_count(void);
/* cudaStreamSynchronize(stream): lets a host binding wait for its steps without another CUDA binding. */
int riab_stream_synchronize(void* stream);

/* -------------------------------------------------- host-buffer (e2e) entry
 * The reference-facing call with HOST buffers: copies drift (may be NULL) to the
 * device, runs riab_step_fused, copies pos (A,2 f64) back.  Buffers should be
 * pinned for the copies to be asynchronous.  staging_* are device scratch. */
int riab_step_fused_host(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                         riab_step_io* io, int32_t cells_kind, const void* cells,
                         const riab_neuron_noise* noise, const riab_rates_out* out,
                         const double* drift_host, double* drift_staging_dev,
                         double* pos_out_host, void* stream);

/* Agent.update with HOST buffers, for per-step control loops (the policy-control caller of
 * ratinabox/contribs/TaskEnvironment.py:399-408 passes one drift velocity per agent and reads the positions back):
 *   1. drift_host (A,2 f64, page-locked; may be NULL) is uploaded to drift_staging_dev by a copy engine on the
 *      library's side stream -- at once, i.e. while kernels queued earlier on `stream` (the previous step's rate
 *      kernels) still run;
 *   2. the motion kernel (riab_agent_update semantics; io->drift_velocity is set to the staging buffer) runs on
 *      `stream` after that copy;
 *   3. the new positions are copied to pos_out_host (page-locked; may be NULL) on the side stream, concurrently with
 *      whatever the caller queues on `stream` next (the rate kernels).
 * riab_positions_wait() blocks until step 3 of the LAST call on this device has finished (not the stream).  The next
 * kernel that overwrites agents->pos must be ordered after that copy: riab_positions_fence(stream) inserts the
 * dependency (riab_agent_update_host does it itself). */
int riab_agent_update_host(const riab_agents* agents, const riab_env* env, const riab_motion_params* prm,
                           riab_step_io* io, const double* drift_host, double* drift_staging_dev,
                           double* pos_out_host, void* stream);
int riab_positions_wait(void);
int riab_positions_fence(void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RIAB_B200_H */
