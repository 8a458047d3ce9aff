/* b2sim.h — C ABI of the H100-native batched physics step (libb2sim.so).
 *
 * Drop-in boundary: these entry points are what mjlab's `Simulation` class
 * (reference src/mjlab/sim/sim.py:94-198) needs from its physics backend. In the reference
 * that backend is the Python package mujoco_warp, reached from four call sites:
 *   mjwarp.put_model  sim.py:110      -> b2_create (model upload)
 *   mjwarp.put_data   sim.py:113-119  -> b2_create (nworld / nconmax / njmax sizing, Data alloc)
 *   mjwarp.step       sim.py:136,195  -> b2_step / b2_step_n
 *   mjwarp.forward    sim.py:139,187  -> b2_forward
 * plus the zero-copy field access that WarpBridge/TorchArray provide (sim_data.py:15-229)
 *   getattr(wp_data, name) / wp.to_torch -> b2_get_field
 * and the per-world model tiling of sim/randomization.py:20-55
 *   expand_model_fields -> b2_expand_model_field.
 * No torch types cross this boundary: plain pointers, sizes and a CUDA stream handle.
 * All functions return 0 on success, non-zero on error (message via b2_last_error()).
 * Nothing in b2_step/b2_forward allocates, synchronises or touches the host: they only enqueue
 * kernels on the given stream and are CUDA-graph capturable (an armed NaN guard's kernels write one word of mapped
 * host memory when they find a non-finite state; b2_nan_guard below).
 */
#ifndef B2SIM_H_
#define B2SIM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- model description handed in by the host (compiled by mjlab_b200.compiler) ---------- */
enum { B2_F64 = 0, B2_I32 = 1, B2_F32 = 2 };

typedef struct B2Array {
  const char* name; /* mjModel-style field name, e.g. "body_pos", "nq", "opt_timestep" */
  int32_t dtype;    /* B2_F64 or B2_I32 */
  int64_t n;        /* number of elements */
  const void* data; /* host pointer, valid during b2_create only */
} B2Array;

typedef struct B2ModelDesc {
  int32_t narray;
  const B2Array* arrays;
  double gravity[3];
} B2ModelDesc;

/* ---- tensor view returned for a Data / Model field ---------------------------------------- */
enum { B2_DATA = 0, B2_MODEL = 1 };

typedef struct B2Tensor {
  void* ptr;         /* device pointer */
  int32_t dtype;     /* B2_F32 or B2_I32 */
  int32_t ndim;      /* <= 4; shape[0] == nworld for Data and for expanded Model fields, else 1 */
  int64_t shape[4];
  int64_t stride[4]; /* in elements; rows are padded to 16 B so they can be bulk-copied (TMA) */
  int32_t device;    /* CUDA ordinal */
} B2Tensor;

typedef struct B2Stats {
  int32_t ncon_max, ncon_cap;   /* max contacts in any world / per-world capacity */
  int32_t nefc_max, nefc_cap;   /* max constraint rows in any world / njmax */
  int32_t overflow_worlds;      /* worlds that hit a capacity (contacts truncated, in pair order) */
  int32_t niter_max;            /* max Newton iterations used by any world in the last step */
  double ncon_mean, nefc_mean, niter_mean;
} B2Stats;

typedef struct b2_sim b2_sim;

/* Create a simulation: uploads the model, allocates Data for `nworld` worlds on `cuda_device`,
 * initialises qpos=qpos0 and runs one forward pass so every derived field is valid
 * (reference sim.py:106-107 relies on a forwarded MjData; SURVEY.md §8a S1b).
 *   ncon_per_world <= 0 : default capacity; njmax <= 0 : default.
 *   njmax is recorded (B2Stats.nefc_cap) but never truncates: the solver is matrix-free, so constraint rows
 *   need no storage and every contact within the contact capacity gets its rows (upstream drops rows past njmax). */
int b2_create(const B2ModelDesc* model, int nworld, int ncon_per_world, int njmax,
              int cuda_device, b2_sim** out);
int b2_destroy(b2_sim* sim);

/* Zero-copy view of a field. Pointers stay valid for the lifetime of the sim, except that
 * b2_expand_model_field re-points the named Model field.  The model-pointer table travels to the
 * kernels as a by-value launch parameter, so CUDA graphs captured before an expansion must be
 * re-captured (mjlab does: manager_based_rl_env.py:102-104; our Simulation does it lazily). */
int b2_get_field(b2_sim* sim, int which, const char* name, B2Tensor* out);
int b2_num_fields(b2_sim* sim, int which);
const char* b2_field_name(b2_sim* sim, int which, int index);

/* Tile a Model field to a real leading nworld dimension (reference randomization.py:20-55). */
int b2_expand_model_field(b2_sim* sim, const char* name, void* cuda_stream, B2Tensor* out);

/* Options, set and read back: "iterations", "ls_iterations", "tolerance", "ls_tolerance", "timestep",
 * "integrator", "solver" (1 = CG, 2 = Newton), "debug_outputs" (also write qfrc_bias, qfrc_smooth, qM,
 * qacc_smooth and qfrc_constraint), "sorted_dispatch" (heavy-first launch order, default on),
 * "dense_factor" (testing: always take the dense factorisation schedule instead of the dof-tree one),
 * "full_solver" (testing: Newton on all dofs even when a leading block suffices).
 * Read only: "smem_bytes_per_env", "maxcon", "resident_ctas", "reduced_block_cap".
 * Any other name is refused as an unknown option. */
int b2_set_option(b2_sim* sim, const char* key, double value);
int b2_get_option(b2_sim* sim, const char* key, double* value);

/* The hot path. */
int b2_step(b2_sim* sim, void* cuda_stream);              /* mjwarp.step    */
int b2_forward(b2_sim* sim, void* cuda_stream);           /* mjwarp.forward */
int b2_step_n(b2_sim* sim, int n, void* cuda_stream);     /* n sub-steps with ctrl held (decimation) */
/* forward() restricted to the worlds whose byte in `world_mask_dev` (device pointer, nworld bytes,
 * e.g. a torch.bool tensor) is non-zero: the partial-reset forward of manager_based_rl_env.py:128-132
 * without recomputing worlds that were not reset (SURVEY.md §8f-3). */
int b2_forward_masked(b2_sim* sim, const unsigned char* world_mask_dev, void* cuda_stream);

/* End-to-end call with HOST buffers (pinned or pageable): copies `ctrl` (nworld*nu floats, row
 * stride nu) to the device, runs `nsteps` sub-steps, copies qpos (nworld*nq) and qvel (nworld*nv)
 * back; asynchronous on `cuda_stream` when the host buffers are pinned. NULL outputs are skipped. */
int b2_step_host(b2_sim* sim, const float* ctrl_host, int nsteps, float* qpos_host,
                 float* qvel_host, void* cuda_stream);

/* Fused MDP glue of the velocity-tracking task around the step (SURVEY.md §8f-1..3): what
 * ManagerBasedRlEnv.step (manager_based_rl_env.py:106-147) does before and after the decimation loop for
 * tasks/velocity/velocity_env_cfg.py, as two launches. All pointers are device pointers. */
#define B2_VELENV_NU(nu) (16 + 9 + 2 * (nu))
#define B2_VELENV_NTERM 14 /* reward terms with an episode sum (B2VelEnvArgs.episode_sums) */
#define B2_VELENV_NSTAGE 8 /* stages of the command-velocity curriculum (B2VelEnvArgs.n_stage) */
#define B2_VELENV_NRESET 4 /* reset state terms (B2VelEnvArgs.reset_term) */
enum { B2_RESET_ROOT = 0, B2_RESET_JOINTS = 1 };
typedef struct B2VelResetTerm {
  int32_t kind, col, count;       /* B2_RESET_ROOT (count 12) / B2_RESET_JOINTS (count joints, <= 32) */
  int32_t joint[32];              /* JOINTS: actuated joint indices 0..nu-1 */
  float lo[12], span[12];         /* ROOT: per draw; JOINTS: [0] position scale, [1] velocity scale */
} B2VelResetTerm;
typedef struct B2VelEnvArgs {
  const float* action;            /* [n][nu] */
  const float* U;                 /* [n][B2_VELENV_NU(nu)] uniforms in [0,1): 0-1 reset xy, 2 yaw, 3-5 command, 6 heading
                                     target, 7 standing draw, 8 command timer, 9-10 push, 11 push timer, 12 terrain
                                     level redraw, 13-15 spare, 16.. observation noise (9 + 2 nu) */
  const float* default_qpos;      /* [nq] */
  const float* default_joint_pos; /* [nu] */
  const float* action_scale;      /* [nu] */
  const float* soft_lo;           /* [nu] */
  const float* soft_hi;           /* [nu] */
  float* env_origins;             /* [n][3] spawn origins; in/out with the terrain curriculum, else only read */
  int32_t* episode_length;        /* [n] in/out */
  float* last_action;             /* [n][nu] in/out */
  float* command;                 /* [n][3] in/out */
  float* push_time_left;          /* [n] in/out */
  float* obs;                     /* [n][9 + 3 nu + 3] out */
  float* reward;                  /* [n] out */
  unsigned char* terminated;      /* [n] out */
  unsigned char* truncated;       /* [n] out */
  unsigned char* done;            /* [n] out: mask for b2_forward_masked */
  float* cmd_time_left;           /* [n] in/out: command resampling timer (velocity_env_cfg.py:69 3..8 s) */
  float* heading_target;          /* [n] in/out: heading command (velocity_command.py:71-75) */
  unsigned char* is_standing;     /* [n] in/out: standing envs get a zero command (rel_standing_envs = 0.1) */
  float* critic;                  /* [n][9 + 3 nu + 3] out: the same terms without noise (PrivilegedCfg) */
  float* log_row;                 /* [n][3] out: (reward, terminated, truncated) packed for the rank-0 log gather */
  float step_dt, fall_angle, push_vel, push_lo, push_hi;
  int32_t max_episode_length;
  /* terrain-level curriculum (terrain_levels_vel, tasks/velocity/mdp/curriculums.py:18-52, and
   * TerrainImporter.update_env_origins, terrains/terrain_importer.py:186-201); curriculum = 0 leaves every field
   * below unread. On reset, before the new pose is written: d = |root_xy - origin_xy|, up = d > move_up_dist,
   * down = d < |command_xy| episode_length_s / 2 and not up; level += up - down; a level >= rows is redrawn as
   * min(floor(U[12] rows), rows - 1), any other is clipped at 0; env_origins = terrain_origins[level][type]. */
  const float* terrain_origins;   /* [rows][cols][3] sub-terrain spawn points */
  int32_t* terrain_levels;        /* [n] in/out: row of each env */
  const int32_t* terrain_types;   /* [n] column of each env */
  float* terrain_level_mean;      /* [1] out: mean of terrain_levels after the update (the curriculum's log value) */
  float move_up_dist, episode_length_s;
  int32_t rows, cols, curriculum;
  /* opt-in reward terms of the reference's velocity task (tasks/velocity/mdp/rewards.py:52-190) and shared penalties
   * (envs/mdp/rewards.py:22-127), with per-term episode sums (managers/reward_manager.py:61-89).  Terms, in the order
   * of the episode-sum columns (B2_VELENV_NTERM):
   *   0-4 the fixed terms: track_lin_vel_exp, track_ang_vel_exp, pose, dof_pos_limits, action_rate_l2 (weights 1, 1,
   *       1, -1, -0.1, not configurable);
   *   5 air_time, 6 feet_slide, 7 foot_clearance, 8 is_alive, 9 is_terminated, 10 joint_torques_l2, 11 joint_acc_l2,
   *   12 electrical_power_cost, 13 flat_orientation_l2.
   * A term at weight 0 is not evaluated and the air-time state does not advance.  reward = (fixed terms + sum of
   * w_i r_i) step_dt.  A foot is in contact when sensordata[adr] > 0; a geom's linear velocity is
   * cvel[3:6] - cvel[0:3] x (subtree_com[root_body] - geom_xpos).  Per-foot state of a done env is zeroed after its
   * reward.  episode_sums[w][i] += w_i r_i step_dt for all 14 terms; a done env's row is copied to finished_sums and
   * zeroed. */
  float weight[B2_VELENV_NTERM - 5]; /* of terms 5-13 */
  float air_threshold_min, air_threshold_max, air_command_threshold, air_command_scale_width;
  float clearance_target_height, clearance_std, clearance_tanh_mult;
  int32_t air_continuous;         /* reward_mode: 0 "on_landing", 1 "continuous" */
  int32_t air_hard_scale;         /* command_scale_type: 0 "smooth", 1 "hard" */
  int32_t n_air, n_slide, n_clear; /* feet of each term, <= 32 */
  int32_t root_body;              /* body whose subtree_com the geom velocities are taken about */
  const int32_t* air_sensor_adr;  /* [n_air] sensordata address of each foot's contact sensor */
  const int32_t* slide_sensor_adr; /* [n_slide] */
  const int32_t* slide_geom;      /* [n_slide] */
  const int32_t* slide_body;      /* [n_slide] body of each geom */
  const int32_t* clear_geom;      /* [n_clear] */
  const int32_t* clear_body;      /* [n_clear] */
  float* air_time;                /* [n][n_air] in/out: current air time */
  float* contact_time;            /* [n][n_air] in/out: current contact time */
  float* last_air_time;           /* [n][n_air] in/out: air time of the last landing */
  float* episode_sums;            /* [n][B2_VELENV_NTERM] in/out */
  float* finished_sums;           /* [n][B2_VELENV_NTERM] out: the sums of the episode a done env just ended */
  /* the command term as the reference's tasks configure it (UniformVelocityCommandCfg,
   * tasks/velocity/mdp/velocity_command.py:179-203), the command-velocity curriculum (commands_vel,
   * tasks/velocity/mdp/curriculums.py:55-74), per-joint posture widths (posture, envs/mdp/rewards.py:73-104) and the
   * command's metrics (velocity_command.py:43-62):
   *   A component is drawn as mid + (2u - 1) half (one IEEE product and one IEEE sum), the timer as resample_lo +
   *   resample_span u (resample_lo > 0), standing as u <= rel_standing; the heading command is
   *   clamp(heading_stiffness wrap(target - heading), ang_lo, ang_hi).
   *   n_stage > 0: counter = *step_counter + 1 is the step's common_step_counter; the lin_vel_x and ang_vel_z ranges
   *     of the step are those of the last stage s in list order with stage_step[s] < counter (the cfg's when none
   *     is).  b2_velenv_post advances *step_counter after the post kernel (one one-thread launch).
   *   The pose term is exp(-mean_j(d_j^2 posture_inv_std2[j])).
   *   Every env adds |cmd_xy - v_b,xy| / metric_steps and |cmd_z - w_b,z| / metric_steps to metric_xy / metric_yaw,
   *     from the command before this step's timer resample and the post-physics velocity.  A done env first moves its
   *     sums to finished_metrics and restarts them at 0; its first increment uses the fresh draw (before heading
   *     control and standing) and the post-reset state. */
  float cmd_mid[4], cmd_half[4];  /* lin_vel_x, lin_vel_y, ang_vel_z, heading: (lo + hi) / 2, (hi - lo) / 2 */
  float ang_lo, ang_hi;           /* ang_vel_z range */
  float heading_stiffness, rel_standing, resample_lo, resample_span;
  int32_t n_stage;                /* <= B2_VELENV_NSTAGE */
  int32_t stage_step[B2_VELENV_NSTAGE];
  float stage_mid[B2_VELENV_NSTAGE], stage_half[B2_VELENV_NSTAGE]; /* of the stage's range, as cmd_mid / cmd_half */
  float stage_lo[B2_VELENV_NSTAGE], stage_hi[B2_VELENV_NSTAGE];
  int32_t* step_counter;          /* [1] in/out: common_step_counter */
  const float* posture_inv_std2;  /* [nu] 1 / std^2 per joint */
  float* metric_xy;               /* [n] in/out: error_vel_xy of the running command episode */
  float* metric_yaw;              /* [n] in/out: error_vel_yaw */
  float* finished_metrics;        /* [n][2] out: (xy, yaw) of the episode a done env just ended */
  float metric_steps;             /* resampling_time_range[1] / step_dt */
  /* (appended) push_off = 1: no built-in push; push_time_left is neither advanced nor redrawn and push_vel is unread */
  int32_t push_off;
  /* (appended) reset state terms (reset_root_state_uniform, reset_joints_by_scale, envs/mdp/events.py:43-124), run in
   * table order in a reset env after the built-in reset (and the terrain curriculum), before the command and the
   * observations.  Draws: d_k = lo[k] + ev_V[w][col + k] span[k] (one fp32 product, then one fp32 sum).
   *   ROOT (12 draws: x y z roll pitch yaw of the pose, then of the velocity): qpos[0:3] = default_qpos[0:3] + d[0:3]
   *     + env_origins[w]; qpos[3:7] = default_qpos[3:7] * quat(euler xyz d[3:6]); qvel[0:3] = d[6:9];
   *     qvel[3:6] = R(qpos[3:7])^T d[9:12].
   *   JOINTS (count joints, joint[j] in 0..nu-1; draws: count position scales, then count velocity scales):
   *     qpos[7 + a] = clamp(default_joint_pos[a] lo[0]-span[0] draw, soft_lo[a], soft_hi[a]); qvel[6 + a] = 0 times
   *     the velocity draw (the default joint velocity is 0). */
  const float* ev_V;              /* [n][ev_v_width] the events' uniforms of this step (B2EventArgs.V) */
  int32_t ev_v_width, n_reset;    /* n_reset <= B2_VELENV_NRESET; 0 leaves the block unread */
  B2VelResetTerm reset_term[B2_VELENV_NRESET];
} B2VelEnvArgs;
int b2_velenv_pre(b2_sim* sim, const float* action, const float* default_joint_pos,
                  const float* action_scale, void* cuda_stream);
int b2_velenv_post(b2_sim* sim, const B2VelEnvArgs* args, void* cuda_stream);

/* ---- fused MDP glue of the motion-tracking task (BASELINE config C; reference tasks/tracking/tracking_env_cfg.py,
 * tasks/tracking/mdp/commands.py:283-388) ------------------------------------------------------------------------
 * post1 runs after the sub-steps (terminations, rewards, RSI resets, clip time step) and leaves the mask for
 * b2_forward_masked; post2 runs after that forward (anchor-relative targets, interval push, observations).
 * Per-step uniforms U[n][B2_TRACKENV_NU(nu)]: with S = 13 + nu, [0, S) reset block (0 clip frame, 1-6 pose noise,
 * 7-12 velocity noise, 13.. joint noise), [S, 2S) the same for envs that ran off the clip, [2S, 2S+7) push (6
 * velocity + timer), then observation noise: anchor pos 3, anchor ori 6, base lin 3, base ang 3, joint pos nu, joint vel nu.
 * Start frames of resets and clip restarts (B2TrackEnvArgs.adaptive) come from the block's first uniform u:
 *   B2_START_UNIFORM   floor(u (T-1));
 *   B2_START_ADAPTIVE  the failure-bin sampler of commands.py:256-297: bin = first b with cdf[b] > u, frac = its
 *                      position inside that bin's CDF step, frame = floor((bin + frac) / nbins (T-1));
 *   B2_START_FIRST     frame 0 (disable_adaptive_sampling, the reference's play mode). */
#define B2_TRACKENV_NU(nu) (48 + 4 * (nu))
enum { B2_START_UNIFORM = 0, B2_START_ADAPTIVE = 1, B2_START_FIRST = 2 };
typedef struct B2TrackEnvArgs {
  const float* action;            /* [n][nu] */
  const float* U;                 /* [n][B2_TRACKENV_NU(nu)] */
  const float* default_joint_pos; /* [nu] */
  const float* soft_lo;           /* [nu] */
  const float* soft_hi;           /* [nu] */
  const float* env_origins;       /* [n][3] */
  const float* m_joint_pos;       /* motion clip, T frames: [T][nu] */
  const float* m_joint_vel;       /* [T][nu] */
  const float* m_body_pos;        /* [T][nb][3] */
  const float* m_body_quat;       /* [T][nb][4] */
  const float* m_body_lin;        /* [T][nb][3] */
  const float* m_body_ang;        /* [T][nb][3] */
  const int32_t* body_idx;        /* [nb] engine body ids of the tracked bodies */
  const int32_t* ee_idx;          /* [nee] end effectors, as indices into the tracked bodies */
  int64_t* time_steps;            /* [n] in/out: clip frame */
  int32_t* episode_length;        /* [n] in/out */
  float* last_action;             /* [n][nu] in/out */
  float* push_time_left;          /* [n] in/out */
  float* body_pos_rel;            /* [n][nb][3] in/out: anchor-relative target positions */
  float* body_quat_rel;           /* [n][nb][4] in/out */
  float* reward;                  /* [n] out */
  unsigned char* terminated;      /* [n] out */
  unsigned char* truncated;       /* [n] out */
  unsigned char* mask;            /* [n] out: envs whose state was rewritten (reset or clip restart) */
  float* log_row;                 /* [n][3] out */
  float* obs;                     /* [n][5 nu + 15] out */
  float* critic;                  /* [n][5 nu + 15 + 9 nb] out */
  float pose_range[12], vel_range[12]; /* (lo, hi) x 6 */
  float step_dt, jp_lo, jp_hi, push_lo, push_hi;
  int32_t nb, nee, anchor, T, self_collision_adr, root_body, max_episode_length;
  /* start-frame sampler; a zeroed tail is B2_START_UNIFORM and leaves every field below unread */
  const float* adaptive_kernel;   /* [adaptive_kernel_size] smoothing weights lambda^i / sum (commands.py:106-110) */
  float* cdf;                     /* [nbins] in/out: CDF of the start-bin distribution post1 draws from */
  float* bin_fail_ema;            /* [nbins] in/out: EMA of terminations per bin (bin_failed_count) */
  float* bin_fail_cur;            /* [nbins] in/out: terminations per bin in this env step (_current_bin_failed) */
  float* metrics;                 /* [3] out: normalised entropy, top-1 probability, top-1 bin / nbins of the
                                     distribution this env step's draws used (1, p, b / nbins for one bin) */
  float adaptive_alpha, adaptive_uniform_ratio;
  int32_t nbins, adaptive, adaptive_kernel_size;
  /* the task as a cfg class configures it (tracking_env_cfg.py:88-278, tasks/tracking/config/g1/flat_env_cfg.py) and
   * the episode logs of its managers.  The RSI ranges are pose_range / vel_range above.
   * Reward terms, in the order of the episode-sum columns (B2_TRACKENV_NREW): 0 motion_global_root_pos,
   * 1 motion_global_root_ori, 2 motion_body_pos, 3 motion_body_ori, 4 motion_body_lin_vel, 5 motion_body_ang_vel
   * (exp(-err / std2[i])), 6 action_rate_l2, 7 joint_limit, 8 self_collisions.  A term at weight 0 is not evaluated.
   * reward = (sum of w_i r_i) step_dt.
   * Terminations, in the order of term_flags (B2_TRACKENV_NTERM): 0 time_out, 1 anchor_pos, 2 anchor_ori,
   * 3 ee_body_pos; term_on[k] = 0 removes term k + 1.
   * policy_state_estimation = 0 drops motion_anchor_pos_b and base_lin_vel from the policy row ([n][5 nu + 9]); their
   * noise columns of U are still drawn.  policy_corruption = 0 writes the policy terms without noise.  push_on = 0:
   * no push, push_time_left untouched.
   * The episode logs are the five arrays at the end, all set or all null (no logs).  episode_sums[w][i] +=
   * w_i r_i step_dt; term_flags[w] holds every env's flags of this step.  Motion errors (B2_TRACKENV_NMETRIC,
   * commands.py:221-255): 0 anchor_pos, 1 anchor_rot, 2 anchor_lin_vel, 3 anchor_ang_vel, 4 body_pos, 5 body_rot,
   * 6 body_lin_vel, 7 body_ang_vel (means of norms over the tracked bodies), 8 joint_pos, 9 joint_vel (norms over the
   * joints).  An env that is not done takes them in post1 at its frame before the clip steps; a done env in post2,
   * after the forward, at frame max(time_steps - 1, 0) against the relative targets of the previous post2.  A done
   * env's episode_sums and motion_metrics rows move to finished_sums / finished_metrics in post1 (the episode sums
   * restart at 0). */
  float weight[9], std2[6];       /* B2_TRACKENV_NREW weights; std^2 of reward terms 0-5 */
  float term_threshold[3];        /* anchor_pos, anchor_ori, ee_body_pos */
  int32_t term_on[3];
  float push_range[12];           /* (lo, hi) x 6 of push_by_setting_velocity */
  int32_t push_on, policy_state_estimation, policy_corruption;
  float* episode_sums;            /* [n][B2_TRACKENV_NREW] in/out */
  float* finished_sums;           /* [n][B2_TRACKENV_NREW] out */
  float* term_flags;              /* [n][B2_TRACKENV_NTERM] out: 1 where the term fired this step */
  float* motion_metrics;          /* [n][B2_TRACKENV_NMETRIC] in/out */
  float* finished_metrics;        /* [n][B2_TRACKENV_NMETRIC] out */
} B2TrackEnvArgs;
#define B2_TRACKENV_NREW 9
#define B2_TRACKENV_NTERM 4
#define B2_TRACKENV_NMETRIC 10
int b2_trackenv_post1(b2_sim* sim, const B2TrackEnvArgs* args, void* cuda_stream);
int b2_trackenv_post2(b2_sim* sim, const B2TrackEnvArgs* args, void* cuda_stream);
/* B2_START_ADAPTIVE only, between post1 and the masked forward (one CTA): metrics of the distribution post1 drew
 * from, bin_fail_ema = alpha bin_fail_cur + (1 - alpha) bin_fail_ema, bin_fail_cur = 0, then the CDF of the next
 * env step's distribution p ~ conv1d(replicate_pad(bin_fail_ema + ratio / nbins), kernel), prefix-summed in a fixed
 * order (run-to-run deterministic). */
int b2_trackenv_bins(b2_sim* sim, const B2TrackEnvArgs* args, void* cuda_stream);

/* ---- clip, scale and history of the observation groups (the reference's ObservationManager,
 * managers/observation_manager.py:153-188, with its CircularBuffer, utils/buffers/circular_buffer.py) ---------------
 * Runs after the env's post kernel (b2_velenv_post, b2_trackenv_post2) on the group rows it wrote, one launch for every
 * group.  For element j of term t of group g in env w:
 *   v = frame[w][src + j], clamped to [lo, hi] when clip = 1, then times scale[t.scale + j] when t.scale >= 0 (one
 *   IEEE fp32 product, subnormals kept);
 *   the term's frames sit in out[w] at columns dst + k stride + j, k = 0 (oldest) .. max(frames, 1) - 1 (newest):
 *   every frame moves one slot older and v is written into the newest; an env whose terminated or truncated byte is
 *   set (the reference's reset_buf) gets v in every slot.
 * The terms tile the frame row in order (src of term 0 is 0, each next src is the previous src + dim, the last ends at
 * frame_width), and their frames tile the out row: every column of out is written by exactly one element.
 *
 * Noise (the block appended at the end of B2ObsHistArgs; ObservationTermCfg.noise, utils/noise/).  A group whose
 * noise[g].source is set reads v from source[w][col + j] (the term's noise-free values) instead of frame, and before
 * the clip, for a term with a bias code (NoiseModelWithAdditiveBias):
 *   when w's terminated or truncated byte is set, bias[w][src + j] = redraw(bias[w][src + j]) and is stored;
 *   v = noise(v) + bias[w][src + j]   (a term without a bias: v = noise(v); with neither code: v as loaded).
 * A noise of class c, operation op, parameter rows p0, p1 (param[p0 + j], param[p1 + j]) and draw r is, in IEEE fp32
 * with one rounding per operation (no contraction, subnormals kept):
 *   CONSTANT: x = p0 (bias);  UNIFORM: x = r p1 + p0 (r = W[w][draw + j], p1 the span, p0 n_min);
 *   GAUSSIAN: x = r p1 + p0 (r = N[w][draw + j], p1 std, p0 mean);
 *   ADD: v + x;  SCALE: v x;  ABS: x (0 + x for CONSTANT).
 * The bias redraw is the same with the bias fields, applied to the old bias; with bias_shared = 1 every element draws
 * from column bias_draw (so the term's copies of a shared bias stay equal).  A term with a code needs the group's
 * source (and bias row for a bias code), its columns inside the source row, its parameter rows inside param, its draws
 * inside W or N, and W / N themselves. */
#define B2_OBSHIST_NTERM 16  /* terms per group */
#define B2_OBSHIST_NGROUP 2  /* groups per launch (policy, critic) */
enum { B2_NOISE_NONE = 0, B2_NOISE_CONSTANT = 1, B2_NOISE_UNIFORM = 2, B2_NOISE_GAUSSIAN = 3 };
enum { B2_NOISE_ADD = 0, B2_NOISE_SCALE = 1, B2_NOISE_ABS = 2 };
typedef struct B2ObsHistTerm {
  int32_t src;                    /* first column of the term in the frame row */
  int32_t dim;                    /* elements of one frame of the term, >= 1 */
  int32_t frames;                 /* history length, >= 0; 0: no history (one frame, as 1) */
  int32_t dst;                    /* column of the term's oldest frame in the out row */
  int32_t stride;                 /* columns from one frame of the term to the next */
  int32_t scale;                  /* offset of the term's dim factors in B2ObsHistArgs.scale; -1: not scaled */
  int32_t clip;                   /* 1: clamp to [lo, hi] (finite, lo <= hi); 0: no clip */
  float lo, hi;
} B2ObsHistTerm;
typedef struct B2ObsHistGroup {
  const float* frame;             /* [n][frame_width] the group's row as the post kernel wrote it (noise applied) */
  float* out;                     /* [n][out_width] in/out: the group's output, which is its history */
  int32_t frame_width, out_width, nterm;
  B2ObsHistTerm term[B2_OBSHIST_NTERM];
} B2ObsHistGroup;
typedef struct B2ObsNoiseTerm {
  int32_t col;                    /* first column of the term in the group's source row */
  int32_t noise, noise_op;        /* B2_NOISE_* class (NONE: no noise) and operation of the per-step noise */
  int32_t noise_p0, noise_p1;     /* offsets of its parameter rows in param (p1 unused by CONSTANT) */
  int32_t noise_draw;             /* first column of its draws in W (UNIFORM) or N (GAUSSIAN) */
  int32_t bias, bias_op;          /* class (NONE: no bias) and operation of the bias redraw */
  int32_t bias_p0, bias_p1, bias_draw;
  int32_t bias_shared;            /* 1: one draw per term; 0: one per element */
} B2ObsNoiseTerm;
typedef struct B2ObsNoiseGroup {
  const float* source;            /* [n][source_width] noise-free term values; null: the group reads frame, no noise */
  float* bias;                    /* [n][frame_width] in/out: the bias of element e at column e */
  int32_t source_width, pad_;
  B2ObsNoiseTerm term[B2_OBSHIST_NTERM];
} B2ObsNoiseGroup;
typedef struct B2ObsHistArgs {
  const unsigned char* terminated; /* [n] this env step's terminations */
  const unsigned char* truncated;  /* [n] this env step's time-outs */
  const float* scale;             /* [nscale] per-element factors of the scaled terms; may be null when nscale = 0 */
  int32_t nscale, ngroup;         /* 1 <= ngroup <= B2_OBSHIST_NGROUP */
  B2ObsHistGroup group[B2_OBSHIST_NGROUP];
  /* noise (all zero: none) */
  const float* W;                 /* [n][nW] this env step's uniforms of the noise; may be null when no term draws */
  const float* N;                 /* [n][nN] this env step's standard normals of the noise */
  const float* param;             /* [nparam] the terms' per-element parameter rows */
  int32_t nW, nN, nparam;
  B2ObsNoiseGroup noise[B2_OBSHIST_NGROUP];  /* noise[g] belongs to group[g] */
} B2ObsHistArgs;
int b2_obs_history(b2_sim* sim, const B2ObsHistArgs* args, void* cuda_stream);

/* ---- reset and interval randomize_field events (the reference's EventManager.apply("reset") / apply("interval") /
 * reset, managers/event_manager.py:76-167, with envs/mdp/events.py:212-397) ------------------------------------------
 * One launch per env step, after the env's post kernel (b2_velenv_post, b2_trackenv_post1 / bins) and before the
 * masked forward.  In env w the terms run in table order; a term fires when
 *   mode RESET:    w's terminated or truncated byte is set (the reference's reset_buf);
 *   mode INTERVAL: t = timers[k][w] (k: the term's rank among the interval terms) takes t -= step_dt; it fires when
 *                  t < 1e-6, and t is then redrawn, t = lo + V[w][col + count] span.  Every step stores t; a reset
 *                  does not redraw it (EventManager.reset redraws only the timers of class-based terms).
 * When it fires, entry j of its count (element, axis) entries, e = elem[first + j] (first: the counts of the terms
 * before it), draws x = lo + V[w][col + j] span (one fp32 product, then one fp32 sum); LOG_UNIFORM takes exp(x).  It
 * then writes row[e.offset] = row + x (ADD), row x (SCALE) or x (ABS), where row is world w's row of model field
 * `field`, the field's index in the library's model-field table (b2_field_name(sim, B2_MODEL, field)).  The field must
 * be a float model field with a per-world copy (b2_expand_model_field) and every offset inside its row. */
#define B2_EVENTS_NTERM 16   /* reset and interval terms per launch */
#define B2_EVENTS_NSTATE 8   /* state terms per launch (B2EventArgs.state) */
enum { B2_EVENT_RESET = 0, B2_EVENT_INTERVAL = 1 };
enum { B2_EVENT_ADD = 0, B2_EVENT_SCALE = 1, B2_EVENT_ABS = 2 };
enum { B2_EVENT_UNIFORM = 0, B2_EVENT_LOG_UNIFORM = 1 };
typedef struct B2EventTerm {
  int32_t mode, operation, distribution;
  int32_t field;                  /* index in the model-field table */
  int32_t count;                  /* (element, axis) entries, >= 1 */
  int32_t col;                    /* first V column: count draws, then (INTERVAL) the timer's redraw */
  float interval_lo, interval_span; /* INTERVAL: the timer's draw lo + u span */
} B2EventTerm;
typedef struct B2EventElem {
  int32_t offset;                 /* element index in the world's row of the field (element * width + axis) */
  float lo, span;                 /* the draw lo + u span (LOG_UNIFORM: of the logarithm) */
} B2EventElem;
enum { B2_EVENT_PUSH = 0, B2_EVENT_WRENCH = 1 };
typedef struct B2EventStateTerm {
  int32_t kind, mode;             /* B2_EVENT_PUSH / B2_EVENT_WRENCH; B2_EVENT_RESET / B2_EVENT_INTERVAL */
  int32_t col, count;             /* first V column; PUSH: 6, WRENCH: bodies */
  int32_t first, timer;           /* WRENCH: first entry of bodies; INTERVAL: row of timers */
  float lo[2], span[2];           /* WRENCH: force (0) and torque (1) draws */
  float lo6[6], span6[6];         /* PUSH: the draw of each axis */
  float interval_lo, interval_span; /* INTERVAL: the timer's draw lo + u span */
} B2EventStateTerm;
typedef struct B2EventArgs {
  const unsigned char* terminated; /* [n] this env step's terminations */
  const unsigned char* truncated;  /* [n] this env step's time-outs */
  const float* V;                 /* [n][v_width] this env step's uniforms of the events */
  float* timers;                  /* [ninterval][n] in/out: time left of each interval term */
  const B2EventElem* elem;        /* [nelem] the terms' entries, term by term */
  int32_t v_width, ninterval, nelem, nterm;
  float step_dt;
  B2EventTerm term[B2_EVENTS_NTERM];
  /* State terms (push_by_setting_velocity, apply_external_force_torque, envs/mdp/events.py:127-164), run after the
   * terms above, in table order.  They fire as the terms above do (mode RESET or INTERVAL; the timer of an INTERVAL
   * state term is row `timer` of timers, a row no term above uses).
   *   clear_xfrc: a reset env's xfrc_applied row is zeroed first (Entity.reset -> clear_state).
   *   WRENCH: `count` bodies, bodies[first .. first + count); force axis a of body j is lo[0] + V[w][col + 3 j + a]
   *     span[0], torque axis a is lo[1] + V[w][col + 3 count + 3 j + a] span[1]; they are written to
   *     xfrc_applied[w][bodies[first + j]][a] and [3 + a].  The timer's redraw is column col + 6 count.
   *   PUSH: count = 6; d_k = lo6[k] + V[w][col + k] span6[k] (x y z roll pitch yaw).  The root's world velocity
   *     (lin, ang) is taken from cvel, xpos and subtree_com of root_body (compute_velocity_from_cvel) with its
   *     orientation xquat[root_body], or, in an env whose `refreshed` byte is set (its state was rewritten this step
   *     and the env's masked forward after this launch recomputes it), from qvel[0:3] and R(q) qvel[3:6] with q the
   *     normalised qpos[3:7].  Then qvel[0:3] = lin + d[0:3] and qvel[3:6] = R(q)^T (ang + d[3:6]).  The timer's
   *     redraw is column col + 6.
   * (appended to B2EventArgs: every offset above is unchanged) */
  const unsigned char* refreshed; /* [n] PUSH: envs the masked forward after this launch recomputes */
  const int32_t* bodies;          /* [nbodies] WRENCH: body ids, term by term */
  int32_t nstate, nbodies, clear_xfrc, root_body;
  B2EventStateTerm state[B2_EVENTS_NSTATE];
} B2EventArgs;
int b2_events(b2_sim* sim, const B2EventArgs* args, void* cuda_stream);

/* ---- NaN guard (the reference's NanGuard, utils/nan_guard.py, on the device) -------------------------------------
 * Armed (flags = B2_NAN_GUARD_ON), every sub-step of b2_step / b2_step_n also
 *   records, before the sub-step, the qpos / qvel of worlds 0..ncapture-1 as its entry of a ring that keeps the last
 *   buffer_size entries (sub-steps are numbered from 0 at arming), and
 *   checks, after it, qpos, qvel, qacc and qacc_warmstart of every world (their nq / nv columns) for NaN / Inf.
 * The first sub-step that finds one is the detection sub-step: its non-finite worlds are flagged, the host-visible word
 * (b2_nan_guard_word) becomes 1, and the ring and flags are frozen, so the guard fires once.  This is stream work of the
 * calls (one launch before the call's first sub-step and one per sub-step and partition after it): a CUDA graph
 * captured while armed carries it.  While armed, b2_step_n's two partitions join every 8 sub-steps.
 * Arming (re)starts the guard on fresh buffers: graphs captured before must be re-captured to see them.  flags = 0
 * disarms: no launch and no allocation from then on (the default; outputs are those of a sim never armed).  Arming
 * refuses ncapture outside [1, nworld] and buffer_size < 1; it synchronises the device (not capturable). */
#define B2_NAN_GUARD_ON 1
int b2_nan_guard(b2_sim* sim, int ncapture, int buffer_size, int flags);
/* Host address of the guard's word (0, or 1 once a non-finite state was found), readable without synchronising;
 * NULL when disarmed. */
const volatile int32_t* b2_nan_guard_word(b2_sim* sim);
/* Synchronises `cuda_stream` and reads the guard: *detected = the detection sub-step d, or -1.  When d >= 0 and the
 * buffers are non-NULL: states[k - first][w][0:nq] = qpos and [nq:nq+nv] = qvel of world w before sub-step k, for
 * k = first .. d (first = max(0, d - buffer_size + 1), w < ncapture); flags[w] = 1 for the worlds non-finite after d. */
int b2_nan_guard_read(b2_sim* sim, void* cuda_stream, int64_t* detected, float* states, unsigned char* flags);

/* ---- offscreen frames (the reference's OffscreenRenderer, viewer/offscreen_renderer.py, by ray casting) ------------
 * One frame of the scene as the last step or forward left it, enqueued on `cuda_stream`; it reads Data and Model and
 * writes only the output buffers.  Drawn: every geom welded to the world once (world 0's values), and the other geoms
 * of worlds 0 .. min(noverlay, nworld) - 1 and of env_idx; not drawn: mesh geoms and geoms with alpha 0.  Camera (a
 * MuJoCo free or tracking camera): forward f = (cos el cos az, cos el sin az, sin el), eye = target - distance f, z up,
 * vertical field of view 45 degrees, one ray through each pixel centre.  Outputs are row-major from the top row:
 *   rgb   [height][width][3] uint8, required;
 *   depth [height][width] float, distance along f, +inf for the background (null: not written);
 *   seg   [height][width][2] int32 (world, geom), (-1, -1) for the background; welded geoms report world 0 (null: not
 *         written).
 * Shading and its constants: DESIGN.md §4.  The first call on a sim builds the list of drawable geoms (it synchronises
 * the device: not capturable); later calls only launch.  Refused: a size outside 1..4096, env_idx outside
 * [0, nworld), noverlay < 0, track_body outside [-1, nbody), a null rgb.
 *
 * Decoration (the debug visualisers: command arrows, a ghost of the robot), one translucent layer over the scene; zero
 * fields mean none.  The nearest decoration item the ray enters before the scene's hit is shaded without shadows and
 * blended, byte = floor(255 (a c_d + (1 - a) c_o) + 1/2), over the scene's colour c_o; decoration casts no shadow and
 * is not in depth or seg.  A frame with decoration is two launches: the scene, with the outputs a frame without
 * decoration has, then the decoration over the pixels it covers.
 *   decor      device array of ndecor arrow records of 12 floats: from[3], to[3], width w, rgba[4], padding.  An
 *              arrow is a cylinder shaft of radius w with flat caps and a solid cone head of base radius 2w, length
 *              min(L/2, 4w) and apex at `to` (L = |to - from|); not drawn when L < 1e-6 or alpha is 0.  Refused:
 *              ndecor outside [0, 64], a null decor with ndecor > 0.
 *   ghost_xpos, ghost_xmat  device geom poses [ngeom][3], [ngeom][9] of one configuration of this model (null: no
 *              ghost); the drawable geoms of bodies not welded to the world are drawn there in ghost_rgba, with world
 *              env_idx's sizes.  Refused: one of the two null, ghost_rgba outside [0, 1] or not finite. */
typedef struct B2RenderArgs {
  int32_t width, height;          /* pixels, 1..4096 */
  float lookat[3];                /* camera target when track_body is -1 */
  int32_t track_body;             /* >= 0: the target is subtree_com of this body in world env_idx (read on the device) */
  float distance, azimuth, elevation; /* metres, degrees, degrees */
  int32_t env_idx;                /* the main world */
  int32_t noverlay;               /* worlds 0 .. noverlay - 1 are drawn too (the reference draws 32) */
  int32_t shadows;                /* 1: one shadow ray per lit pixel toward the directional light */
  int32_t brute;                  /* measurement: 1 casts every ray against every geom, without the tile cull */
  unsigned char* rgb;
  float* depth;
  int32_t* seg;
  const float* decor;             /* [ndecor][12] arrow records (device), or null */
  int32_t ndecor;
  const float* ghost_xpos;        /* [ngeom][3] (device), or null: no ghost */
  const float* ghost_xmat;        /* [ngeom][9] (device) */
  float ghost_rgba[4];
} B2RenderArgs;
int b2_render(b2_sim* sim, const B2RenderArgs* args, void* cuda_stream);

/* Diagnostics (synchronises `cuda_stream`). */
int b2_stats(b2_sim* sim, void* cuda_stream, B2Stats* out);
/* Number of kernels this library has launched for `sim` since creation. */
int64_t b2_launch_count(b2_sim* sim);
/* Algorithmic bytes of one step for the roofline (DESIGN.md): solver stage and whole step,
 * evaluated with the mean nefc of the last step. */
int b2_algorithmic_bytes(b2_sim* sim, void* cuda_stream, double* solver_bytes, double* step_bytes);

const char* b2_last_error(void);
const char* b2_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B2SIM_H_ */
