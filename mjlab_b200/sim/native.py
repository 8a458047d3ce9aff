"""ctypes binding of libb2sim.so (the C ABI declared in include/b2sim.h)."""

from __future__ import annotations

import ctypes
import math
import os
from pathlib import Path

import numpy as np

from mjlab_b200.compiler.compile import MODEL_ARRAYS, MODEL_SCALARS_F, MODEL_SCALARS_I

LIB_PATH = Path(os.environ.get("B2SIM_LIB") or Path(__file__).resolve().parents[1] / "csrc" / "libb2sim.so")


class B2Array(ctypes.Structure):
  _fields_ = [
    ("name", ctypes.c_char_p), ("dtype", ctypes.c_int32), ("n", ctypes.c_int64),
    ("data", ctypes.c_void_p),
  ]


class B2ModelDesc(ctypes.Structure):
  _fields_ = [
    ("narray", ctypes.c_int32), ("arrays", ctypes.POINTER(B2Array)),
    ("gravity", ctypes.c_double * 3),
  ]


class B2Tensor(ctypes.Structure):
  _fields_ = [
    ("ptr", ctypes.c_void_p), ("dtype", ctypes.c_int32), ("ndim", ctypes.c_int32),
    ("shape", ctypes.c_int64 * 4), ("stride", ctypes.c_int64 * 4), ("device", ctypes.c_int32),
  ]


class B2Stats(ctypes.Structure):
  _fields_ = [
    ("ncon_max", ctypes.c_int32), ("ncon_cap", ctypes.c_int32), ("nefc_max", ctypes.c_int32),
    ("nefc_cap", ctypes.c_int32), ("overflow_worlds", ctypes.c_int32),
    ("niter_max", ctypes.c_int32), ("ncon_mean", ctypes.c_double),
    ("nefc_mean", ctypes.c_double), ("niter_mean", ctypes.c_double),
  ]


VELENV_NTERM = 14  # B2_VELENV_NTERM: reward terms with an episode sum
VELENV_NSTAGE = 8  # B2_VELENV_NSTAGE: stages of the command-velocity curriculum


VELENV_NRESET = 4  # B2_VELENV_NRESET: reset state terms
RESET_ROOT, RESET_JOINTS = 0, 1  # B2VelResetTerm.kind


class B2VelResetTerm(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_int32) for n in ("kind", "col", "count")] + [("joint", ctypes.c_int32 * 32)]
              + [("lo", ctypes.c_float * 12), ("span", ctypes.c_float * 12)])


class B2VelEnvArgs(ctypes.Structure):
  _fields_ = (
    [(n, ctypes.c_void_p) for n in (
      "action", "U", "default_qpos", "default_joint_pos", "action_scale", "soft_lo", "soft_hi",
      "env_origins", "episode_length", "last_action", "command", "push_time_left", "obs", "reward",
      "terminated", "truncated", "done", "cmd_time_left", "heading_target", "is_standing", "critic", "log_row")]
    + [(n, ctypes.c_float) for n in ("step_dt", "fall_angle", "push_vel", "push_lo", "push_hi")]
    + [("max_episode_length", ctypes.c_int32)]
    + [(n, ctypes.c_void_p) for n in ("terrain_origins", "terrain_levels", "terrain_types", "terrain_level_mean")]
    + [(n, ctypes.c_float) for n in ("move_up_dist", "episode_length_s")]
    + [(n, ctypes.c_int32) for n in ("rows", "cols", "curriculum")]
    + [("weight", ctypes.c_float * (VELENV_NTERM - 5))]
    + [(n, ctypes.c_float) for n in (
      "air_threshold_min", "air_threshold_max", "air_command_threshold", "air_command_scale_width",
      "clearance_target_height", "clearance_std", "clearance_tanh_mult")]
    + [(n, ctypes.c_int32) for n in ("air_continuous", "air_hard_scale", "n_air", "n_slide", "n_clear", "root_body")]
    + [(n, ctypes.c_void_p) for n in (
      "air_sensor_adr", "slide_sensor_adr", "slide_geom", "slide_body", "clear_geom", "clear_body", "air_time",
      "contact_time", "last_air_time", "episode_sums", "finished_sums")]
    + [(n, ctypes.c_float * 4) for n in ("cmd_mid", "cmd_half")]
    + [(n, ctypes.c_float) for n in ("ang_lo", "ang_hi", "heading_stiffness", "rel_standing", "resample_lo",
                                     "resample_span")]
    + [("n_stage", ctypes.c_int32)]
    + [("stage_step", ctypes.c_int32 * VELENV_NSTAGE)]
    + [(n, ctypes.c_float * VELENV_NSTAGE) for n in ("stage_mid", "stage_half", "stage_lo", "stage_hi")]
    + [(n, ctypes.c_void_p) for n in ("step_counter", "posture_inv_std2", "metric_xy", "metric_yaw",
                                      "finished_metrics")]
    + [("metric_steps", ctypes.c_float)]
    + [("push_off", ctypes.c_int32)]
    + [("ev_V", ctypes.c_void_p), ("ev_v_width", ctypes.c_int32), ("n_reset", ctypes.c_int32),
       ("reset_term", B2VelResetTerm * VELENV_NRESET)]
  )


class B2TrackEnvArgs(ctypes.Structure):
  _fields_ = (
    [(n, ctypes.c_void_p) for n in (
      "action", "U", "default_joint_pos", "soft_lo", "soft_hi", "env_origins", "m_joint_pos", "m_joint_vel",
      "m_body_pos", "m_body_quat", "m_body_lin", "m_body_ang", "body_idx", "ee_idx", "time_steps",
      "episode_length", "last_action", "push_time_left", "body_pos_rel", "body_quat_rel", "reward", "terminated",
      "truncated", "mask", "log_row", "obs", "critic")]
    + [("pose_range", ctypes.c_float * 12), ("vel_range", ctypes.c_float * 12)]
    + [(n, ctypes.c_float) for n in ("step_dt", "jp_lo", "jp_hi", "push_lo", "push_hi")]
    + [(n, ctypes.c_int32) for n in ("nb", "nee", "anchor", "T", "self_collision_adr", "root_body", "max_episode_length")]
    + [(n, ctypes.c_void_p) for n in ("adaptive_kernel", "cdf", "bin_fail_ema", "bin_fail_cur", "metrics")]
    + [(n, ctypes.c_float) for n in ("adaptive_alpha", "adaptive_uniform_ratio")]
    + [(n, ctypes.c_int32) for n in ("nbins", "adaptive", "adaptive_kernel_size")]
    + [("weight", ctypes.c_float * 9), ("std2", ctypes.c_float * 6),
       ("term_threshold", ctypes.c_float * 3), ("term_on", ctypes.c_int32 * 3), ("push_range", ctypes.c_float * 12)]
    + [(n, ctypes.c_int32) for n in ("push_on", "policy_state_estimation", "policy_corruption")]
    + [(n, ctypes.c_void_p) for n in ("episode_sums", "finished_sums", "term_flags", "motion_metrics",
                                      "finished_metrics")]
  )


TRACKENV_NREW, TRACKENV_NTERM, TRACKENV_NMETRIC = 9, 4, 10  # B2_TRACKENV_N*: log columns of B2TrackEnvArgs


OBSHIST_NTERM, OBSHIST_NGROUP = 16, 2  # B2_OBSHIST_NTERM / B2_OBSHIST_NGROUP: terms per group, groups per launch


class B2ObsHistTerm(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_int32) for n in ("src", "dim", "frames", "dst", "stride", "scale", "clip")]
              + [(n, ctypes.c_float) for n in ("lo", "hi")])


class B2ObsHistGroup(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_void_p) for n in ("frame", "out")]
              + [(n, ctypes.c_int32) for n in ("frame_width", "out_width", "nterm")]
              + [("term", B2ObsHistTerm * OBSHIST_NTERM)])


NOISE_NONE, NOISE_CONSTANT, NOISE_UNIFORM, NOISE_GAUSSIAN = 0, 1, 2, 3  # B2_NOISE_* classes (add / scale / abs: 0-2)


class B2ObsNoiseTerm(ctypes.Structure):
  _fields_ = [(n, ctypes.c_int32) for n in ("col", "noise", "noise_op", "noise_p0", "noise_p1", "noise_draw", "bias",
                                            "bias_op", "bias_p0", "bias_p1", "bias_draw", "bias_shared")]


class B2ObsNoiseGroup(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_void_p) for n in ("source", "bias")]
              + [(n, ctypes.c_int32) for n in ("source_width", "pad_")]
              + [("term", B2ObsNoiseTerm * OBSHIST_NTERM)])


class B2ObsHistArgs(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_void_p) for n in ("terminated", "truncated", "scale")]
              + [(n, ctypes.c_int32) for n in ("nscale", "ngroup")]
              + [("group", B2ObsHistGroup * OBSHIST_NGROUP)]
              + [(n, ctypes.c_void_p) for n in ("W", "N", "param")]
              + [(n, ctypes.c_int32) for n in ("nW", "nN", "nparam")]
              + [("noise", B2ObsNoiseGroup * OBSHIST_NGROUP)])


EVENTS_NTERM = 16  # B2_EVENTS_NTERM: reset and interval terms per b2_events launch
EVENT_RESET, EVENT_INTERVAL = 0, 1  # B2EventTerm.mode (B2_EVENT_* of include/b2sim.h); operation and distribution are
# the indices of events.OPERATIONS ("add", "scale", "abs") and events.DISTRIBUTIONS ("uniform", "log_uniform")


class B2EventTerm(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_int32) for n in ("mode", "operation", "distribution", "field", "count", "col")]
              + [(n, ctypes.c_float) for n in ("interval_lo", "interval_span")])


class B2EventElem(ctypes.Structure):
  _fields_ = [("offset", ctypes.c_int32), ("lo", ctypes.c_float), ("span", ctypes.c_float)]


EVENTS_NSTATE = 8  # B2_EVENTS_NSTATE: state terms per b2_events launch
EVENT_PUSH, EVENT_WRENCH = 0, 1  # B2EventStateTerm.kind


class B2EventStateTerm(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_int32) for n in ("kind", "mode", "col", "count", "first", "timer")]
              + [("lo", ctypes.c_float * 2), ("span", ctypes.c_float * 2), ("lo6", ctypes.c_float * 6),
                 ("span6", ctypes.c_float * 6), ("interval_lo", ctypes.c_float), ("interval_span", ctypes.c_float)])


class B2EventArgs(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_void_p) for n in ("terminated", "truncated", "V", "timers", "elem")]
              + [(n, ctypes.c_int32) for n in ("v_width", "ninterval", "nelem", "nterm")]
              + [("step_dt", ctypes.c_float), ("term", B2EventTerm * EVENTS_NTERM)]
              + [(n, ctypes.c_void_p) for n in ("refreshed", "bodies")]
              + [(n, ctypes.c_int32) for n in ("nstate", "nbodies", "clear_xfrc", "root_body")]
              + [("state", B2EventStateTerm * EVENTS_NSTATE)])


NAN_GUARD_ON = 1  # B2_NAN_GUARD_ON: b2_nan_guard's flag that arms the guard


class B2RenderArgs(ctypes.Structure):
  _fields_ = ([(n, ctypes.c_int32) for n in ("width", "height")] + [("lookat", ctypes.c_float * 3)]
              + [("track_body", ctypes.c_int32)] + [(n, ctypes.c_float) for n in ("distance", "azimuth", "elevation")]
              + [(n, ctypes.c_int32) for n in ("env_idx", "noverlay", "shadows", "brute")]
              + [(n, ctypes.c_void_p) for n in ("rgb", "depth", "seg", "decor")] + [("ndecor", ctypes.c_int32)]
              + [(n, ctypes.c_void_p) for n in ("ghost_xpos", "ghost_xmat")] + [("ghost_rgba", ctypes.c_float * 4)])


RENDER_MAXDECOR, RENDER_DECOR = 64, 12  # B2R_MAXDECOR arrows per frame of B2R_DECOR floats (csrc/b2_render.cuh)


START_UNIFORM, START_ADAPTIVE, START_FIRST = 0, 1, 2  # B2TrackEnvArgs.adaptive (B2_START_* of include/b2sim.h)


def make_model_desc(model):
  """Pack a compiled Model into a B2ModelDesc. Returns (desc, keepalive)."""
  keep = []
  names = [a.name for a in MODEL_ARRAYS] + MODEL_SCALARS_I + MODEL_SCALARS_F
  arrs = (B2Array * len(names))()
  for i, n in enumerate(names):
    a = np.asarray(model.arrays[n])
    if a.dtype.kind in "iu":
      a = np.ascontiguousarray(a, dtype=np.int32).reshape(-1)
      dt = 1
    else:
      a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
      dt = 0
    keep.append(a)
    nb = n.encode()
    keep.append(nb)
    arrs[i].name = nb
    arrs[i].dtype = dt
    arrs[i].n = a.size
    arrs[i].data = a.ctypes.data if a.size else None
  desc = B2ModelDesc()
  desc.narray = len(names)
  desc.arrays = arrs
  for k in range(3):
    desc.gravity[k] = float(model.opt_gravity[k])
  keep.append(arrs)
  return desc, keep


def bind(L: ctypes.CDLL) -> ctypes.CDLL:
  """Declare the signature of every entry point of include/b2sim.h on ``L`` (the CUDA library or its host emulation).

  Without ``argtypes`` ctypes passes a Python int as a C ``int``, which truncates a 64-bit pointer."""
  vp, ci, cd, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_char_p
  P = ctypes.POINTER
  signatures = {
    "b2_create": ([P(B2ModelDesc), ci, ci, ci, ci, P(vp)], ci),
    "b2_destroy": ([vp], ci),
    "b2_get_field": ([vp, ci, cs, P(B2Tensor)], ci),
    "b2_num_fields": ([vp, ci], ci),
    "b2_field_name": ([vp, ci, ci], cs),
    "b2_expand_model_field": ([vp, cs, vp, P(B2Tensor)], ci),
    "b2_set_option": ([vp, cs, cd], ci),
    "b2_get_option": ([vp, cs, P(cd)], ci),
    "b2_step": ([vp, vp], ci),
    "b2_forward": ([vp, vp], ci),
    "b2_step_n": ([vp, ci, vp], ci),
    "b2_forward_masked": ([vp, vp, vp], ci),
    "b2_step_host": ([vp, vp, ci, vp, vp, vp], ci),
    "b2_velenv_pre": ([vp, vp, vp, vp, vp], ci),
    "b2_velenv_post": ([vp, P(B2VelEnvArgs), vp], ci),
    "b2_trackenv_post1": ([vp, P(B2TrackEnvArgs), vp], ci),
    "b2_trackenv_post2": ([vp, P(B2TrackEnvArgs), vp], ci),
    "b2_trackenv_bins": ([vp, P(B2TrackEnvArgs), vp], ci),
    "b2_obs_history": ([vp, P(B2ObsHistArgs), vp], ci),
    "b2_events": ([vp, P(B2EventArgs), vp], ci),
    "b2_nan_guard": ([vp, ci, ci, ci], ci),
    "b2_nan_guard_word": ([vp], vp),
    "b2_nan_guard_read": ([vp, vp, P(ctypes.c_int64), vp, vp], ci),
    "b2_render": ([vp, P(B2RenderArgs), vp], ci),
    "b2_stats": ([vp, vp, P(B2Stats)], ci),
    "b2_launch_count": ([vp], ctypes.c_int64),
    "b2_algorithmic_bytes": ([vp, vp, P(cd), P(cd)], ci),
    "b2_last_error": ([], cs),
    "b2_version": ([], cs),
  }
  for name, (args, res) in signatures.items():
    fn = getattr(L, name)
    fn.argtypes, fn.restype = args, res
  return L


_lib = None


def load_library() -> ctypes.CDLL:
  """Load libb2sim.so; fails loudly when the CUDA extension has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not LIB_PATH.exists():
    raise RuntimeError(
      f"{LIB_PATH} not found: build the CUDA extension first "
      "(python -c 'import __graft_entry__ as g; g.build()'). There is no CPU fallback."
    )
  _lib = bind(ctypes.CDLL(str(LIB_PATH)))
  return _lib


def check(rc: int) -> None:
  if rc != 0:
    raise RuntimeError(f"b2sim: {load_library().b2_last_error().decode()}")


def ncon_per_world(nconmax: int | None, nworld: int) -> int:
  """Per-world contact capacity for upstream's global ``nconmax`` pool (SURVEY.md App. C); 0: the engine's default."""
  if nconmax is None:
    return 0
  return max(16, min(96, math.ceil(nconmax / max(nworld, 1))))


class Engine:
  """One ``b2_sim`` of a bound library (the CUDA library or its host emulation): created with the contact-capacity
  rule and destroyed once, with its field names, field descriptors and options.  Errors are read from the library
  that made the sim.  Subclasses wrap fields as tensors (device or host memory) and pick the stream."""

  def __init__(self, lib: ctypes.CDLL, model, nworld: int, nconmax: int | None = None, njmax: int | None = None,
               cuda_device: int = 0):
    self.lib = lib
    self.nworld = int(nworld)
    self.h = None
    desc, self._keep = make_model_desc(model)
    h = ctypes.c_void_p()
    self.check(lib.b2_create(ctypes.byref(desc), self.nworld, ncon_per_world(nconmax, self.nworld), int(njmax or 0),
                             cuda_device, ctypes.byref(h)))
    self.h = h

  def check(self, rc: int) -> None:
    if rc != 0:
      raise RuntimeError(f"b2sim: {self.lib.b2_last_error().decode()}")

  def names(self, which: int) -> list[str]:
    return [self.lib.b2_field_name(self.h, which, i).decode() for i in range(self.lib.b2_num_fields(self.h, which))]

  def get_field(self, which: int, name: str) -> B2Tensor:
    t = B2Tensor()
    self.check(self.lib.b2_get_field(self.h, which, name.encode(), ctypes.byref(t)))
    return t

  def set_option(self, key: str, value: float) -> None:
    self.check(self.lib.b2_set_option(self.h, key.encode(), float(value)))

  def get_option(self, key: str) -> float:
    v = ctypes.c_double()
    self.check(self.lib.b2_get_option(self.h, key.encode(), ctypes.byref(v)))
    return v.value

  def close(self) -> None:
    if self.h:
      self.lib.b2_destroy(self.h)
      self.h = None

  def __del__(self):
    # Tensors handed out keep their owner alive, so this only runs once no view of engine memory exists any more.
    try:
      self.close()
    except Exception:
      pass
