"""CSV recordings converted into the tracking task's motion files (mjlab_b200.envs.motion: read_csv, resample,
record_motion, convert_csv), on the host-emulated library (tests/emul): the resampling and the whole file against the
reference's own scripts/csv_to_npz.py where oracle/_ref is installed, chunking, the refusals, the round trip into the
tracking env, and the synthetic clip of tools/make_motion_clip.py unchanged.

The CSV fixtures are written here from tools/make_motion_clip.py's motion law: joints in a shuffled column order, one
row with its quaternion's sign flipped (slerp's negative-dot branch) and one row repeated (its ``|d| = 1`` branch)."""

import hashlib
import importlib.util
import sys
import types
import zipfile
from pathlib import Path

import numpy as np
import pytest
import torch

import refload
from mjlab_b200.sim import SimulationCfg, native
from test_kernel_emul import EmulSimulation

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tools"))

_ORDER = np.random.default_rng(12).permutation(29)
FLIP_ROW, REPEAT_ROW = 17, 30


def _g1():
  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.entity_data import EntityIndexing

  m = load_compiled("g1_tracking_flat")
  return m, EntityIndexing.from_model(m, "robot", "cpu")


def csv_joints():
  from mjlab_b200.envs.motion import G1_CSV_JOINTS

  return tuple(G1_CSV_JOINTS[i] for i in _ORDER)


def write_csv(path, fps=30.0, frames=60, joints=None, flip=FLIP_ROW, repeat=REPEAT_ROW):
  """make_motion_clip's motion sampled at ``fps``, as CSV rows (root position, quaternion xyzw, ``joints``)."""
  from make_motion_clip import motion_law

  from mjlab_b200.entity_data import EntityData

  m, ix = _g1()
  joints = csv_joints() if joints is None else joints
  lim = EntityData(ix, None, types.SimpleNamespace(jnt_range=torch.tensor(m.jnt_range)[None]), "cpu", 1,
                   soft_joint_pos_limit_factor=0.9).soft_joint_pos_limits[0]
  pos, quat, _, _, jp, _ = motion_law(m, ix, lim, frames, fps, "cpu")
  cols = [ix.joint_names.index(j) for j in joints]
  rows = torch.cat([pos, quat[:, [1, 2, 3, 0]], jp[:, cols]], dim=1).double().numpy()
  if flip is not None:
    rows[flip, 3:7] *= -1
  if repeat is not None:
    rows = np.insert(rows, repeat + 1, rows[repeat], axis=0)
  np.savetxt(path, rows, delimiter=",", fmt="%.9g")
  return Path(path)


@pytest.fixture(scope="module")
def emul():
  mp = pytest.MonkeyPatch()
  mp.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)
  yield
  mp.undo()


def convert(paths, out, chunk=4096, **kw):
  from mjlab_b200.envs.motion import convert_csv

  kw.setdefault("joint_names", csv_joints())
  return convert_csv(paths, out, device="cpu", chunk=chunk, simulation=EmulSimulation, **kw)


def _edit(a, f):
  a = a.copy()
  f(a)
  return a


def members(path):
  with zipfile.ZipFile(path) as z:
    return {n: z.read(n) for n in z.namelist()}


# ---- the reference's scripts/csv_to_npz.py ----------------------------------------------------------------------------
def _ref_script(monkeypatch):
  """scripts/csv_to_npz.py executed from oracle/_ref, its module-level imports of the task config, the viewer, tyro
  and tqdm stood in (none of them is used by MotionLoader or run_sim without rendering)."""
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  refload.load()

  class Bar:
    def __init__(self, *a, **k):
      pass

    update = set_description = close = lambda self, *a, **k: None

  stubs = {"tyro": {}, "tqdm": {"tqdm": Bar}, "mjlab.viewer": {},
           "mjlab.viewer.offscreen_renderer": {"OffscreenRenderer": type("OffscreenRenderer", (), {})},
           "mjlab.viewer.viewer_config": {"ViewerConfig": type("ViewerConfig", (), {})},
           "mjlab.tasks.tracking.config.g1.flat_env_cfg": {"G1FlatEnvCfg": type("G1FlatEnvCfg", (), {})}}
  for name, attrs in stubs.items():
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    monkeypatch.setitem(sys.modules, name, mod)
  name = "mjlab.scripts.csv_to_npz"
  spec = importlib.util.spec_from_file_location(name, refload.REF / "mjlab" / "scripts" / "csv_to_npz.py")
  mod = importlib.util.module_from_spec(spec)
  monkeypatch.setitem(sys.modules, name, mod)
  spec.loader.exec_module(mod)
  return mod


@pytest.mark.parametrize("fps_in,fps_out,line_range", [(30.0, 50.0, None), (30.0, 50.0, (5, 48)), (60.0, 50.0, None),
                                                        (60.0, 50.0, (3, 90)), (50.0, 50.0, None),
                                                        (50.0, 50.0, (10, 40))])
def test_resampling_matches_the_reference_motion_loader(fps_in, fps_out, line_range, tmp_path, monkeypatch):
  from mjlab_b200.envs.motion import frame_blend, read_csv, resample

  path = write_csv(tmp_path / "m.csv", fps=fps_in, frames=int(2 * fps_in))
  mod = _ref_script(monkeypatch)
  ref = mod.MotionLoader(str(path), fps_in, fps_out, "cpu", line_range=line_range)
  raw = read_csv(path, fps_in, line_range, csv_joints())
  ours = resample(*raw, fps_in, fps_out)
  T = ref.output_frames
  assert ours["root_pos"].shape[0] == T and T >= 30
  i0, i1, blend = frame_blend(raw[0].shape[0], fps_in, fps_out, "cpu")
  r0, r1, rb = ref._compute_frame_blend(torch.arange(0, ref.duration, ref.output_dt, dtype=torch.float32))
  assert torch.equal(i0, r0) and torch.equal(i1, r1) and torch.equal(blend, rb)
  # the fixture reaches slerp's negative-dot and |d| = 1 branches where its rows are in range
  if line_range is None or line_range[0] <= FLIP_ROW + 1 <= line_range[1]:
    assert (ours["root_quat"][:, 0] < 0).any()
  for k, r, tol in (("root_pos", ref.motion_base_poss, 2e-6), ("root_quat", ref.motion_base_rots, 2e-6),
                    ("joint_pos", ref.motion_dof_poss, 2e-6), ("root_lin_vel_w", ref.motion_base_lin_vels, 1e-4),
                    ("root_ang_vel_w", ref.motion_base_ang_vels, 1e-4), ("joint_vel", ref.motion_dof_vels, 1e-4)):
    assert ours[k].shape == r.shape, k
    assert (ours[k] - r).abs().max() <= tol, (k, float((ours[k] - r).abs().max()))


def test_whole_file_matches_the_reference_run_sim(emul, tmp_path, monkeypatch):
  """The reference's unmodified run_sim (one world, frame by frame) on its own Simulation and Entity over the
  emulated engine, against convert_csv's file: same keys, shapes and order; poses within 1e-5 and velocities within
  1e-4 (fp32 rounding of the interpolation, carried through the finite differences)."""
  import mjlab_b200.compat.mujoco_warp_shim as mw

  sys.path.insert(0, str(ROOT / "tests" / "emul"))
  from engine import EmulEngine

  path = write_csv(tmp_path / "clip.csv", frames=25, flip=9, repeat=15)  # 26 rows at 30 fps: 42 output frames at 50 fps
  mine = dict(np.load(convert([path], tmp_path)[0]))
  mod = _ref_script(monkeypatch)
  monkeypatch.setattr(mw, "_Engine", EmulEngine)
  import mujoco

  ref = refload.load()
  m, ix = _g1()
  sim = ref.sim.Simulation(1, ref.sim.SimulationCfg(nconmax=140, njmax=300), m, "cpu")
  E = ref.entity
  key = m.keys["robot/init_state"]
  ent = E.Entity.__new__(E.Entity)  # Entity.__init__ edits an MjSpec; the scene here is already compiled
  ent.cfg = E.EntityCfg(
    init_state=E.EntityCfg.InitialStateCfg(pos=tuple(key["qpos"][0:3]), rot=tuple(key["qpos"][3:7]),
                                           joint_pos={n: float(v) for n, v in zip(ix.joint_names, key["qpos"][7:])}),
    articulation=E.EntityArticulationInfoCfg(soft_joint_pos_limit_factor=0.9))
  ent._spec = mujoco.EntitySpecView(m, "robot/")
  ent._free_joint = ent._spec.joints[0]
  ent._non_free_joints = tuple(ent._spec.joints[1:])
  ent.initialize(sim.mj_model, sim.model, sim.data, "cpu")
  assert tuple(ent.body_names) == ix.body_names and tuple(ent.joint_names) == ix.joint_names

  class Scene:
    env_origins = torch.zeros(1, 3)

    def __getitem__(self, k):
      return ent

    def reset(self):
      ent.reset()

    def update(self, dt):
      ent.update(dt)

  saved = {}
  run = types.SimpleNamespace(log_artifact=lambda **k: None, link_artifact=lambda **k: None)
  wandb = types.ModuleType("wandb")
  wandb.init, wandb.finish = (lambda **k: run), (lambda: None)
  monkeypatch.setitem(sys.modules, "wandb", wandb)
  monkeypatch.setattr(np, "savez", lambda f, **arrays: saved.update(arrays))
  class Sim:  # the compiled model has no mjModel.opt; run_sim reads its timestep only for scene.update, which drops it
    mj_model = types.SimpleNamespace(opt=types.SimpleNamespace(timestep=0.02))

    def __getattr__(self, k):
      return getattr(sim, k)

  mod.run_sim(sim=Sim(), scene=Scene(), joint_names=list(csv_joints()), input_file=str(path), input_fps=30.0,
              output_fps=50.0, output_name="clip", render=False, line_range=None)
  monkeypatch.undo()
  assert list(saved) == list(mine)
  assert np.asarray(saved["fps"]).tolist() == mine["fps"].tolist() == [50.0]
  assert mine["joint_pos"].shape == (42, 29) and mine["body_pos_w"].shape == (42, len(ix.body_names), 3)
  for k in ("joint_pos", "joint_vel", "body_pos_w", "body_quat_w", "body_lin_vel_w", "body_ang_vel_w"):
    r = np.asarray(saved[k])
    assert r.shape == mine[k].shape and r.dtype == mine[k].dtype == np.float32, k
    tol = 1e-5 if k in ("joint_pos", "body_pos_w", "body_quat_w") else 1e-4
    assert np.abs(r - mine[k]).max() <= tol, (k, np.abs(r - mine[k]).max())


# ---- chunking, joints, the round trip ----------------------------------------------------------------------------
def test_chunk_sizes_and_batched_clips_give_identical_files(emul, tmp_path):
  a = write_csv(tmp_path / "a.csv", frames=20, flip=5, repeat=11)
  b = write_csv(tmp_path / "b.csv", frames=14, flip=None, repeat=3)
  files = {}
  for chunk in (1, 7, 4096):
    files[chunk] = members(convert([a], tmp_path / f"c{chunk}", chunk=chunk)[0])
  assert files[1] == files[7] == files[4096]
  both = convert([a, b], tmp_path / "both", chunk=7)
  alone = [convert([p], tmp_path / "alone", chunk=7)[0] for p in (a, b)]
  for x, y in zip(both, alone):
    assert members(x) == members(y)
  assert members(both[0]) == files[1]


def test_round_trip_into_the_tracking_env(emul, tmp_path, monkeypatch):
  """The file loads with MotionClip.load and drives the tracking env; joints the CSV lacks keep the keyframe."""
  from test_motion_clip import _emul_env

  from mjlab_b200.envs.motion import G1_CSV_JOINTS, MotionClip
  from mjlab_b200.envs.tracking_env import BODY_NAMES

  m, ix = _g1()
  joints = tuple(j for j in G1_CSV_JOINTS if j != "waist_roll_joint")
  out = convert([write_csv(tmp_path / "walk.csv", joints=joints)], tmp_path, joint_names=joints)[0]
  assert Path(out).name == "walk.npz"
  raw = np.load(out)
  j = ix.joint_names.index("waist_roll_joint")
  assert (raw["joint_pos"][:, j] == np.float32(m.keys["robot/init_state"]["qpos"][7 + j])).all()
  assert (raw["joint_vel"][:, j] == 0).all() and np.abs(raw["joint_vel"]).max() > 0.1
  clip = MotionClip.load(out, ix, BODY_NAMES, 0.02, "cpu")
  assert clip.num_frames == raw["joint_pos"].shape[0] > 90
  env = _emul_env(monkeypatch, num_envs=3, motion_file=out, native_mdp=True)
  assert env.T == clip.num_frames
  for _ in range(4):
    ob, rb, _, _, x = env.step(torch.zeros(3, env.nu))
    assert torch.isfinite(ob).all() and torch.isfinite(rb).all()
  env.close()


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_refusals(emul, tmp_path):
  from mjlab_b200.envs.motion import G1_CSV_JOINTS, read_csv, record_motion, resample

  good = write_csv(tmp_path / "good.csv", frames=30, joints=G1_CSV_JOINTS, flip=None, repeat=None)
  rows = np.loadtxt(good, delimiter=",")

  def bad(name, a):
    p = tmp_path / f"{name}.csv"
    np.savetxt(p, a, delimiter=",", fmt="%.9g")
    return p

  cases = [
    (bad("cols", rows[:, :-1]), {}, r"cols\.csv: 35 columns, expected 36"),
    (bad("nan", _edit(rows, lambda a: a.__setitem__((4, 9), np.nan))), {}, r"nan\.csv: line 5, column 10 is not finite"),
    (bad("quat", _edit(rows, lambda a: a.__setitem__((6, slice(3, 7)), a[6, 3:7] * 1.01))), {},
     r"quat\.csv: line 7: the root quaternion \(columns 4-7\) has norm 1\.01, more than 1e-3 from 1"),
    (good, dict(input_fps=0.0), r"good\.csv: input_fps is 0\.0, expected > 0"),
    (good, dict(input_fps=-30.0), r"input_fps is -30\.0, expected > 0"),
    (good, dict(line_range=(9, 4)), r"line_range \(9, 4\) is reversed or starts before line 1"),
    (good, dict(line_range=(0, 4)), r"line_range \(0, 4\) is reversed or starts before line 1"),
    (good, dict(line_range=(20, 40)), r"line_range \(20, 40\) is outside the file, which has 30 line\(s\)"),
    (good, dict(line_range=(40, 45)), r"line_range \(40, 45\) is outside the file"),
    (good, dict(line_range=(3, 3)), r"good\.csv: 1 frame\(s\), expected at least 2"),
    (bad("one", rows[:1]), {}, r"one\.csv: 1 frame\(s\), expected at least 2"),
  ]
  for path, kw, msg in cases:
    kw = dict(dict(input_fps=30.0, line_range=None), **kw)
    with pytest.raises(ValueError, match=msg):
      read_csv(path, kw["input_fps"], kw["line_range"], G1_CSV_JOINTS)
  # two input frames at 30 fps are 2 output frames at 50 fps: too few
  with pytest.raises(ValueError, match=r"2 input frames at 30 fps give 2 output frame\(s\) at 50 fps, expected at "
                                       r"least 3"):
    resample(*read_csv(good, 30.0, (1, 2), G1_CSV_JOINTS), 30.0, 50.0)
  with pytest.raises(ValueError, match=r"output_fps is 0\.0, expected > 0"):
    resample(*read_csv(good, 30.0, None, G1_CSV_JOINTS), 30.0, 0.0)
  with pytest.raises(ValueError, match=r"CSV joints \['tail_joint'\] are not joints of the G1"):
    convert([good], tmp_path, joint_names=G1_CSV_JOINTS[:-1] + ("tail_joint",))
  with pytest.raises(ValueError, match=r"chunk is 0, expected >= 1"):
    convert([good], tmp_path, chunk=0, joint_names=G1_CSV_JOINTS)
  (tmp_path / "d").mkdir()
  twin = tmp_path / "d" / "good.csv"
  twin.write_bytes(good.read_bytes())
  with pytest.raises(ValueError, match=r"share a stem"):
    convert([good, twin], tmp_path, joint_names=G1_CSV_JOINTS)
  # the consistency check: a root quaternion off the unit sphere (the engine normalises it) makes the angular velocity
  # read back differ from the motion's; refused, naming the first bad frame, and nothing is written
  from mjlab_b200.entity_data import EntityData, EntityIndexing

  m, _ = _g1()
  c = resample(*read_csv(good, 30.0, None, G1_CSV_JOINTS), 30.0, 50.0)
  T = c["joint_pos"].shape[0]
  c["root_ang_vel_w"][:, 0] += 0.5  # (a roll rate: the clip's yaw rate is parallel to its quaternions' axes)
  c["root_quat"][11:] *= 1.01
  sim = EmulSimulation(T, SimulationCfg(), m, "cpu")
  robot = EntityData(EntityIndexing.from_model(m, "robot", "cpu"), sim.data, sim.model, "cpu", T)
  with pytest.raises(ValueError, match=r"bad\.npz: frame 11: the root link's velocity after the forward differs"):
    record_motion(sim, robot, c["root_pos"], c["root_quat"], c["root_lin_vel_w"], c["root_ang_vel_w"],
                  c["joint_pos"], c["joint_vel"], 50.0, tmp_path / "bad.npz")
  sim.close()
  assert not (tmp_path / "bad.npz").exists()


# ---- tools/make_motion_clip.py -------------------------------------------------------------------------------------
# sha256 (first 16 hex digits) of every archive member, written by the script before it called record_motion
SYNTHETIC = {
  (96, 50.0): {"fps.npy": "35288fe19967bef1", "joint_pos.npy": "d719aae6a2474a0c", "joint_vel.npy": "7b40e48d67ac88bc",
               "body_pos_w.npy": "ec89dfb4d489524f", "body_quat_w.npy": "18c57fd9b20ce7b2",
               "body_lin_vel_w.npy": "191385e418503d3c", "body_ang_vel_w.npy": "265911b4ae7ea836"},
  (40, 30.0): {"fps.npy": "ecd984aec1667122", "joint_pos.npy": "7278d5782b657b75", "joint_vel.npy": "bff992d35fbf2417",
               "body_pos_w.npy": "7577b5fc95a5eb93", "body_quat_w.npy": "3cb0a85a6632824e",
               "body_lin_vel_w.npy": "d9467817f4eb81b5", "body_ang_vel_w.npy": "d3759108a164d8f9"},
}


@pytest.mark.parametrize("frames,fps", list(SYNTHETIC))
def test_synthetic_clip_is_unchanged(frames, fps, emul, tmp_path):
  from make_motion_clip import make_clip

  m, _ = _g1()
  sim = EmulSimulation(frames, SimulationCfg(), m, "cpu")
  path = make_clip(tmp_path / "clip.npz", frames=frames, fps=fps, device="cpu", sim=sim, model=m)
  sim.close()
  got = {n: hashlib.sha256(b).hexdigest()[:16] for n, b in members(path).items()}
  assert list(got.items()) == list(SYNTHETIC[(frames, fps)].items())
