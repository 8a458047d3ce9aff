"""Synthetic articulated robots for tools/emul_fuzz.py (host fuzzing) and tests/test_model_shapes_gpu.py (the product
build on the GPU): one generator, so that both build the same kind of model."""

import numpy as np


def robot_xml(rng, limbs, joints, *, dofs=58, joints_per_body=1, offsets=False, unlimited=False, actuate_all=False,
              box_links=False, feet=False):
  """Random articulated robot: a floating base with `limbs` chains of up to `joints` bodies (hinge / slide joints with
  random axes, limits, per-geom margin, gap, condim, friction, solref / solimp variations, position actuators with
  force ranges on a third of the bodies, Euler or implicitfast).  The chains hold at most `dofs` degrees of freedom
  between them (nv <= 6 + dofs).

  The keyword options widen the model; with all of them off the XML (and the draws taken from `rng`) are those of
  the original generator, seed for seed:
    joints_per_body  1-3 joints on each body (hinge and slide mixed): the kinematics take the generic walk
    offsets          joint anchors off the body origin and rotated bodies (`quat`)
    unlimited        hinges without limits (slides keep theirs)
    actuate_all      an actuator on every joint: position, motor or velocity, gear in [0.5, 2], ctrllimited
    box_links        box links instead of capsules (up to four contacts each against the floor)
    feet             a jointless (welded) foot body at the end of every chain"""
  axes = ["1 0 0", "0 1 0", "0 0 1"]
  body, acts = "", ""
  budget = dofs
  for li in range(limbs):
    n = int(rng.integers(max(1, joints - 3), joints + 1))
    ang = 2 * np.pi * li / limbs
    pos = f"{0.2 * np.cos(ang):.3f} {0.15 * np.sin(ang):.3f} -0.06"
    s, close = "", ""
    for k in range(n):
      if budget == 0:
        break
      # children are offset sideways: exactly coincident capsule axes give zero-length contact normals,
      # which no implementation defines
      p = pos if k == 0 else f"{rng.uniform(-0.03, 0.03):.3f} {rng.uniform(-0.03, 0.03):.3f} -0.12"
      ax = axes[int(rng.integers(0, 3))]
      slide = rng.uniform() < 0.15
      gopt = ""
      if rng.uniform() < 0.3:
        gopt += f' margin="{rng.uniform(0.0, 0.01):.4f}" gap="{rng.uniform(0.0, 0.004):.4f}"'
      if rng.uniform() < 0.3:
        gopt += ' condim="1"'
      if rng.uniform() < 0.3:
        gopt += f' friction="{rng.uniform(0.2, 1.5):.2f} 0.005 0.0001"'
      u = rng.uniform()
      if u < 0.25:
        gopt += f' solref="{rng.uniform(0.01, 0.05):.3f} {rng.uniform(0.7, 1.3):.2f}" solimp="0.8 0.97 0.002 0.4 {rng.uniform(1, 3):.1f}"'
      elif u < 0.35:
        gopt += ' solref="-2000 -50"'
      nj = min(budget, int(rng.integers(1, joints_per_body + 1))) if joints_per_body > 1 else 1
      budget -= nj
      bopt = ""
      if offsets:
        q = np.array([1.0, 0.0, 0.0, 0.0]) + rng.uniform(-0.3, 0.3, 4)
        bopt = f' quat="{" ".join(f"{x:.4f}" for x in q / np.linalg.norm(q))}"'
      joint_xml, names = "", []
      for j in range(nj):
        if j > 0:
          ax, slide = axes[int(rng.integers(0, 3))], rng.uniform() < 0.3
        name = f"j{li}_{k}" if j == 0 else f"j{li}_{k}_{j}"
        names.append(name)
        if slide:
          jt = 'type="slide" range="-0.05 0.05" limited="true"'
        else:
          jt = 'range="-1.2 1.2" limited="false"' if unlimited else 'range="-1.2 1.2" limited="true"'
        jpos = f' pos="{" ".join(f"{x:.3f}" for x in rng.uniform(-0.03, 0.03, 3))}"' if offsets else ""
        joint_xml += (f'<joint name="{name}"{jpos} axis="{ax}" {jt} '
                      f'damping="{rng.uniform(0.0, 0.5):.2f}" armature="0.01"/>')
      geom = ('<geom type="box" pos="0 0 -0.06" size="0.035 0.025 0.06"' if box_links else
              '<geom type="capsule" fromto="0 0 0 0 0 -0.12" size="0.03"')
      s += f'<body name="l{li}_{k}" pos="{p}"{bopt}>{joint_xml}{geom} mass="0.4"{gopt}/>'
      close += "</body>"
      if actuate_all:
        for name in names:
          kind = int(rng.integers(0, 3))
          g = f' gear="{rng.uniform(0.5, 2.0):.3f}" ctrllimited="true" ctrlrange="-{rng.uniform(0.3, 1.5):.2f} {rng.uniform(0.3, 1.5):.2f}"'
          if kind == 0:
            acts += f'<position joint="{name}" kp="{rng.uniform(5, 80):.1f}" kv="{rng.uniform(0.1, 3):.2f}"{g}/>'
          elif kind == 1:
            acts += f'<motor joint="{name}"{g}/>'
          else:
            acts += f'<velocity joint="{name}" kv="{rng.uniform(0.5, 5):.2f}"{g}/>'
      elif rng.uniform() < 0.33:
        fr = f' forcerange="-{rng.uniform(2, 20):.1f} {rng.uniform(2, 20):.1f}" forcelimited="true"' if rng.uniform() < 0.5 else ""
        acts += f'<position joint="j{li}_{k}" kp="{rng.uniform(5, 80):.1f}" kv="{rng.uniform(0.1, 3):.2f}"{fr}/>'
    if feet and s:
      s += f'<body name="f{li}" pos="0 0 -0.12"><geom type="sphere" size="0.035" mass="0.2"/></body>'
    body += s + close
  integ = ["implicitfast", "Euler"][int(rng.integers(0, 2))]
  return f"""<mujoco><compiler angle="radian"/><option timestep="0.004" integrator="{integ}"/>
  <worldbody><geom name="floor" type="plane" size="0 0 1"/>
  <body name="base" pos="0 0 0.55"><freejoint/><geom type="box" size="0.2 0.15 0.06" mass="4"/>{body}</body>
  </worldbody><actuator>{acts}</actuator></mujoco>"""
