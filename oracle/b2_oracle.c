/* b2_oracle.c — CPU ORACLE (test infrastructure, NOT the product).
 *
 * Plain-C restatement of the batched MuJoCo forward-dynamics step that mjlab reaches through
 * mjwarp.step / mjwarp.forward (reference call sites src/mjlab/sim/sim.py:136,139,187,195).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
 * load this library; the product path (mjlab_b200/csrc) never links or calls it.
 *
 * PARITY UNPINNED: the arithmetic of this path lives in third-party packages that are not
 * vendored in the reference and are absent from this image — mujoco-warp @486642c3
 * (pyproject.toml:94), mujoco==3.3.7.dev811775910 (uv.lock:1057-1058) — and the reference's own
 * tests hold no golden vectors for step() (SURVEY.md §4, §8c). Each function below therefore
 * restates the *published* MuJoCo algorithm (function names of MuJoCo's engine_*.c are cited)
 * and is pinned only by (a) the reference's qualitative tests (tests/test_entity.py:292-388),
 * (b) analytic cases and conservation invariants in tests/test_oracle.py.
 *
 * Serial, one world at a time, explicit dense constraint Jacobian — deliberately the textbook
 * formulation, structurally different from the matrix-free warp-parallel CUDA path it checks.
 * real = double (B2O_FLOAT -> float, used for the fp32 CPU baseline timing).
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "../include/b2sim.h"

#ifdef B2O_FLOAT
typedef float real;
#else
typedef double real;
#endif

#define MINVAL ((real)1e-15)
#define MINIMP ((real)0.0001)
#define MAXIMP ((real)0.9999)
#define MINMU ((real)1e-5)
enum { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };
enum { G_PLANE = 0, G_HFIELD = 1, G_SPHERE = 2, G_CAPSULE = 3, G_ELLIPSOID = 4, G_CYLINDER = 5, G_BOX = 6, G_MESH = 7 };
enum { OBJ_BODY = 1, OBJ_XBODY = 2, OBJ_GEOM = 5 };
enum { INT_EULER = 0, INT_IMPLICITFAST = 3 };
enum { EFC_LIMIT = 3, EFC_FRICTIONLESS = 4, EFC_PYRAMIDAL = 5 };

/* ---------------------------------------------------------------------------------------------
 * model / data containers
 * ------------------------------------------------------------------------------------------- */
#define MODEL_INT(X)                                                                            \
  X(body_parentid) X(body_rootid) X(body_weldid) X(body_jntadr) X(body_jntnum) X(body_dofadr)  \
  X(body_dofnum) X(jnt_type) X(jnt_qposadr) X(jnt_dofadr) X(jnt_bodyid) X(jnt_limited)          \
  X(dof_bodyid) X(dof_jntid) X(dof_parentid) X(geom_type) X(geom_bodyid) X(geom_condim)         \
  X(geom_priority) X(site_bodyid) X(actuator_trnid) X(actuator_ctrllimited)                     \
  X(actuator_forcelimited) X(pair_geom1) X(pair_geom2) X(sensor_type) X(sensor_objtype)         \
  X(sensor_objid) X(sensor_reftype) X(sensor_refid) X(sensor_intprm) X(sensor_adr) X(sensor_dim)          \
  X(geom_contype) X(geom_conaffinity) X(static_geom) X(static_cell0) X(dyn_cgeom) X(grid_start) X(grid_items) \
  X(geom_dataid) X(mesh_vertadr) X(mesh_vertnum) X(hfield_adr) X(hfield_nrow) X(hfield_ncol)

/* float model arrays: (name, row length per element group) — all expandable per world */
#define MODEL_REAL(X)                                                                           \
  X(body_pos) X(body_quat) X(body_ipos) X(body_iquat) X(body_mass) X(body_subtreemass)          \
  X(body_inertia) X(body_invweight0) X(jnt_pos) X(jnt_axis) X(jnt_range) X(jnt_solref)          \
  X(jnt_solimp) X(jnt_margin) X(jnt_stiffness) X(dof_armature) X(dof_damping)                   \
  X(dof_frictionloss) X(dof_invweight0) X(geom_size) X(geom_pos) X(geom_quat) X(geom_friction)  \
  X(geom_solref) X(geom_solimp) X(geom_solmix) X(geom_margin) X(geom_gap) X(geom_rbound)        \
  X(geom_rgba) X(site_pos) X(site_quat) X(actuator_gainprm) X(actuator_biasprm)                 \
  X(actuator_ctrlrange) X(actuator_forcerange) X(actuator_gear) X(qpos0)                        \
  X(mesh_vert) X(hfield_size) X(hfield_data)

/* scalars read from the model description: (member, model array, element) */
#define MODEL_SCALAR(X)                                                                         \
  X(nq, nq, 0) X(nv, nv, 0) X(nu, nu, 0) X(nbody, nbody, 0) X(njnt, njnt, 0) X(ngeom, ngeom, 0)  \
  X(nsite, nsite, 0) X(nsensor, nsensor, 0) X(nsensordata, nsensordata, 0) X(npair, npair, 0)    \
  X(integrator, opt_integrator, 0) X(cone, opt_cone, 0) X(solver, opt_solver, 0)                \
  X(iterations, opt_iterations, 0) X(ls_iterations, opt_ls_iterations, 0)                       \
  X(timestep, opt_timestep, 0) X(tolerance, opt_tolerance, 0) X(ls_tolerance, opt_ls_tolerance, 0) \
  X(impratio, opt_impratio, 0) X(meaninertia, stat_meaninertia, 0) X(nstatic, nstatic, 0)       \
  X(grid_x0, grid_params, 0) X(grid_y0, grid_params, 1) X(grid_cell, grid_params, 2)            \
  X(grid_nx, grid_params, 3) X(grid_ny, grid_params, 4)

/* options b2o_set_option accepts: (member, type); the option's name is the member's */
#define OPTIONS(X)                                                                              \
  X(iterations, int) X(ls_iterations, int) X(tolerance, real) X(ls_tolerance, real)            \
  X(timestep, real) X(integrator, int)

/* Data fields, [nworld][row length] each: (name, row length).  A field whose rows are empty still gets
 * one element per world. */
#define DATA_REAL(X)                                                                            \
  X(qpos, nq) X(qvel, nv) X(qacc, nv) X(qacc_warmstart, nv) X(ctrl, nu) X(qfrc_applied, nv)      \
  X(xfrc_applied, 6*nbody) X(xpos, 3*nbody) X(xquat, 4*nbody) X(xmat, 9*nbody)                 \
  X(xipos, 3*nbody) X(ximat, 9*nbody) X(subtree_com, 3*nbody) X(cinert, 10*nbody) X(cdof, 6*nv) \
  X(cdof_dot, 6*nv) X(cvel, 6*nbody) X(xanchor, 3*njnt) X(xaxis, 3*njnt) X(geom_xpos, 3*ngeom)  \
  X(geom_xmat, 9*ngeom) X(site_xpos, 3*nsite) X(site_xmat, 9*nsite) X(qM, nv*nv) X(qL, nv*nv)   \
  X(qfrc_bias, nv) X(qfrc_passive, nv) X(qfrc_actuator, nv) X(actuator_force, nu)              \
  X(qfrc_smooth, nv) X(qacc_smooth, nv) X(qfrc_constraint, nv) X(sensordata, nsensordata)      \
  X(time, 1) X(contact_dist, maxcon) X(contact_pos, 3*maxcon) X(contact_frame, 9*maxcon)       \
  X(contact_friction, 5*maxcon) X(contact_solref, 2*maxcon) X(contact_solimp, 5*maxcon)        \
  X(contact_includemargin, maxcon) X(contact_force, 3*maxcon) X(efc_J, njmax*nv)               \
  X(efc_pos, njmax) X(efc_margin, njmax) X(efc_D, njmax) X(efc_R, njmax) X(efc_aref, njmax)    \
  X(efc_vel, njmax) X(efc_force, njmax) X(solver_cost, 1)
#define DATA_INT(X)                                                                             \
  X(ncon, 1) X(nefc, 1) X(contact_dim, maxcon) X(contact_geom, 2*maxcon) X(contact_efc, maxcon) \
  X(efc_type, njmax) X(efc_id, njmax) X(solver_niter, 1) X(overflow, 1)

typedef struct { real* p; int n; int stride; } MF; /* stride 0 = shared by all worlds */

typedef struct B2Oracle {
  int nq, nv, nu, nbody, njnt, ngeom, nsite, nsensor, nsensordata, npair;
  int nworld, maxcon, njmax;
  int nstatic, ndyn, grid_nx, grid_ny; real grid_x0, grid_y0, grid_cell;
  int integrator, cone, solver, iterations, ls_iterations;
  real timestep, tolerance, ls_tolerance, impratio, meaninertia, gravity[3];
#define X(n) int* n;
  MODEL_INT(X)
#undef X
#define X(n) MF n;
  MODEL_REAL(X)
#undef X
  struct {
#define R(n, len) struct { real* p; int rowlen; } n;
#define I(n, len) struct { int* p; int rowlen; } n;
    DATA_REAL(R) DATA_INT(I)
#undef R
#undef I
  } data;
} B2Oracle;

static const B2Array* find_arr(const B2ModelDesc* d, const char* name) {
  for (int i = 0; i < d->narray; i++)
    if (!strcmp(d->arrays[i].name, name)) return &d->arrays[i];
  fprintf(stderr, "b2_oracle: model array '%s' missing\n", name);
  abort();
}
static double get_scalar(const B2ModelDesc* d, const char* name, int k) {
  const B2Array* a = find_arr(d, name);
  if (k >= a->n) { fprintf(stderr, "b2_oracle: model array '%s' has no element %d\n", name, k); abort(); }
  return a->dtype == B2_I32 ? ((const int32_t*)a->data)[k] : ((const double*)a->data)[k];
}
static int* dup_i(const B2ModelDesc* d, const char* name) {
  const B2Array* a = find_arr(d, name);
  int* p = (int*)malloc(sizeof(int) * (a->n ? a->n : 1));
  for (int64_t i = 0; i < a->n; i++) p[i] = ((const int32_t*)a->data)[i];
  return p;
}
static MF dup_f(const B2ModelDesc* d, const char* name) {
  const B2Array* a = find_arr(d, name);
  MF m;
  m.n = (int)a->n; m.stride = 0;
  m.p = (real*)malloc(sizeof(real) * (a->n ? a->n : 1));
  for (int64_t i = 0; i < a->n; i++) m.p[i] = (real)((const double*)a->data)[i];
  return m;
}
#define M_(o, name, w) ((o)->name.p + (size_t)(w) * (o)->name.stride)

/* ---------------------------------------------------------------------------------------------
 * small math (MuJoCo engine_util_blas.c / engine_util_spatial.c conventions)
 * ------------------------------------------------------------------------------------------- */
static real dot3(const real* a, const real* b) { return a[0]*b[0] + a[1]*b[1] + a[2]*b[2]; }
static void cross3(real* r, const real* a, const real* b) {
  real x = a[1]*b[2] - a[2]*b[1], y = a[2]*b[0] - a[0]*b[2], z = a[0]*b[1] - a[1]*b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
static real norm3(const real* a) { return sqrt(dot3(a, a)); }
static real normalize3(real* a) {
  real n = norm3(a);
  if (n < MINVAL) { a[0] = 1; a[1] = 0; a[2] = 0; return n; }
  a[0] /= n; a[1] /= n; a[2] /= n;
  return n;
}
static void normalize4(real* q) {
  real n = sqrt(q[0]*q[0] + q[1]*q[1] + q[2]*q[2] + q[3]*q[3]);
  if (n < MINVAL) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
static void mulquat(real* r, const real* a, const real* b) {
  real w = a[0]*b[0] - a[1]*b[1] - a[2]*b[2] - a[3]*b[3];
  real x = a[0]*b[1] + a[1]*b[0] + a[2]*b[3] - a[3]*b[2];
  real y = a[0]*b[2] - a[1]*b[3] + a[2]*b[0] + a[3]*b[1];
  real z = a[0]*b[3] + a[1]*b[2] - a[2]*b[1] + a[3]*b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
static void quat2mat(real* m, const real* q) {
  real q00 = q[0]*q[0], q11 = q[1]*q[1], q22 = q[2]*q[2], q33 = q[3]*q[3];
  real q01 = q[0]*q[1], q02 = q[0]*q[2], q03 = q[0]*q[3];
  real q12 = q[1]*q[2], q13 = q[1]*q[3], q23 = q[2]*q[3];
  m[0] = q00 + q11 - q22 - q33; m[4] = q00 - q11 + q22 - q33; m[8] = q00 - q11 - q22 + q33;
  m[1] = 2*(q12 - q03); m[2] = 2*(q13 + q02);
  m[3] = 2*(q12 + q03); m[5] = 2*(q23 - q01);
  m[6] = 2*(q13 - q02); m[7] = 2*(q23 + q01);
}
static void mulmatvec3(real* r, const real* m, const real* v) {
  real x = m[0]*v[0] + m[1]*v[1] + m[2]*v[2];
  real y = m[3]*v[0] + m[4]*v[1] + m[5]*v[2];
  real z = m[6]*v[0] + m[7]*v[1] + m[8]*v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
static void axisangle2quat(real* q, const real* axis, real angle) {
  real s = sin(angle * (real)0.5);
  q[0] = cos(angle * (real)0.5); q[1] = axis[0]*s; q[2] = axis[1]*s; q[3] = axis[2]*s;
}
/* mju_inertCom: 10-number inertia about the reference point (offset dif from body com) */
static void inert_com(real* res, const real* inert, const real* mat, const real* dif, real mass) {
  real tmp[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      tmp[3*i+j] = mat[3*i]*inert[0]*mat[3*j] + mat[3*i+1]*inert[1]*mat[3*j+1] + mat[3*i+2]*inert[2]*mat[3*j+2];
  res[0] = tmp[0] + mass*(dif[1]*dif[1] + dif[2]*dif[2]);
  res[1] = tmp[4] + mass*(dif[0]*dif[0] + dif[2]*dif[2]);
  res[2] = tmp[8] + mass*(dif[0]*dif[0] + dif[1]*dif[1]);
  res[3] = tmp[1] - mass*dif[0]*dif[1];
  res[4] = tmp[2] - mass*dif[0]*dif[2];
  res[5] = tmp[5] - mass*dif[1]*dif[2];
  res[6] = mass*dif[0]; res[7] = mass*dif[1]; res[8] = mass*dif[2];
  res[9] = mass;
}
/* mju_mulInertVec */
static void mul_inert_vec(real* r, const real* i, const real* v) {
  r[0] = i[0]*v[0] + i[3]*v[1] + i[4]*v[2] - i[8]*v[4] + i[7]*v[5];
  r[1] = i[3]*v[0] + i[1]*v[1] + i[5]*v[2] + i[8]*v[3] - i[6]*v[5];
  r[2] = i[4]*v[0] + i[5]*v[1] + i[2]*v[2] - i[7]*v[3] + i[6]*v[4];
  r[3] = i[8]*v[1] - i[7]*v[2] + i[9]*v[3];
  r[4] = i[6]*v[2] - i[8]*v[0] + i[9]*v[4];
  r[5] = i[7]*v[0] - i[6]*v[1] + i[9]*v[5];
}
/* mju_crossMotion / mju_crossForce */
static void cross_motion(real* r, const real* vel, const real* v) {
  r[0] = -vel[2]*v[1] + vel[1]*v[2];
  r[1] =  vel[2]*v[0] - vel[0]*v[2];
  r[2] = -vel[1]*v[0] + vel[0]*v[1];
  r[3] = -vel[2]*v[4] + vel[1]*v[5] - vel[5]*v[1] + vel[4]*v[2];
  r[4] =  vel[2]*v[3] - vel[0]*v[5] + vel[5]*v[0] - vel[3]*v[2];
  r[5] = -vel[1]*v[3] + vel[0]*v[4] - vel[4]*v[0] + vel[3]*v[1];
}
static void cross_force(real* r, const real* vel, const real* f) {
  r[0] = -vel[2]*f[1] + vel[1]*f[2] - vel[5]*f[4] + vel[4]*f[5];
  r[1] =  vel[2]*f[0] - vel[0]*f[2] + vel[5]*f[3] - vel[3]*f[5];
  r[2] = -vel[1]*f[0] + vel[0]*f[1] - vel[4]*f[3] + vel[3]*f[4];
  r[3] = -vel[2]*f[4] + vel[1]*f[5];
  r[4] =  vel[2]*f[3] - vel[0]*f[5];
  r[5] = -vel[1]*f[3] + vel[0]*f[4];
}
static real dot6(const real* a, const real* b) {
  return a[0]*b[0] + a[1]*b[1] + a[2]*b[2] + a[3]*b[3] + a[4]*b[4] + a[5]*b[5];
}
/* dense Cholesky, lower factor stored in-place (row-major n x n); returns rank */
static int chol_factor(real* A, int n) {
  int rank = n;
  for (int j = 0; j < n; j++) {
    real t = A[j*n+j];
    for (int k = 0; k < j; k++) t -= A[j*n+k]*A[j*n+k];
    if (t < MINVAL) { t = MINVAL; rank--; }
    t = sqrt(t);
    A[j*n+j] = t;
    for (int i = j+1; i < n; i++) {
      real s = A[i*n+j];
      for (int k = 0; k < j; k++) s -= A[i*n+k]*A[j*n+k];
      A[i*n+j] = s / t;
    }
  }
  return rank;
}
static void chol_solve(const real* L, int n, real* x) { /* x <- (L L')^-1 x */
  for (int i = 0; i < n; i++) {
    real s = x[i];
    for (int k = 0; k < i; k++) s -= L[i*n+k]*x[k];
    x[i] = s / L[i*n+i];
  }
  for (int i = n-1; i >= 0; i--) {
    real s = x[i];
    for (int k = i+1; k < n; k++) s -= L[k*n+i]*x[k];
    x[i] = s / L[i*n+i];
  }
}

/* ---------------------------------------------------------------------------------------------
 * per-world view
 * ------------------------------------------------------------------------------------------- */
typedef struct W {
  const B2Oracle* o; int w;
#define R(n, len) real* n;
#define I(n, len) int* n;
  DATA_REAL(R) DATA_INT(I)
#undef R
#undef I
} W;

static W bind(const B2Oracle* o, int w) {
  W d; d.o = o; d.w = w;
#define X(n, len) d.n = o->data.n.p + (size_t)w * o->data.n.rowlen;
  DATA_REAL(X) DATA_INT(X)
#undef X
  return d;
}

/* ---------------------------------------------------------------------------------------------
 * position stage: mj_kinematics, mj_comPos, mj_crb, mj_factorM (engine_core_smooth.c)
 * ------------------------------------------------------------------------------------------- */
static void kinematics(W* d) {
  const B2Oracle* o = d->o; int w = d->w;
  real* xpos = d->xpos; real* xquat = d->xquat; real* xmat = d->xmat;
  xpos[0] = xpos[1] = xpos[2] = 0; xquat[0] = 1; xquat[1] = xquat[2] = xquat[3] = 0;
  quat2mat(xmat, xquat);
  const real* qpos0 = M_(o, qpos0, w);
  for (int i = 1; i < o->nbody; i++) {
    int jn = o->body_jntnum[i], ja = o->body_jntadr[i], pid = o->body_parentid[i];
    real pos[3], quat[4];
    if (jn == 1 && o->jnt_type[ja] == JNT_FREE) {
      int a = o->jnt_qposadr[ja];
      for (int k = 0; k < 3; k++) pos[k] = d->qpos[a+k];
      for (int k = 0; k < 4; k++) quat[k] = d->qpos[a+3+k];
      normalize4(quat);
      for (int k = 0; k < 3; k++) d->xanchor[3*ja+k] = pos[k];
      real m[9]; quat2mat(m, quat);
      mulmatvec3(d->xaxis + 3*ja, m, M_(o, jnt_axis, w) + 3*ja);
    } else {
      const real* bp = M_(o, body_pos, w) + 3*i; const real* bq = M_(o, body_quat, w) + 4*i;
      mulmatvec3(pos, xmat + 9*pid, bp);
      for (int k = 0; k < 3; k++) pos[k] += xpos[3*pid+k];
      mulquat(quat, xquat + 4*pid, bq);
      for (int j = ja; j < ja + jn; j++) {
        real m[9]; quat2mat(m, quat);
        real* anchor = d->xanchor + 3*j; real* axis = d->xaxis + 3*j;
        mulmatvec3(anchor, m, M_(o, jnt_pos, w) + 3*j);
        for (int k = 0; k < 3; k++) anchor[k] += pos[k];
        mulmatvec3(axis, m, M_(o, jnt_axis, w) + 3*j);
        int qa = o->jnt_qposadr[j];
        real dq = d->qpos[qa] - qpos0[qa];
        if (o->jnt_type[j] == JNT_SLIDE) {
          for (int k = 0; k < 3; k++) pos[k] += axis[k]*dq;
        } else { /* hinge */
          real ql[4], qn[4], v[3];
          axisangle2quat(ql, M_(o, jnt_axis, w) + 3*j, dq);
          mulquat(qn, quat, ql);
          for (int k = 0; k < 4; k++) quat[k] = qn[k];
          quat2mat(m, quat);
          mulmatvec3(v, m, M_(o, jnt_pos, w) + 3*j);
          for (int k = 0; k < 3; k++) pos[k] = anchor[k] - v[k]; /* off-centre rotation */
        }
      }
    }
    normalize4(quat);
    for (int k = 0; k < 3; k++) xpos[3*i+k] = pos[k];
    for (int k = 0; k < 4; k++) xquat[4*i+k] = quat[k];
    quat2mat(xmat + 9*i, quat);
  }
  for (int i = 0; i < o->nbody; i++) {
    real q[4];
    mulmatvec3(d->xipos + 3*i, xmat + 9*i, M_(o, body_ipos, w) + 3*i);
    for (int k = 0; k < 3; k++) d->xipos[3*i+k] += xpos[3*i+k];
    mulquat(q, xquat + 4*i, M_(o, body_iquat, w) + 4*i);
    quat2mat(d->ximat + 9*i, q);
  }
  for (int g = 0; g < o->ngeom; g++) {
    int b = o->geom_bodyid[g]; real q[4];
    mulmatvec3(d->geom_xpos + 3*g, xmat + 9*b, M_(o, geom_pos, w) + 3*g);
    for (int k = 0; k < 3; k++) d->geom_xpos[3*g+k] += xpos[3*b+k];
    mulquat(q, xquat + 4*b, M_(o, geom_quat, w) + 4*g);
    quat2mat(d->geom_xmat + 9*g, q);
  }
  for (int s = 0; s < o->nsite; s++) {
    int b = o->site_bodyid[s]; real q[4];
    mulmatvec3(d->site_xpos + 3*s, xmat + 9*b, M_(o, site_pos, w) + 3*s);
    for (int k = 0; k < 3; k++) d->site_xpos[3*s+k] += xpos[3*b+k];
    mulquat(q, xquat + 4*b, M_(o, site_quat, w) + 4*s);
    quat2mat(d->site_xmat + 9*s, q);
  }
}

static void com_pos(W* d) {
  const B2Oracle* o = d->o; int w = d->w; int nb = o->nbody;
  const real* mass = M_(o, body_mass, w); const real* sub = M_(o, body_subtreemass, w);
  for (int i = 0; i < nb; i++)
    for (int k = 0; k < 3; k++) d->subtree_com[3*i+k] = mass[i]*d->xipos[3*i+k];
  for (int i = nb-1; i > 0; i--)
    for (int k = 0; k < 3; k++) d->subtree_com[3*o->body_parentid[i]+k] += d->subtree_com[3*i+k];
  for (int i = 0; i < nb; i++) {
    if (sub[i] < MINVAL) for (int k = 0; k < 3; k++) d->subtree_com[3*i+k] = d->xipos[3*i+k];
    else for (int k = 0; k < 3; k++) d->subtree_com[3*i+k] /= sub[i];
  }
  memset(d->cinert, 0, sizeof(real)*10);
  for (int i = 1; i < nb; i++) {
    real off[3];
    for (int k = 0; k < 3; k++) off[k] = d->xipos[3*i+k] - d->subtree_com[3*o->body_rootid[i]+k];
    inert_com(d->cinert + 10*i, M_(o, body_inertia, w) + 3*i, d->ximat + 9*i, off, mass[i]);
  }
  for (int j = 0; j < o->njnt; j++) {
    int b = o->jnt_bodyid[j], da = o->jnt_dofadr[j];
    real off[3];
    for (int k = 0; k < 3; k++) off[k] = d->subtree_com[3*o->body_rootid[b]+k] - d->xanchor[3*j+k];
    if (o->jnt_type[j] == JNT_FREE) {
      memset(d->cdof + 6*da, 0, sizeof(real)*18);
      for (int k = 0; k < 3; k++) d->cdof[6*(da+k)+3+k] = 1;
      for (int k = 0; k < 3; k++) { /* rotations about body-frame axes */
        real ax[3] = { d->xmat[9*b+k], d->xmat[9*b+3+k], d->xmat[9*b+6+k] };
        real* c = d->cdof + 6*(da+3+k);
        c[0] = ax[0]; c[1] = ax[1]; c[2] = ax[2];
        cross3(c+3, ax, off);
      }
    } else if (o->jnt_type[j] == JNT_SLIDE) {
      real* c = d->cdof + 6*da;
      c[0] = c[1] = c[2] = 0;
      for (int k = 0; k < 3; k++) c[3+k] = d->xaxis[3*j+k];
    } else {
      real* c = d->cdof + 6*da;
      for (int k = 0; k < 3; k++) c[k] = d->xaxis[3*j+k];
      cross3(c+3, d->xaxis + 3*j, off);
    }
  }
}

static void crb_and_factor(W* d, real* crb /* nb*10 scratch */) {
  const B2Oracle* o = d->o; int w = d->w; int nb = o->nbody, nv = o->nv;
  memcpy(crb, d->cinert, sizeof(real)*10*nb);
  for (int i = nb-1; i > 0; i--) {
    int p = o->body_parentid[i];
    if (p > 0) for (int k = 0; k < 10; k++) crb[10*p+k] += crb[10*i+k];
  }
  memset(d->qM, 0, sizeof(real)*nv*nv);
  const real* arm = M_(o, dof_armature, w);
  for (int i = 0; i < nv; i++) {
    real buf[6];
    mul_inert_vec(buf, crb + 10*o->dof_bodyid[i], d->cdof + 6*i);
    for (int j = i; j >= 0; j = o->dof_parentid[j]) {
      real v = dot6(d->cdof + 6*j, buf);
      d->qM[i*nv+j] = v; d->qM[j*nv+i] = v;
    }
    d->qM[i*nv+i] += arm[i];
  }
  memcpy(d->qL, d->qM, sizeof(real)*nv*nv);
  chol_factor(d->qL, nv);
}

/* mj_jac: 3 x nv translational / rotational Jacobians of a point fixed to `body` */
static void jac_point(const W* d, real* jacp, real* jacr, const real* point, int body) {
  const B2Oracle* o = d->o; int nv = o->nv;
  if (jacp) memset(jacp, 0, sizeof(real)*3*nv);
  if (jacr) memset(jacr, 0, sizeof(real)*3*nv);
  while (body && o->body_dofnum[body] == 0) body = o->body_parentid[body];
  if (!body) return;
  real off[3];
  const real* com = d->subtree_com + 3*o->body_rootid[body];
  for (int k = 0; k < 3; k++) off[k] = point[k] - com[k];
  int i = o->body_dofadr[body] + o->body_dofnum[body] - 1;
  for (; i >= 0; i = o->dof_parentid[i]) {
    const real* c = d->cdof + 6*i;
    if (jacr) for (int k = 0; k < 3; k++) jacr[k*nv+i] = c[k];
    if (jacp) {
      real t[3]; cross3(t, c, off);
      for (int k = 0; k < 3; k++) jacp[k*nv+i] = c[3+k] + t[k];
    }
  }
}

/* ---------------------------------------------------------------------------------------------
 * collision: static pair table + bounding-sphere filter + primitive narrowphase
 * (engine_collision_driver.c mj_collision; engine_collision_primitive.c)
 * ------------------------------------------------------------------------------------------- */
typedef struct { real dist, pos[3], frame[9]; } RawCon;

/* mesh / height-field narrowphase: the product's single-source routines (mjlab_b200/csrc/b2_convex.h) compiled
 * in this file's precision; pinned independently in tests/test_convex.py (see that header's note) */
#define B2C_REAL real
#define B2C_FN static
#define B2C_INL static inline
#define B2C_SQRT sqrt
#include "../mjlab_b200/csrc/b2_convex.h"
static int from_b2c(RawCon* rc, const B2CCon* c, int n) {
  for (int i = 0; i < n; i++) {
    rc[i].dist = c[i].dist;
    for (int k = 0; k < 3; k++) { rc[i].pos[k] = c[i].pos[k]; rc[i].frame[k] = c[i].n[k]; rc[i].frame[3+k] = 0; }
  }
  return n;
}

static int sphere_sphere(RawCon* c, real margin, const real* p1, real r1, const real* p2, real r2) {
  real dif[3] = { p2[0]-p1[0], p2[1]-p1[1], p2[2]-p1[2] };
  real cd = norm3(dif);
  if (cd > margin + r1 + r2) return 0;
  c->dist = cd - r1 - r2;
  normalize3(dif);
  for (int k = 0; k < 3; k++) { c->frame[k] = dif[k]; c->pos[k] = p1[k] + dif[k]*(r1 + (real)0.5*c->dist); }
  for (int k = 3; k < 9; k++) c->frame[k] = 0;
  return 1;
}
static int plane_sphere(RawCon* c, real margin, const real* pp, const real* pm, const real* sp, real r) {
  real n[3] = { pm[2], pm[5], pm[8] };
  real dif[3] = { sp[0]-pp[0], sp[1]-pp[1], sp[2]-pp[2] };
  real cd = dot3(dif, n);
  if (cd > margin + r) return 0;
  c->dist = cd - r;
  for (int k = 0; k < 3; k++) { c->frame[k] = n[k]; c->pos[k] = sp[k] - n[k]*(r + (real)0.5*c->dist); }
  for (int k = 3; k < 9; k++) c->frame[k] = 0;
  return 1;
}
static int plane_capsule(RawCon* c, real margin, const real* pp, const real* pm, const real* cp,
                         const real* cm, const real* size) {
  real axis[3] = { cm[2], cm[5], cm[8] }, s[3];
  int n = 0;
  for (int k = 0; k < 3; k++) s[k] = cp[k] + axis[k]*size[1];
  int n1 = plane_sphere(c + n, margin, pp, pm, s, size[0]);
  if (n1) { for (int k = 0; k < 3; k++) c[n].frame[3+k] = axis[k]; n++; }
  for (int k = 0; k < 3; k++) s[k] = cp[k] - axis[k]*size[1];
  int n2 = plane_sphere(c + n, margin, pp, pm, s, size[0]);
  if (n2) { for (int k = 0; k < 3; k++) c[n].frame[3+k] = axis[k]; n++; }
  return n;
}
static int plane_box(RawCon* c, real margin, const real* pp, const real* pm, const real* bp,
                     const real* bm, const real* size) {
  real n[3] = { pm[2], pm[5], pm[8] };
  real dif[3] = { bp[0]-pp[0], bp[1]-pp[1], bp[2]-pp[2] };
  real dist = dot3(dif, n);
  int cnt = 0;
  for (int i = 0; i < 8; i++) {
    real v[3] = { (i&1 ? size[0] : -size[0]), (i&2 ? size[1] : -size[1]), (i&4 ? size[2] : -size[2]) };
    real corner[3]; mulmatvec3(corner, bm, v);
    real ld = dot3(n, corner);
    if (dist + ld > margin || ld > 0) continue;
    c[cnt].dist = dist + ld;
    for (int k = 0; k < 3; k++) {
      c[cnt].pos[k] = bp[k] + corner[k] - n[k]*(c[cnt].dist*(real)0.5);
      c[cnt].frame[k] = n[k];
    }
    for (int k = 3; k < 9; k++) c[cnt].frame[k] = 0;
    if (++cnt >= 4) return 4;
  }
  return cnt;
}
static int sphere_capsule(RawCon* c, real margin, const real* sp, real sr, const real* cp,
                          const real* cm, const real* size) {
  real axis[3] = { cm[2], cm[5], cm[8] };
  real vec[3] = { sp[0]-cp[0], sp[1]-cp[1], sp[2]-cp[2] };
  real x = dot3(axis, vec);
  x = x > size[1] ? size[1] : (x < -size[1] ? -size[1] : x);
  real pt[3] = { cp[0] + axis[0]*x, cp[1] + axis[1]*x, cp[2] + axis[2]*x };
  return sphere_sphere(c, margin, sp, sr, pt, size[0]);
}
static int capsule_capsule(RawCon* c, real margin, const real* p1, const real* m1, const real* s1,
                           const real* p2, const real* m2, const real* s2) {
  real a1[3] = { m1[2], m1[5], m1[8] }, a2[3] = { m2[2], m2[5], m2[8] };
  real dif[3] = { p1[0]-p2[0], p1[1]-p2[1], p1[2]-p2[2] };
  real ma = dot3(a1, a1), mb = -dot3(a1, a2), mc = dot3(a2, a2);
  real u = -dot3(a1, dif), v = dot3(a2, dif);
  real det = ma*mc - mb*mb;
  real len1 = s1[1], len2 = s2[1];
  /* parallel test at fp64 resolution (mjMINVAL) or, in the fp32 build, at what fp32 can resolve (det ~ 1e-7 noise) */
  if (fabs(det) >= (sizeof(real) == 4 ? (real)1e-6 : MINVAL)) { /* general configuration */
    real x1 = (mc*u - mb*v)/det, x2 = (ma*v - mb*u)/det;
    if (x1 > len1) { x1 = len1; x2 = (v - mb*len1)/mc; }
    else if (x1 < -len1) { x1 = -len1; x2 = (v + mb*len1)/mc; }
    if (x2 > len2) { x2 = len2; x1 = (u - mb*len2)/ma; }
    else if (x2 < -len2) { x2 = -len2; x1 = (u + mb*len2)/ma; }
    if (x1 > len1) x1 = len1; else if (x1 < -len1) x1 = -len1;
    real v1[3], v2[3];
    for (int k = 0; k < 3; k++) { v1[k] = p1[k] + a1[k]*x1; v2[k] = p2[k] + a2[k]*x2; }
    return sphere_sphere(c, margin, v1, s1[0], v2, s2[0]);
  }
  /* parallel axes: test both ends of capsule 1 against segment 2, at most 2 contacts */
  int n = 0;
  for (int e = 0; e < 2 && n < 2; e++) {
    real x1 = e ? -len1 : len1, v1[3], v2[3], t[3];
    for (int k = 0; k < 3; k++) { v1[k] = p1[k] + a1[k]*x1; t[k] = v1[k] - p2[k]; }
    real x2 = dot3(a2, t);
    x2 = x2 > len2 ? len2 : (x2 < -len2 ? -len2 : x2);
    for (int k = 0; k < 3; k++) v2[k] = p2[k] + a2[k]*x2;
    n += sphere_sphere(c + n, margin, v1, s1[0], v2, s2[0]);
  }
  return n;
}
/* sphere - box (sphere is geom1): closest point of the box to the sphere centre; a centre inside the box
 * leaves through the nearest face.  Own restatement of the textbook test (MuJoCo's mjc_SphereBox follows the
 * same idea; its source is not available here). */
static int sphere_box(RawCon* c, real margin, const real* sp, real r, const real* bp, const real* bm,
                      const real* h) {
  real d[3] = { sp[0]-bp[0], sp[1]-bp[1], sp[2]-bp[2] }, l[3], cl[3], nl[3];
  for (int k = 0; k < 3; k++) l[k] = bm[k]*d[0] + bm[3+k]*d[1] + bm[6+k]*d[2];   /* R^T d */
  int inside = 1;
  for (int k = 0; k < 3; k++) {
    cl[k] = l[k] > h[k] ? h[k] : (l[k] < -h[k] ? -h[k] : l[k]);
    if (cl[k] != l[k]) inside = 0;
  }
  real dist;
  if (!inside) {
    real e[3] = { l[0]-cl[0], l[1]-cl[1], l[2]-cl[2] };
    real dc = norm3(e);
    if (dc > r + margin) return 0;
    dist = dc - r;
    for (int k = 0; k < 3; k++) nl[k] = -e[k]/dc;
  } else {
    int best = 0; real depth = h[0] - fabs(l[0]);
    for (int k = 1; k < 3; k++) { real t = h[k] - fabs(l[k]); if (t < depth) { depth = t; best = k; } }
    nl[0] = nl[1] = nl[2] = 0;
    nl[best] = l[best] >= 0 ? (real)-1 : (real)1;
    dist = -(depth + r);
  }
  real n[3];
  mulmatvec3(n, bm, nl);
  c->dist = dist;
  for (int k = 0; k < 3; k++) { c->frame[k] = n[k]; c->pos[k] = sp[k] + n[k]*(r + (real)0.5*dist); }
  for (int k = 3; k < 9; k++) c->frame[k] = 0;
  return 1;
}
static real point_box_dist2(const real* pt, const real* bp, const real* bm, const real* h) {
  real d[3] = { pt[0]-bp[0], pt[1]-bp[1], pt[2]-bp[2] }, s = 0;
  for (int k = 0; k < 3; k++) {
    real l = bm[k]*d[0] + bm[3+k]*d[1] + bm[6+k]*d[2];
    real e = l > h[k] ? l - h[k] : (l < -h[k] ? l + h[k] : 0);
    s += e*e;
  }
  return s;
}
/* capsule - box (capsule is geom1).  The distance d(t) from the axis point c + t*a to the box is convex in
 * t: golden-section search (24 steps) gives d_min; the contact set is the sub-segment [ta, tb] on which
 * d(t) <= d_min + 1e-3*radius (its ends found by 16 bisection steps each, well conditioned because d crosses
 * that level transversally).  A short sub-segment gives one sphere-box contact at its middle, a long one (the
 * capsule lies along a face or across an edge) gives one at each end - chosen this way, rather than "closest
 * point + an end cap", so that the result does not depend on which of many equidistant points a search lands
 * on.  Own definition (MuJoCo's mjc_CapsuleBox source is not available here). */
/* distance from the axis point l0 + t*al (box frame) to the box; working in the box frame keeps the
 * profile's shape free of the rounding of large world coordinates */
static real axis_box_dist(const real* l0, const real* al, real t, const real* h) {
  real s = 0;
  for (int k = 0; k < 3; k++) {
    real l = l0[k] + al[k]*t;
    real e = l > h[k] ? l - h[k] : (l < -h[k] ? l + h[k] : 0);
    s += e*e;
  }
  return sqrt(s);
}
static int capsule_box(RawCon* c, real margin, const real* cp, const real* cm, const real* cs,
                       const real* bp, const real* bm, const real* h) {
  real ax[3] = { cm[2], cm[5], cm[8] }, len = cs[1], r = cs[0];
  real d0[3] = { cp[0]-bp[0], cp[1]-bp[1], cp[2]-bp[2] }, l0[3], al[3];
  for (int k = 0; k < 3; k++) {
    l0[k] = bm[k]*d0[0] + bm[3+k]*d0[1] + bm[6+k]*d0[2];
    al[k] = bm[k]*ax[0] + bm[3+k]*ax[1] + bm[6+k]*ax[2];
  }
  real lo = -len, hi = len;
  const real gr = (real)0.6180339887498949;
  real x1 = hi - gr*(hi-lo), x2 = lo + gr*(hi-lo);
  real f1 = axis_box_dist(l0, al, x1, h), f2 = axis_box_dist(l0, al, x2, h);
  for (int it = 0; it < 24; it++) {
    if (f1 <= f2) { hi = x2; x2 = x1; f2 = f1; x1 = hi - gr*(hi-lo); f1 = axis_box_dist(l0, al, x1, h); }
    else { lo = x1; x1 = x2; f1 = f2; x2 = lo + gr*(hi-lo); f2 = axis_box_dist(l0, al, x2, h); }
  }
  real ts = (real)0.5*(lo+hi);
  real dmin = axis_box_dist(l0, al, ts, h);
  if (dmin > r + margin) return 0;
  real level = dmin + (real)1e-3*r;
  real ta = -len, tb = len;
  if (axis_box_dist(l0, al, -len, h) > level) {
    real a = -len, b = ts;
    for (int it = 0; it < 16; it++) { real mid = (real)0.5*(a+b); if (axis_box_dist(l0, al, mid, h) > level) a = mid; else b = mid; }
    ta = b;
  }
  if (axis_box_dist(l0, al, len, h) > level) {
    real a = ts, b = len;
    for (int it = 0; it < 16; it++) { real mid = (real)0.5*(a+b); if (axis_box_dist(l0, al, mid, h) > level) b = mid; else a = mid; }
    tb = a;
  }
  int n = 0; real p[3];
  if (tb - ta < (real)0.02*len) {
    real tm = (real)0.5*(ta+tb);
    for (int k = 0; k < 3; k++) p[k] = cp[k] + ax[k]*tm;
    n += sphere_box(c + n, margin, p, r, bp, bm, h);
  } else {
    for (int k = 0; k < 3; k++) p[k] = cp[k] + ax[k]*ta;
    n += sphere_box(c + n, margin, p, r, bp, bm, h);
    for (int k = 0; k < 3; k++) p[k] = cp[k] + ax[k]*tb;
    n += sphere_box(c + n, margin, p, r, bp, bm, h);
  }
  return n;
}
/* box - box: separating-axis test over the 15 candidate axes (3 + 3 face normals, 9 edge cross products), then
 *   face case  - the incident face of the other box (the one most anti-parallel to the reference normal) is clipped
 *                against the four side planes of the reference face (Sutherland-Hodgman); every clipped vertex
 *                within `margin` of the reference face is a contact (<= 8), position = midpoint between the surfaces;
 *   edge case  - one contact at the midpoint of the closest points of the two edges.
 * The axis of least penetration wins; a later axis replaces an earlier one only when it is better by more than
 * 1e-5 (relative), and an edge axis only when its depth is 5 % smaller than the best face axis (the usual bias
 * towards face contacts) - so ties (stacked, aligned boxes) resolve the same way in fp32 and fp64.
 * The normal points from box 1 to box 2.  (Own statement of the textbook algorithm: the source of MuJoCo's
 * mjc_BoxBox is not available in this image; contact counts and positions for face and edge cases are pinned by
 * statics in tests/test_boxes_terrain.py.) */
static int box_box(RawCon* c, real margin, const real* p1, const real* m1, const real* h1,
                   const real* p2, const real* m2, const real* h2) {
  real A[3][3], B[3][3], R[3][3], Q[3][3], t[3] = { p2[0]-p1[0], p2[1]-p1[1], p2[2]-p1[2] }, tA[3], tB[3];
  for (int i = 0; i < 3; i++) for (int k = 0; k < 3; k++) { A[i][k] = m1[3*k+i]; B[i][k] = m2[3*k+i]; }  /* axes = columns */
  for (int i = 0; i < 3; i++) {
    tA[i] = dot3(t, A[i]); tB[i] = dot3(t, B[i]);
    for (int j = 0; j < 3; j++) { R[i][j] = dot3(A[i], B[j]); Q[i][j] = fabs(R[i][j]) + (real)1e-6; }
  }
  int best = -1; real bdepth = 0;
  /* face axes of box 1 (codes 0-2) and box 2 (codes 3-5) */
  for (int i = 0; i < 3; i++) {
    real depth = h1[i] + h2[0]*Q[i][0] + h2[1]*Q[i][1] + h2[2]*Q[i][2] - fabs(tA[i]);
    if (depth < -margin) return 0;
    if (best < 0 || depth < bdepth - (real)1e-5*((real)1 + fabs(bdepth))) { best = i; bdepth = depth; }
  }
  for (int j = 0; j < 3; j++) {
    real depth = h2[j] + h1[0]*Q[0][j] + h1[1]*Q[1][j] + h1[2]*Q[2][j] - fabs(tB[j]);
    if (depth < -margin) return 0;
    if (depth < bdepth - (real)1e-5*((real)1 + fabs(bdepth))) { best = 3 + j; bdepth = depth; }
  }
  /* edge axes a_i x b_j (codes 6 + 3 i + j) */
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    real l2 = (real)1 - R[i][j]*R[i][j];
    if (l2 < (real)1e-6) continue;  /* (nearly) parallel edges: covered by the face axes */
    int i1 = (i+1)%3, i2 = (i+2)%3, j1 = (j+1)%3, j2 = (j+2)%3;
    real il = (real)1 / sqrt(l2);
    real depth = (h1[i1]*Q[i2][j] + h1[i2]*Q[i1][j] + h2[j1]*Q[i][j2] + h2[j2]*Q[i][j1]
                  - fabs(tA[i2]*R[i1][j] - tA[i1]*R[i2][j])) * il;
    if (depth < -margin) return 0;
    if (depth + (real)0.05*fabs(depth) + (real)1e-6 < bdepth) { best = 6 + 3*i + j; bdepth = depth; }
  }
  if (best >= 6) {
    int i = (best-6)/3, j = (best-6)%3;
    real L[3]; cross3(L, A[i], B[j]); normalize3(L);
    if (dot3(L, t) < 0) { L[0] = -L[0]; L[1] = -L[1]; L[2] = -L[2]; }
    real pa[3] = { p1[0], p1[1], p1[2] }, pb[3] = { p2[0], p2[1], p2[2] };
    for (int k = 0; k < 3; k++) {
      if (k != i) { real sg = dot3(A[k], L) >= 0 ? h1[k] : -h1[k]; for (int x = 0; x < 3; x++) pa[x] += sg*A[k][x]; }
      if (k != j) { real sg = dot3(B[k], L) >= 0 ? -h2[k] : h2[k]; for (int x = 0; x < 3; x++) pb[x] += sg*B[k][x]; }
    }
    /* closest points of the lines pa + s a_i and pb + u b_j, clamped to the edges */
    real d[3] = { pb[0]-pa[0], pb[1]-pa[1], pb[2]-pa[2] }, r = R[i][j], da = dot3(d, A[i]), db = dot3(d, B[j]);
    real den = (real)1 - r*r;
    real sA = (da - r*db) / den, sB = (r*da - db) / den;
    sA = sA > h1[i] ? h1[i] : (sA < -h1[i] ? -h1[i] : sA);
    sB = sB > h2[j] ? h2[j] : (sB < -h2[j] ? -h2[j] : sB);
    c[0].dist = -bdepth;
    for (int x = 0; x < 3; x++) {
      c[0].pos[x] = (real)0.5*(pa[x] + sA*A[i][x] + pb[x] + sB*B[j][x]);
      c[0].frame[x] = L[x];
    }
    for (int k = 3; k < 9; k++) c[0].frame[k] = 0;
    return 1;
  }
  /* face case: reference box `ref` (0: box 1, 1: box 2), reference axis `ax`, n = outward normal towards the other box */
  int ref = best >= 3, ax = ref ? best-3 : best;
  real (*Ar)[3] = ref ? B : A; real (*Ai)[3] = ref ? A : B;
  const real *pr = ref ? p2 : p1, *pi = ref ? p1 : p2, *hr = ref ? h2 : h1, *hi = ref ? h1 : h2;
  real sgn = (ref ? -tB[ax] : tA[ax]) >= 0 ? (real)1 : (real)-1;
  real n[3] = { sgn*Ar[ax][0], sgn*Ar[ax][1], sgn*Ar[ax][2] };
  /* incident face: the face of the other box whose outward normal is most anti-parallel to n */
  int inc = 0; real bd = fabs(dot3(n, Ai[0]));
  for (int k = 1; k < 3; k++) { real v = fabs(dot3(n, Ai[k])); if (v > bd + (real)1e-6) { bd = v; inc = k; } }
  real si = dot3(n, Ai[inc]) > 0 ? (real)-1 : (real)1;
  int k1 = (inc+1)%3, k2 = (inc+2)%3, u1 = (ax+1)%3, u2 = (ax+2)%3;
  real poly[16][3], tmp[16][3]; int np_ = 4;
  for (int v = 0; v < 4; v++) {
    real s1 = (v == 0 || v == 3) ? hi[k1] : -hi[k1], s2 = (v < 2) ? hi[k2] : -hi[k2];
    for (int x = 0; x < 3; x++) poly[v][x] = pi[x] + si*hi[inc]*Ai[inc][x] + s1*Ai[k1][x] + s2*Ai[k2][x];
  }
  /* clip against the four side planes of the reference face: +-u1, +-u2 */
  for (int pl = 0; pl < 4 && np_ > 0; pl++) {
    const real* u = Ar[pl < 2 ? u1 : u2]; real lim = hr[pl < 2 ? u1 : u2] + (real)1e-6, sg = (pl & 1) ? (real)-1 : (real)1;
    int nt = 0;
    for (int v = 0; v < np_; v++) {
      const real *P = poly[v], *Qv = poly[(v+1)%np_];
      real dP = sg*((P[0]-pr[0])*u[0] + (P[1]-pr[1])*u[1] + (P[2]-pr[2])*u[2]) - lim;
      real dQ = sg*((Qv[0]-pr[0])*u[0] + (Qv[1]-pr[1])*u[1] + (Qv[2]-pr[2])*u[2]) - lim;
      if (dP <= 0) { for (int x = 0; x < 3; x++) tmp[nt][x] = P[x]; nt++; }
      if ((dP <= 0) != (dQ <= 0)) { real f = dP / (dP - dQ); for (int x = 0; x < 3; x++) tmp[nt][x] = P[x] + f*(Qv[x]-P[x]); nt++; }
    }
    np_ = nt > 8 ? 8 : nt;
    for (int v = 0; v < np_; v++) for (int x = 0; x < 3; x++) poly[v][x] = tmp[v][x];
  }
  int nc = 0;
  for (int v = 0; v < np_ && nc < 8; v++) {
    real depth = hr[ax] - ((poly[v][0]-pr[0])*n[0] + (poly[v][1]-pr[1])*n[1] + (poly[v][2]-pr[2])*n[2]);
    if (depth < -margin) continue;
    c[nc].dist = -depth;
    for (int x = 0; x < 3; x++) {
      c[nc].pos[x] = poly[v][x] + (real)0.5*depth*n[x];
      c[nc].frame[x] = ref ? -n[x] : n[x];  /* from box 1 to box 2 */
    }
    for (int k = 3; k < 9; k++) c[nc].frame[k] = 0;
    nc++;
  }
  return nc;
}
/* mju_makeFrame */
static void make_frame(real* f) {
  normalize3(f);
  if (norm3(f+3) < (real)0.5) {
    f[3] = f[4] = f[5] = 0;
    if (f[1] < (real)0.5 && f[1] > (real)-0.5) f[4] = 1; else f[5] = 1;
  }
  real t = dot3(f, f+3);
  for (int k = 0; k < 3; k++) f[3+k] -= t*f[k];
  normalize3(f+3);
  cross3(f+6, f, f+3);
}

/* contact parameters (mj_contactParam) + append to the contact list; returns the new count */
static int emit_contacts(W* d, int ncon, int g1, int g2, RawCon* rc, int n, real margin) {
  const B2Oracle* o = d->o; int w = d->w;
  const real* ggap = M_(o, geom_gap, w);
  const real* gfri = M_(o, geom_friction, w); const real* gsolref = M_(o, geom_solref, w);
  const real* gsolimp = M_(o, geom_solimp, w); const real* gsolmix = M_(o, geom_solmix, w);
  int condim; real fri[3], solref[2], solimp[5];
  int pr1 = o->geom_priority[g1], pr2 = o->geom_priority[g2];
  if (pr1 != pr2) {
    int g = pr1 > pr2 ? g1 : g2;
    condim = o->geom_condim[g];
    for (int k = 0; k < 3; k++) fri[k] = gfri[3*g+k];
    for (int k = 0; k < 2; k++) solref[k] = gsolref[2*g+k];
    for (int k = 0; k < 5; k++) solimp[k] = gsolimp[5*g+k];
  } else {
    condim = o->geom_condim[g1] > o->geom_condim[g2] ? o->geom_condim[g1] : o->geom_condim[g2];
    for (int k = 0; k < 3; k++) fri[k] = gfri[3*g1+k] > gfri[3*g2+k] ? gfri[3*g1+k] : gfri[3*g2+k];
    real mix, s1 = gsolmix[g1], s2 = gsolmix[g2];
    if (s1 >= MINVAL && s2 >= MINVAL) mix = s1/(s1+s2);
    else if (s1 < MINVAL && s2 < MINVAL) mix = (real)0.5;
    else mix = s1 < MINVAL ? 0 : 1;
    if (gsolref[2*g1] > 0 && gsolref[2*g2] > 0)
      for (int k = 0; k < 2; k++) solref[k] = mix*gsolref[2*g1+k] + (1-mix)*gsolref[2*g2+k];
    else
      for (int k = 0; k < 2; k++) solref[k] = gsolref[2*g1+k] < gsolref[2*g2+k] ? gsolref[2*g1+k] : gsolref[2*g2+k];
    for (int k = 0; k < 5; k++) solimp[k] = mix*gsolimp[5*g1+k] + (1-mix)*gsolimp[5*g2+k];
  }
  real gap = ggap[g1] > ggap[g2] ? ggap[g1] : ggap[g2];
  for (int i = 0; i < n; i++) {
    if (ncon >= o->maxcon) { *d->overflow = 1; break; }
    make_frame(rc[i].frame);
    d->contact_dist[ncon] = rc[i].dist;
    memcpy(d->contact_pos + 3*ncon, rc[i].pos, sizeof(real)*3);
    memcpy(d->contact_frame + 9*ncon, rc[i].frame, sizeof(real)*9);
    real* f5 = d->contact_friction + 5*ncon;
    f5[0] = f5[1] = fri[0]; f5[2] = fri[1]; f5[3] = f5[4] = fri[2];
    for (int k = 0; k < 5; k++) if (f5[k] < MINMU) f5[k] = MINMU;
    memcpy(d->contact_solref + 2*ncon, solref, sizeof(real)*2);
    memcpy(d->contact_solimp + 5*ncon, solimp, sizeof(real)*5);
    d->contact_includemargin[ncon] = margin - gap;
    d->contact_dim[ncon] = condim;
    d->contact_geom[2*ncon] = g1; d->contact_geom[2*ncon+1] = g2;
    d->contact_efc[ncon] = -1;
    ncon++;
  }
  return ncon;
}

/* narrowphase dispatch; geoms are ordered so that type(g1) <= type(g2) */
static int narrowphase(const W* d, RawCon* rc, int g1, int g2, real margin) {
  const B2Oracle* o = d->o; int w = d->w;
  const real* gsize = M_(o, geom_size, w);
  int t1 = o->geom_type[g1], t2 = o->geom_type[g2];
  const real *p1 = d->geom_xpos + 3*g1, *p2 = d->geom_xpos + 3*g2;
  const real *m1 = d->geom_xmat + 9*g1, *m2 = d->geom_xmat + 9*g2;
  const real *s1 = gsize + 3*g1, *s2 = gsize + 3*g2;
  if (t1 == G_PLANE && t2 == G_SPHERE) return plane_sphere(rc, margin, p1, m1, p2, s2[0]);
  if (t1 == G_PLANE && t2 == G_CAPSULE) return plane_capsule(rc, margin, p1, m1, p2, m2, s2);
  if (t1 == G_PLANE && t2 == G_BOX) return plane_box(rc, margin, p1, m1, p2, m2, s2);
  if (t1 == G_SPHERE && t2 == G_SPHERE) return sphere_sphere(rc, margin, p1, s1[0], p2, s2[0]);
  if (t1 == G_SPHERE && t2 == G_CAPSULE) return sphere_capsule(rc, margin, p1, s1[0], p2, m2, s2);
  if (t1 == G_CAPSULE && t2 == G_CAPSULE) return capsule_capsule(rc, margin, p1, m1, s1, p2, m2, s2);
  if (t1 == G_SPHERE && t2 == G_BOX) return sphere_box(rc, margin, p1, s1[0], p2, m2, s2);
  if (t1 == G_CAPSULE && t2 == G_BOX) return capsule_box(rc, margin, p1, m1, s1, p2, m2, s2);
  if (t1 == G_BOX && t2 == G_BOX) return box_box(rc, margin, p1, m1, s1, p2, m2, s2);
  if (t2 == G_MESH || t1 == G_HFIELD || t1 == G_ELLIPSOID || t1 == G_CYLINDER || t2 == G_ELLIPSOID || t2 == G_CYLINDER) {  /* convex routines (b2_convex.h) */
    const real* rb = M_(o, geom_rbound, w);
    B2CCon cc[B2C_MAXOUT];
    B2CShape A, B;
    const real* v2 = NULL; int n2 = 0;
    if (t2 == G_MESH) { int id = o->geom_dataid[g2]; v2 = o->mesh_vert.p + 3*o->mesh_vertadr[id]; n2 = o->mesh_vertnum[id]; }
    real r2 = b2c_shape(&B, t2, p2, m2, s2, v2, n2);
    if (t1 == G_PLANE) {
      real pn[3] = { m1[2], m1[5], m1[8] };
      if (t2 == G_CYLINDER) return from_b2c(rc, cc, b2c_plane_cylinder(cc, margin, p1, pn, p2, m2, s2));
      if (t2 == G_ELLIPSOID) return from_b2c(rc, cc, b2c_plane_ellipsoid(cc, margin, p1, pn, &B));
      return from_b2c(rc, cc, b2c_plane_mesh(cc, margin, p1, pn, &B));
    }
    if (t1 == G_HFIELD) {
      if (t2 == G_HFIELD) return 0;
      int id = o->geom_dataid[g1];
      return from_b2c(rc, cc, b2c_hfield(cc, margin, p1, m1, o->hfield_size.p + 4*id, o->hfield_nrow[id], o->hfield_ncol[id],
                                         o->hfield_data.p + o->hfield_adr[id], &B, r2, p2, rb[g2]));
    }
    const real* v1 = NULL; int n1 = 0;
    if (t1 == G_MESH) { int id = o->geom_dataid[g1]; v1 = o->mesh_vert.p + 3*o->mesh_vertadr[id]; n1 = o->mesh_vertnum[id]; }
    real r1 = b2c_shape(&A, t1, p1, m1, s1, v1, n1);
    return from_b2c(rc, cc, b2c_pair(cc, margin, &A, r1, &B, r2, p1, p2, rb[g1] + rb[g2]));
  }
  return 0;
}

static void collision(W* d) {
  const B2Oracle* o = d->o; int w = d->w;
  int ncon = 0; *d->overflow = 0;
  const real* rb = M_(o, geom_rbound, w);
  const real* gmargin = M_(o, geom_margin, w);
  /* (1) static pair table with a bounding-sphere filter (mj_collideSphere / plane variant) */
  for (int p = 0; p < o->npair; p++) {
    int g1 = o->pair_geom1[p], g2 = o->pair_geom2[p];
    real margin = gmargin[g1] > gmargin[g2] ? gmargin[g1] : gmargin[g2];
    const real *p1 = d->geom_xpos + 3*g1, *p2 = d->geom_xpos + 3*g2;
    const real *m1 = d->geom_xmat + 9*g1;
    if (o->geom_type[g1] == G_PLANE) {
      real n[3] = { m1[2], m1[5], m1[8] }, dif[3] = { p2[0]-p1[0], p2[1]-p1[1], p2[2]-p1[2] };
      if (dot3(dif, n) > margin + rb[g2]) continue;
    } else {
      real dif[3] = { p2[0]-p1[0], p2[1]-p1[1], p2[2]-p1[2] };
      real bound = margin + rb[g1] + rb[g2];
      if (dot3(dif, dif) > bound*bound) continue;
    }
    RawCon rc[8];
    int n = narrowphase(d, rc, g1, g2, margin);
    if (n) ncon = emit_contacts(d, ncon, g1, g2, rc, n, margin);
  }
  /* (2) grid-static geoms: every dynamic collision geom (id order) visits the cells under its bounding
   * sphere; a static geom spanning several cells is taken only in the first common cell.  The candidates of one
   * dynamic geom are processed in ascending static index, so the contact order does not depend on which cell a
   * candidate was found in (a bounding sphere touching a cell border lands in either cell in fp32). */
  for (int q = 0; q < o->ndyn; q++) {
    int g = o->dyn_cgeom[q];
    const real* c = d->geom_xpos + 3*g;
    int ix0 = (int)floor((c[0] - rb[g] - o->grid_x0) / o->grid_cell), ix1 = (int)floor((c[0] + rb[g] - o->grid_x0) / o->grid_cell);
    int iy0 = (int)floor((c[1] - rb[g] - o->grid_y0) / o->grid_cell), iy1 = (int)floor((c[1] + rb[g] - o->grid_y0) / o->grid_cell);
    if (ix0 < 0) ix0 = 0;
    if (iy0 < 0) iy0 = 0;
    if (ix1 >= o->grid_nx) ix1 = o->grid_nx - 1;
    if (iy1 >= o->grid_ny) iy1 = o->grid_ny - 1;
    int cand[1024], ncand = 0;
    for (int ix = ix0; ix <= ix1; ix++)
      for (int iy = iy0; iy <= iy1; iy++) {
        int cell = ix*o->grid_ny + iy;
        for (int it = o->grid_start[cell]; it < o->grid_start[cell+1]; it++) {
          int k = o->grid_items[it], sg = o->static_geom[k];
          int fx = o->static_cell0[2*k] > ix0 ? o->static_cell0[2*k] : ix0;
          int fy = o->static_cell0[2*k+1] > iy0 ? o->static_cell0[2*k+1] : iy0;
          if (ix != fx || iy != fy) continue;   /* duplicate: handled in an earlier cell */
          if (!((o->geom_contype[g] & o->geom_conaffinity[sg]) || (o->geom_contype[sg] & o->geom_conaffinity[g]))) continue;
          if (ncand < 1024) cand[ncand++] = k;
        }
      }
    for (int a = 1; a < ncand; a++) {  /* insertion sort by static index */
      int v = cand[a], b = a - 1;
      while (b >= 0 && cand[b] > v) { cand[b+1] = cand[b]; b--; }
      cand[b+1] = v;
    }
    for (int a = 0; a < ncand; a++) {
      int sg = o->static_geom[cand[a]];
      real margin = gmargin[g] > gmargin[sg] ? gmargin[g] : gmargin[sg];
      int g1 = g, g2 = sg;
      if (o->geom_type[g1] > o->geom_type[g2] || (o->geom_type[g1] == o->geom_type[g2] && g1 > g2)) { g1 = sg; g2 = g; }
      RawCon rc[8];
      int n = narrowphase(d, rc, g1, g2, margin);
      if (n) ncon = emit_contacts(d, ncon, g1, g2, rc, n, margin);
    }
  }
  *d->ncon = ncon;
}

/* ---------------------------------------------------------------------------------------------
 * constraints: mj_makeConstraint / mj_makeImpedance / mj_referenceConstraint
 * (engine_core_constraint.c)
 * ------------------------------------------------------------------------------------------- */
typedef struct { real solref[2], solimp[5]; } RowPar;

static void make_constraint(W* d, RowPar* par, real* diag, real* jacp1, real* jacp2) {
  const B2Oracle* o = d->o; int w = d->w; int nv = o->nv, nefc = 0;
  const real* range = M_(o, jnt_range, w); const real* jmargin = M_(o, jnt_margin, w);
  const real* qpos = d->qpos;
  /* joint limits (mj_instantiateLimit) */
  for (int j = 0; j < o->njnt; j++) {
    if (!o->jnt_limited[j]) continue;
    if (o->jnt_type[j] != JNT_HINGE && o->jnt_type[j] != JNT_SLIDE) continue;
    real value = qpos[o->jnt_qposadr[j]];
    for (int side = -1; side <= 1; side += 2) {
      real dist = side * (range[2*j + (side+1)/2] - value);
      if (dist < jmargin[j]) {
        if (nefc >= o->njmax) { *d->overflow = 1; continue; }
        real* J = d->efc_J + (size_t)nefc*nv;
        memset(J, 0, sizeof(real)*nv);
        J[o->jnt_dofadr[j]] = -(real)side;
        d->efc_pos[nefc] = dist; d->efc_margin[nefc] = jmargin[j];
        d->efc_type[nefc] = EFC_LIMIT; d->efc_id[nefc] = j;
        memcpy(par[nefc].solref, M_(o, jnt_solref, w) + 2*j, sizeof(real)*2);
        memcpy(par[nefc].solimp, M_(o, jnt_solimp, w) + 5*j, sizeof(real)*5);
        diag[nefc] = M_(o, dof_invweight0, w)[o->jnt_dofadr[j]];
        nefc++;
      }
    }
  }
  /* contacts (mj_instantiateContact), pyramidal cone */
  const real* inv = M_(o, body_invweight0, w);
  for (int c = 0; c < *d->ncon; c++) {
    if (d->contact_dist[c] >= d->contact_includemargin[c]) continue; /* con->exclude */
    int dim = d->contact_dim[c];
    int nrow = dim == 1 ? 1 : 2*(dim-1);
    if (nefc + nrow > o->njmax) { *d->overflow = 1; continue; }
    int b1 = o->geom_bodyid[d->contact_geom[2*c]], b2 = o->geom_bodyid[d->contact_geom[2*c+1]];
    jac_point(d, jacp1, NULL, d->contact_pos + 3*c, b1);
    jac_point(d, jacp2, NULL, d->contact_pos + 3*c, b2);
    const real* fr = d->contact_frame + 9*c; const real* mu = d->contact_friction + 5*c;
    real tran = inv[2*b1] + inv[2*b2];
    d->contact_efc[c] = nefc;
    for (int r = 0; r < nrow; r++) {
      real* J = d->efc_J + (size_t)(nefc+r)*nv;
      real sgn = (r & 1) ? (real)-1 : (real)1; int t = r/2;
      for (int i = 0; i < nv; i++) {
        real dif[3] = { jacp2[i]-jacp1[i], jacp2[nv+i]-jacp1[nv+i], jacp2[2*nv+i]-jacp1[2*nv+i] };
        real jn = dot3(fr, dif);
        if (dim == 1) J[i] = jn;
        else J[i] = jn + sgn*mu[t]*dot3(fr + 3*(t+1), dif);
      }
      d->efc_pos[nefc+r] = d->contact_dist[c]; d->efc_margin[nefc+r] = d->contact_includemargin[c];
      d->efc_type[nefc+r] = dim == 1 ? EFC_FRICTIONLESS : EFC_PYRAMIDAL; d->efc_id[nefc+r] = c;
      memcpy(par[nefc+r].solref, d->contact_solref + 2*c, sizeof(real)*2);
      memcpy(par[nefc+r].solimp, d->contact_solimp + 5*c, sizeof(real)*5);
      /* mj_diagApprox */
      diag[nefc+r] = dim == 1 ? tran : tran + mu[t]*mu[t]*tran;
    }
    nefc += nrow;
  }
  *d->nefc = nefc;
}

static void make_impedance_and_ref(W* d, const RowPar* par, const real* diag) {
  const B2Oracle* o = d->o; int nv = o->nv, nefc = *d->nefc;
  real* kb = (real*)malloc(sizeof(real)*3*(nefc ? nefc : 1));
  for (int i = 0; i < nefc; i++) {
    const real* si = par[i].solimp; const real* sr = par[i].solref;
    real dmin = fmin(fmax(si[0], MINIMP), MAXIMP), dmax = fmin(fmax(si[1], MINIMP), MAXIMP);
    real width = fmax(si[2], MINVAL), mid = fmin(fmax(si[3], MINIMP), MAXIMP), power = fmax(si[4], 1);
    real x = fabs(d->efc_pos[i] - d->efc_margin[i]) / width, y, imp;
    if (x >= 1) imp = dmax;
    else if (x <= 0) imp = dmin;
    else {
      if (power == 1) y = x;
      else if (x <= mid) y = pow(x, power) / pow(mid, power-1);
      else y = 1 - pow(1-x, power) / pow(1-mid, power-1);
      imp = dmin + y*(dmax-dmin);
    }
    real K, B;
    if (sr[0] > 0) {
      real tc = fmax(sr[0], 2*o->timestep), dr = sr[1]; /* refsafe */
      K = 1 / fmax(MINVAL, dmax*dmax*tc*tc*dr*dr);
      B = 2 / fmax(MINVAL, dmax*tc);
    } else { K = -sr[0]/(dmax*dmax); B = -sr[1]/dmax; }
    kb[3*i] = K; kb[3*i+1] = B; kb[3*i+2] = imp;
    d->efc_R[i] = fmax(MINVAL, (1-imp)*diag[i]/imp);
  }
  /* pyramidal: all edges of a contact share R = 2 mu^2 R(first edge) */
  for (int i = 0; i < nefc; i++) {
    if (d->efc_type[i] != EFC_PYRAMIDAL) continue;
    int c = d->efc_id[i]; int nrow = 2*(d->contact_dim[c]-1);
    real mu = d->contact_friction[5*c] / sqrt(o->impratio);
    real Rpy = 2*mu*mu*d->efc_R[i];
    for (int r = 0; r < nrow; r++) d->efc_R[i+r] = fmax(MINVAL, Rpy);
    i += nrow-1;
  }
  for (int i = 0; i < nefc; i++) {
    d->efc_D[i] = 1/d->efc_R[i];
    real vel = 0; const real* J = d->efc_J + (size_t)i*nv;
    for (int k = 0; k < nv; k++) vel += J[k]*d->qvel[k];
    d->efc_vel[i] = vel;
    d->efc_aref[i] = -kb[3*i+1]*vel - kb[3*i]*kb[3*i+2]*(d->efc_pos[i] - d->efc_margin[i]);
  }
  free(kb);
}

/* ---------------------------------------------------------------------------------------------
 * velocity / actuation / acceleration stages
 * ------------------------------------------------------------------------------------------- */
static void com_vel(W* d) {
  const B2Oracle* o = d->o; int nb = o->nbody;
  memset(d->cvel, 0, sizeof(real)*6);
  for (int i = 1; i < nb; i++) {
    real cvel[6]; memcpy(cvel, d->cvel + 6*o->body_parentid[i], sizeof(real)*6);
    int bda = o->body_dofadr[i];
    for (int j = o->body_jntadr[i]; j < o->body_jntadr[i] + o->body_jntnum[i]; j++) {
      if (o->jnt_type[j] == JNT_FREE) {
        memset(d->cdof_dot + 6*bda, 0, sizeof(real)*18);
        for (int k = 0; k < 3; k++) for (int c = 0; c < 6; c++) cvel[c] += d->cdof[6*(bda+k)+c]*d->qvel[bda+k];
        bda += 3;
        for (int k = 0; k < 3; k++) cross_motion(d->cdof_dot + 6*(bda+k), cvel, d->cdof + 6*(bda+k));
        for (int k = 0; k < 3; k++) for (int c = 0; c < 6; c++) cvel[c] += d->cdof[6*(bda+k)+c]*d->qvel[bda+k];
        bda += 3;
      } else {
        cross_motion(d->cdof_dot + 6*bda, cvel, d->cdof + 6*bda);
        for (int c = 0; c < 6; c++) cvel[c] += d->cdof[6*bda+c]*d->qvel[bda];
        bda++;
      }
    }
    memcpy(d->cvel + 6*i, cvel, sizeof(real)*6);
  }
}

static void rne_bias(W* d, real* cacc, real* cfrc) { /* mj_rne with flg_acc = 0 */
  const B2Oracle* o = d->o; int nb = o->nbody, nv = o->nv;
  cacc[0] = cacc[1] = cacc[2] = 0;
  for (int k = 0; k < 3; k++) cacc[3+k] = -o->gravity[k];
  memset(cfrc, 0, sizeof(real)*6);
  for (int i = 1; i < nb; i++) {
    int bda = o->body_dofadr[i];
    memcpy(cacc + 6*i, cacc + 6*o->body_parentid[i], sizeof(real)*6);
    for (int k = 0; k < o->body_dofnum[i]; k++)
      for (int c = 0; c < 6; c++) cacc[6*i+c] += d->cdof_dot[6*(bda+k)+c]*d->qvel[bda+k];
    real t[6], t1[6];
    mul_inert_vec(t, d->cinert + 10*i, d->cvel + 6*i);
    cross_force(t1, d->cvel + 6*i, t);
    mul_inert_vec(t, d->cinert + 10*i, cacc + 6*i);
    for (int c = 0; c < 6; c++) cfrc[6*i+c] = t[c] + t1[c];
  }
  for (int i = nb-1; i > 0; i--) {
    int p = o->body_parentid[i];
    if (p) for (int c = 0; c < 6; c++) cfrc[6*p+c] += cfrc[6*i+c];
  }
  for (int i = 0; i < nv; i++) d->qfrc_bias[i] = dot6(d->cdof + 6*i, cfrc + 6*o->dof_bodyid[i]);
}

static void passive_and_actuation(W* d) {
  const B2Oracle* o = d->o; int w = d->w; int nv = o->nv;
  const real* damp = M_(o, dof_damping, w); const real* stiff = M_(o, jnt_stiffness, w);
  const real* qpos0 = M_(o, qpos0, w); /* spring reference = qpos0 (qpos_spring) */
  for (int i = 0; i < nv; i++) d->qfrc_passive[i] = -damp[i]*d->qvel[i];
  for (int j = 0; j < o->njnt; j++)
    if (stiff[j] != 0 && (o->jnt_type[j] == JNT_HINGE || o->jnt_type[j] == JNT_SLIDE))
      d->qfrc_passive[o->jnt_dofadr[j]] -= stiff[j]*(d->qpos[o->jnt_qposadr[j]] - qpos0[o->jnt_qposadr[j]]);
  memset(d->qfrc_actuator, 0, sizeof(real)*nv);
  const real* gp = M_(o, actuator_gainprm, w); const real* bp = M_(o, actuator_biasprm, w);
  const real* cr = M_(o, actuator_ctrlrange, w); const real* fr = M_(o, actuator_forcerange, w);
  const real* gear = M_(o, actuator_gear, w);
  for (int a = 0; a < o->nu; a++) { /* mj_fwdActuation: fixed gain, affine bias, joint trn */
    int j = o->actuator_trnid[a];
    real len = d->qpos[o->jnt_qposadr[j]]*gear[a], vel = d->qvel[o->jnt_dofadr[j]]*gear[a];
    real c = d->ctrl[a];
    if (o->actuator_ctrllimited[a]) c = fmin(fmax(c, cr[2*a]), cr[2*a+1]);
    real f = gp[10*a]*c + bp[10*a] + bp[10*a+1]*len + bp[10*a+2]*vel;
    if (o->actuator_forcelimited[a]) f = fmin(fmax(f, fr[2*a]), fr[2*a+1]);
    d->actuator_force[a] = f;
    d->qfrc_actuator[o->jnt_dofadr[j]] += gear[a]*f;
  }
}

static void fwd_acceleration(W* d, real* jacp, real* jacr) {
  const B2Oracle* o = d->o; int nv = o->nv;
  for (int i = 0; i < nv; i++)
    d->qfrc_smooth[i] = d->qfrc_passive[i] - d->qfrc_bias[i] + d->qfrc_applied[i] + d->qfrc_actuator[i];
  for (int b = 1; b < o->nbody; b++) { /* mj_xfrcAccumulate */
    const real* x = d->xfrc_applied + 6*b;
    if (x[0] == 0 && x[1] == 0 && x[2] == 0 && x[3] == 0 && x[4] == 0 && x[5] == 0) continue;
    jac_point(d, jacp, jacr, d->xipos + 3*b, b);
    for (int i = 0; i < nv; i++)
      for (int k = 0; k < 3; k++) d->qfrc_smooth[i] += jacp[k*nv+i]*x[k] + jacr[k*nv+i]*x[3+k];
  }
  memcpy(d->qacc_smooth, d->qfrc_smooth, sizeof(real)*nv);
  chol_solve(d->qL, nv, d->qacc_smooth);
}

/* ---------------------------------------------------------------------------------------------
 * Newton solver, primal (engine_solver.c: mj_solPrimal / PrimalSearch / warmstart)
 * ------------------------------------------------------------------------------------------- */
typedef struct { real alpha, cost, d0, d1; } LSPoint;
typedef struct {
  int nv, nefc; const real *D, *jar, *jv; real g0, g1, g2; /* Gauss quadratic */
} LSCtx;
static LSPoint ls_eval(const LSCtx* c, real a) {
  LSPoint p; p.alpha = a;
  real cost = c->g0 + a*c->g1 + a*a*c->g2, d0 = c->g1 + 2*a*c->g2, d1 = 2*c->g2;
  for (int i = 0; i < c->nefc; i++) {
    real x = c->jar[i] + a*c->jv[i];
    if (x < 0) {
      cost += (real)0.5*c->D[i]*x*x;
      d0 += c->D[i]*x*c->jv[i];
      d1 += c->D[i]*c->jv[i]*c->jv[i];
    }
  }
  p.cost = cost; p.d0 = d0; p.d1 = d1 < MINVAL ? MINVAL : d1;
  return p;
}
static real ls_search(const LSCtx* c, real gtol, int maxit) {
  LSPoint p0 = ls_eval(c, 0);
  LSPoint p1 = ls_eval(c, -p0.d0/p0.d1);
  if (p0.cost < p1.cost) p1 = p0;
  if (fabs(p1.d0) < gtol) return p1.alpha;
  int it = 0; real dir = p1.d0 < 0 ? 1 : -1;
  LSPoint p2 = p1;
  /* Newton steps in one direction until the derivative changes sign (bracket) */
  while (p1.d0*dir <= -gtol && it < maxit) {
    p2 = p1;
    p1 = ls_eval(c, p1.alpha - p1.d0/p1.d1);
    it++;
    if (fabs(p1.d0) < gtol) return p1.alpha;
  }
  if (it >= maxit) return p1.alpha;
  /* bracket [p2, p1] holds the root: Newton from both ends + midpoint, keep tightening */
  while (it < maxit) {
    LSPoint c1 = ls_eval(c, p1.alpha - p1.d0/p1.d1);
    LSPoint c2 = ls_eval(c, p2.alpha - p2.d0/p2.d1);
    LSPoint cm = ls_eval(c, (real)0.5*(p1.alpha + p2.alpha));
    it++;
    LSPoint cand[3] = { c1, c2, cm };
    real lo = fmin(p1.alpha, p2.alpha), hi = fmax(p1.alpha, p2.alpha);
    int moved = 0;
    for (int k = 0; k < 3; k++) {
      if (fabs(cand[k].d0) < gtol) return cand[k].alpha;
      if (cand[k].alpha <= lo || cand[k].alpha >= hi) continue;
      if (cand[k].d0*dir < 0) { /* same side as p2 */
        if (fabs(cand[k].alpha - p1.alpha) < fabs(p2.alpha - p1.alpha)) { p2 = cand[k]; moved = 1; }
      } else {
        if (fabs(cand[k].alpha - p2.alpha) < fabs(p1.alpha - p2.alpha)) { p1 = cand[k]; moved = 1; }
      }
      lo = fmin(p1.alpha, p2.alpha); hi = fmax(p1.alpha, p2.alpha);
    }
    if (!moved) break;
  }
  return p1.cost < p2.cost ? p1.alpha : p2.alpha;
}

typedef struct { real *Ma, *jar, *grad, *search, *Mv, *jv, *H, *force; } SolveBuf;

static real update_constraint(W* d, SolveBuf* s) { /* PrimalUpdateConstraint + gradient */
  const B2Oracle* o = d->o; int nv = o->nv, nefc = *d->nefc;
  real cost = 0;
  memset(d->qfrc_constraint, 0, sizeof(real)*nv);
  for (int i = 0; i < nefc; i++) {
    if (s->jar[i] < 0) {
      d->efc_force[i] = -d->efc_D[i]*s->jar[i];
      cost += (real)0.5*d->efc_D[i]*s->jar[i]*s->jar[i];
      const real* J = d->efc_J + (size_t)i*nv;
      for (int k = 0; k < nv; k++) d->qfrc_constraint[k] += J[k]*d->efc_force[i];
    } else d->efc_force[i] = 0;
  }
  real gauss = 0;
  for (int k = 0; k < nv; k++) gauss += (s->Ma[k] - d->qfrc_smooth[k])*(d->qacc[k] - d->qacc_smooth[k]);
  return cost + (real)0.5*gauss;
}
static void update_gradient(W* d, SolveBuf* s) { /* Newton: search = -H^-1 grad */
  const B2Oracle* o = d->o; int nv = o->nv, nefc = *d->nefc;
  for (int k = 0; k < nv; k++) s->grad[k] = s->Ma[k] - d->qfrc_smooth[k] - d->qfrc_constraint[k];
  memcpy(s->H, d->qM, sizeof(real)*nv*nv);
  for (int i = 0; i < nefc; i++) {
    if (!(s->jar[i] < 0)) continue;
    const real* J = d->efc_J + (size_t)i*nv; real Di = d->efc_D[i];
    for (int a = 0; a < nv; a++) {
      if (J[a] == 0) continue;
      real t = Di*J[a];
      for (int b = 0; b <= a; b++) s->H[a*nv+b] += t*J[b];
    }
  }
  for (int a = 0; a < nv; a++) for (int b = a+1; b < nv; b++) s->H[a*nv+b] = s->H[b*nv+a];
  chol_factor(s->H, nv);
  for (int k = 0; k < nv; k++) s->search[k] = -s->grad[k];
  chol_solve(s->H, nv, s->search);
}

static void solve(W* d, SolveBuf* s) {
  const B2Oracle* o = d->o; int nv = o->nv, nefc = *d->nefc;
  *d->solver_niter = 0;
  if (nefc == 0) {
    memcpy(d->qacc, d->qacc_smooth, sizeof(real)*nv);
    memset(d->qfrc_constraint, 0, sizeof(real)*nv);
    return;
  }
  /* warmstart (mj_fwdConstraint): keep qacc_warmstart unless qacc_smooth has lower cost */
  real cost_warm = 0, cost_smooth = 0;
  memcpy(d->qacc, d->qacc_warmstart, sizeof(real)*nv);
  for (int i = 0; i < nv; i++) {
    real t = 0; for (int k = 0; k < nv; k++) t += d->qM[i*nv+k]*d->qacc[k];
    s->Ma[i] = t;
  }
  for (int i = 0; i < nefc; i++) {
    const real* J = d->efc_J + (size_t)i*nv; real jw = -d->efc_aref[i], js = -d->efc_aref[i];
    for (int k = 0; k < nv; k++) { jw += J[k]*d->qacc[k]; js += J[k]*d->qacc_smooth[k]; }
    if (jw < 0) cost_warm += (real)0.5*d->efc_D[i]*jw*jw;
    if (js < 0) cost_smooth += (real)0.5*d->efc_D[i]*js*js;
  }
  real g = 0;
  for (int k = 0; k < nv; k++) g += (s->Ma[k] - d->qfrc_smooth[k])*(d->qacc[k] - d->qacc_smooth[k]);
  cost_warm += (real)0.5*g;
  if (cost_warm > cost_smooth) memcpy(d->qacc, d->qacc_smooth, sizeof(real)*nv);
  /* initialise */
  for (int i = 0; i < nv; i++) {
    real t = 0; for (int k = 0; k < nv; k++) t += d->qM[i*nv+k]*d->qacc[k];
    s->Ma[i] = t;
  }
  for (int i = 0; i < nefc; i++) {
    const real* J = d->efc_J + (size_t)i*nv; real t = -d->efc_aref[i];
    for (int k = 0; k < nv; k++) t += J[k]*d->qacc[k];
    s->jar[i] = t;
  }
  real scale = 1 / (o->meaninertia * (nv > 1 ? nv : 1));
  real cost = update_constraint(d, s);
  update_gradient(d, s);
  int iter = 0;
  for (; iter < o->iterations; ) {
    /* line search along `search` */
    real snorm = 0; for (int k = 0; k < nv; k++) snorm += s->search[k]*s->search[k];
    snorm = sqrt(snorm);
    if (snorm < MINVAL) break;
    for (int i = 0; i < nv; i++) {
      real t = 0; for (int k = 0; k < nv; k++) t += d->qM[i*nv+k]*s->search[k];
      s->Mv[i] = t;
    }
    for (int i = 0; i < nefc; i++) {
      const real* J = d->efc_J + (size_t)i*nv; real t = 0;
      for (int k = 0; k < nv; k++) t += J[k]*s->search[k];
      s->jv[i] = t;
    }
    LSCtx c; c.nv = nv; c.nefc = nefc; c.D = d->efc_D; c.jar = s->jar; c.jv = s->jv;
    c.g0 = 0; c.g1 = 0; c.g2 = 0;
    for (int k = 0; k < nv; k++) {
      c.g1 += s->search[k]*(s->Ma[k] - d->qfrc_smooth[k]);
      c.g2 += (real)0.5*s->search[k]*s->Mv[k];
    }
    real gtol = o->tolerance * o->ls_tolerance * snorm / scale;
    real alpha = ls_search(&c, gtol, o->ls_iterations);
    if (alpha == 0) break;
    for (int k = 0; k < nv; k++) { d->qacc[k] += alpha*s->search[k]; s->Ma[k] += alpha*s->Mv[k]; }
    for (int i = 0; i < nefc; i++) s->jar[i] += alpha*s->jv[i];
    real oldcost = cost;
    cost = update_constraint(d, s);
    update_gradient(d, s);
    iter++;
    real improvement = scale*(oldcost - cost), gn = 0;
    for (int k = 0; k < nv; k++) gn += s->grad[k]*s->grad[k];
    if (improvement < o->tolerance || scale*sqrt(gn) < o->tolerance) break;
  }
  *d->solver_niter = iter;
  *d->solver_cost = cost;
}

/* contact force in the contact frame (mj_contactForce / mju_decodePyramid) */
static void contact_forces(W* d) {
  for (int c = 0; c < *d->ncon; c++) {
    real* f = d->contact_force + 3*c; f[0] = f[1] = f[2] = 0;
    int a = d->contact_efc[c]; if (a < 0) continue;
    int dim = d->contact_dim[c];
    if (dim == 1) { f[0] = d->efc_force[a]; continue; }
    const real* mu = d->contact_friction + 5*c;
    for (int t = 0; t < dim-1 && t < 2; t++) {
      f[0] += d->efc_force[a+2*t] + d->efc_force[a+2*t+1];
      f[1+t] = (d->efc_force[a+2*t] - d->efc_force[a+2*t+1])*mu[t];
    }
  }
}

/* contact sensors (engine_sensor.c, mjSENS_CONTACT): data in {found,force,dist,pos,normal},
 * reduce in {none, netforce} */
static int in_subtree(const B2Oracle* o, int body, int rootb) {
  while (body) { if (body == rootb) return 1; body = o->body_parentid[body]; }
  return rootb == 0;
}
static int match_obj(const B2Oracle* o, int type, int id, int geom) {
  if (type < 0) return 1;
  int b = o->geom_bodyid[geom];
  if (type == OBJ_GEOM) return geom == id;
  if (type == OBJ_BODY) return b == id;
  if (type == OBJ_XBODY) return in_subtree(o, b, id);
  return 0;
}
static void sensors(W* d) {
  const B2Oracle* o = d->o;
  memset(d->sensordata, 0, sizeof(real)*o->nsensordata);
  for (int s = 0; s < o->nsensor; s++) {
    int dataspec = o->sensor_intprm[3*s], reduce = o->sensor_intprm[3*s+1], num = o->sensor_intprm[3*s+2];
    real* out = d->sensordata + o->sensor_adr[s];
    int slot = o->sensor_dim[s] / (num > 0 ? num : 1);
    int nmatch = 0; real net[3] = {0,0,0}, wpos[3] = {0,0,0}, wsum = 0;
    for (int c = 0; c < *d->ncon; c++) {
      if (d->contact_efc[c] < 0) continue;
      int g1 = d->contact_geom[2*c], g2 = d->contact_geom[2*c+1];
      int dir = 0;
      if (match_obj(o, o->sensor_objtype[s], o->sensor_objid[s], g1) &&
          match_obj(o, o->sensor_reftype[s], o->sensor_refid[s], g2)) dir = 1;
      else if (match_obj(o, o->sensor_objtype[s], o->sensor_objid[s], g2) &&
               match_obj(o, o->sensor_reftype[s], o->sensor_refid[s], g1)) dir = -1;
      if (!dir) continue;
      const real* fr = d->contact_frame + 9*c; const real* cf = d->contact_force + 3*c;
      real fw[3];
      for (int k = 0; k < 3; k++) fw[k] = dir*(fr[k]*cf[0] + fr[3+k]*cf[1] + fr[6+k]*cf[2]);
      if (reduce == 3) {
        real mag = norm3(fw);
        for (int k = 0; k < 3; k++) { net[k] += fw[k]; wpos[k] += mag*d->contact_pos[3*c+k]; }
        wsum += mag;
      } else if (reduce == 0 && nmatch < num) {
        real* q = out + nmatch*slot; int a = 0;
        if (dataspec & 1) q[a++] = 0; /* filled with the count below */
        if (dataspec & 2) { q[a] = cf[0]; q[a+1] = dir*cf[1]; q[a+2] = dir*cf[2]; a += 3; }
        if (dataspec & 4) a += 3;
        if (dataspec & 8) q[a++] = d->contact_dist[c];
        if (dataspec & 16) { for (int k = 0; k < 3; k++) q[a+k] = d->contact_pos[3*c+k]; a += 3; }
        if (dataspec & 32) { for (int k = 0; k < 3; k++) q[a+k] = dir*fr[k]; a += 3; }
      }
      nmatch++;
    }
    if (reduce == 3 && nmatch) {
      int a = 0;
      if (dataspec & 1) out[a++] = (real)nmatch;
      if (dataspec & 2) { for (int k = 0; k < 3; k++) out[a+k] = net[k]; a += 3; }
      if (dataspec & 4) a += 3;
      if (dataspec & 8) out[a++] = 0;
      if (dataspec & 16) { for (int k = 0; k < 3; k++) out[a+k] = wsum > 0 ? wpos[k]/wsum : 0; a += 3; }
      if (dataspec & 32) { real n[3] = {net[0],net[1],net[2]}; normalize3(n); for (int k = 0; k < 3; k++) out[a+k] = n[k]; }
    } else if (reduce == 0 && (dataspec & 1)) {
      int filled = nmatch < num ? nmatch : num;
      for (int i = 0; i < filled; i++) out[i*slot] = (real)nmatch;
    }
  }
}

/* ---------------------------------------------------------------------------------------------
 * integrators (engine_forward.c: mj_Euler / mj_implicit with implicitfast, mj_advance)
 * ------------------------------------------------------------------------------------------- */
static void integrate(W* d, real* H, real* rhs) {
  const B2Oracle* o = d->o; int w = d->w; int nv = o->nv; real h = o->timestep;
  const real* damp = M_(o, dof_damping, w);
  const real* bp = M_(o, actuator_biasprm, w); const real* fr = M_(o, actuator_forcerange, w);
  const real* gear = M_(o, actuator_gear, w);
  int need = 0;
  memcpy(H, d->qM, sizeof(real)*nv*nv);
  for (int i = 0; i < nv; i++) if (damp[i] > 0) { H[i*nv+i] += h*damp[i]; need = 1; }
  if (o->integrator == INT_IMPLICITFAST) {
    /* qDeriv = d(qfrc_actuator)/d(qvel) (mjd_actuator_vel): affine bias velocity term;
       skipped when the actuator force is clamped by forcerange */
    for (int a = 0; a < o->nu; a++) {
      real bv = bp[10*a+2];
      if (bv == 0) continue;
      if (o->actuator_forcelimited[a]) {
        real f = d->actuator_force[a];
        if (f <= fr[2*a] || f >= fr[2*a+1]) continue;
      }
      int dof = o->jnt_dofadr[o->actuator_trnid[a]];
      H[dof*nv+dof] -= h*gear[a]*gear[a]*bv;
      need = 1;
    }
    need = 1;
  }
  for (int i = 0; i < nv; i++) rhs[i] = d->qfrc_smooth[i] + d->qfrc_constraint[i];
  if (need) { chol_factor(H, nv); chol_solve(H, nv, rhs); }
  else memcpy(rhs, d->qacc, sizeof(real)*nv);
  /* mj_advance */
  memcpy(d->qacc_warmstart, d->qacc, sizeof(real)*nv);
  for (int i = 0; i < nv; i++) d->qvel[i] += h*rhs[i];
  for (int j = 0; j < o->njnt; j++) { /* mj_integratePos */
    int qa = o->jnt_qposadr[j], da = o->jnt_dofadr[j];
    if (o->jnt_type[j] == JNT_FREE) {
      for (int k = 0; k < 3; k++) d->qpos[qa+k] += h*d->qvel[da+k];
      real* q = d->qpos + qa + 3; real v[3] = { d->qvel[da+3], d->qvel[da+4], d->qvel[da+5] };
      real n = norm3(v);
      if (n > MINVAL) {
        real ax[3] = { v[0]/n, v[1]/n, v[2]/n }, qr[4], qn[4];
        axisangle2quat(qr, ax, h*n);
        mulquat(qn, q, qr);
        memcpy(q, qn, sizeof(real)*4);
      }
      normalize4(q);
    } else d->qpos[qa] += h*d->qvel[da];
  }
  *d->time += h;
}

/* ---------------------------------------------------------------------------------------------
 * pipeline
 * ------------------------------------------------------------------------------------------- */
static void world_forward(const B2Oracle* o, int w, int do_step) {
  W d = bind(o, w);
  int nv = o->nv, nb = o->nbody, nj = o->njmax;
  real* buf = (real*)malloc(sizeof(real) * ((size_t)nb*22 + (size_t)nv*(6 + 2*nv + 6) + (size_t)nj*4 + 64));
  real* crb = buf; real* cacc = crb + 10*nb; real* cfrc = cacc + 6*nb;
  real* jac1 = cfrc + 6*nb; real* jac2 = jac1 + 3*nv;
  SolveBuf s;
  s.Ma = jac2 + 3*nv; s.grad = s.Ma + nv; s.search = s.grad + nv; s.Mv = s.search + nv;
  s.H = s.Mv + nv; real* H2 = s.H + nv*nv; real* rhs = H2 + nv*nv;
  s.jar = rhs + nv; s.jv = s.jar + nj; s.force = s.jv + nj; real* diag = s.force + nj;
  RowPar* par = (RowPar*)malloc(sizeof(RowPar) * (nj ? nj : 1));
  /* position */
  kinematics(&d); com_pos(&d); crb_and_factor(&d, crb); collision(&d);
  make_constraint(&d, par, diag, jac1, jac2);
  /* velocity */
  com_vel(&d); make_impedance_and_ref(&d, par, diag); rne_bias(&d, cacc, cfrc);
  /* actuation, acceleration, constraint */
  passive_and_actuation(&d); fwd_acceleration(&d, jac1, jac2);
  solve(&d, &s); contact_forces(&d); sensors(&d);
  if (do_step) integrate(&d, H2, rhs);
  free(par); free(buf);
}

/* ---------------------------------------------------------------------------------------------
 * public API (test-only)
 * ------------------------------------------------------------------------------------------- */
static void alloc_data(B2Oracle* o) {
  /* the names the Data table's row lengths are written in */
  int nq = o->nq, nv = o->nv, nu = o->nu, nbody = o->nbody, njnt = o->njnt, ngeom = o->ngeom, nsite = o->nsite;
  int nsensordata = o->nsensordata, maxcon = o->maxcon, njmax = o->njmax;
#define X(n, len)                                                                               \
  o->data.n.rowlen = len;                                                                       \
  o->data.n.p = calloc((size_t)o->nworld * (o->data.n.rowlen ? o->data.n.rowlen : 1), sizeof *o->data.n.p);
  DATA_REAL(X) DATA_INT(X)
#undef X
}
B2Oracle* b2o_create(const B2ModelDesc* desc, int nworld, int maxcon, int njmax) {
  B2Oracle* o = (B2Oracle*)calloc(1, sizeof(B2Oracle));
#define X(m, arr, k) o->m = get_scalar(desc, #arr, k);
  MODEL_SCALAR(X)
#undef X
  for (int k = 0; k < 3; k++) o->gravity[k] = (real)desc->gravity[k];
  o->nworld = nworld; o->maxcon = maxcon > 0 ? maxcon : 64; o->njmax = njmax > 0 ? njmax : 300;
  o->ndyn = (int)find_arr(desc, "dyn_cgeom")->n;
#define X(n) o->n = dup_i(desc, #n);
  MODEL_INT(X)
#undef X
#define X(n) o->n = dup_f(desc, #n);
  MODEL_REAL(X)
#undef X
  alloc_data(o);
  for (int w = 0; w < nworld; w++)
    for (int i = 0; i < o->nq; i++) o->data.qpos.p[(size_t)w*o->nq + i] = o->qpos0.p[i];
  return o;
}
void b2o_destroy(B2Oracle* o) {
  if (!o) return;
#define X(n, len) free(o->data.n.p);
  DATA_REAL(X) DATA_INT(X)
#undef X
#define X(n) free(o->n);
  MODEL_INT(X)
#undef X
#define X(n) free(o->n.p);
  MODEL_REAL(X)
#undef X
  free(o);
}
int b2o_real_size(void) { return (int)sizeof(real); }
/* Data field [nworld][*rowlen] by name, of int (*is_int = 1) or real elements; NULL for an unknown name */
void* b2o_field(B2Oracle* o, const char* name, int* rowlen, int* is_int) {
#define X(n, len) if (!strcmp(name, #n)) { *rowlen = o->data.n.rowlen; *is_int = 0; return o->data.n.p; }
  DATA_REAL(X)
#undef X
#define X(n, len) if (!strcmp(name, #n)) { *rowlen = o->data.n.rowlen; *is_int = 1; return o->data.n.p; }
  DATA_INT(X)
#undef X
  return NULL;
}
/* per-world model field (expands it on first use); returns pointer to [nworld][n] reals */
void* b2o_model_field(B2Oracle* o, const char* name, int* n) {
  MF* f = NULL;
#define X(nm) if (!strcmp(name, #nm)) f = &o->nm;
  MODEL_REAL(X)
#undef X
  if (!f) return NULL;
  if (f->stride == 0) {
    real* p = (real*)malloc(sizeof(real) * (size_t)o->nworld * (f->n ? f->n : 1));
    for (int w = 0; w < o->nworld; w++) memcpy(p + (size_t)w*f->n, f->p, sizeof(real)*f->n);
    free(f->p); f->p = p; f->stride = f->n;
  }
  *n = f->n;
  return f->p;
}
/* returns 0, or 1 for a name not in OPTIONS */
int b2o_set_option(B2Oracle* o, const char* key, double v) {
#define X(n, type) if (!strcmp(key, #n)) { o->n = (type)v; return 0; }
  OPTIONS(X)
#undef X
  return 1;
}
static void run(B2Oracle* o, int do_step, int nthread) {
#ifdef _OPENMP
  if (nthread > 0) omp_set_num_threads(nthread);
#pragma omp parallel for schedule(static)
#endif
  for (int w = 0; w < o->nworld; w++) world_forward(o, w, do_step);
  (void)nthread;
}
void b2o_forward(B2Oracle* o, int nthread) { run(o, 0, nthread); }
void b2o_step(B2Oracle* o, int nthread) { run(o, 1, nthread); }
int b2o_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* ---------------------------------------------------------------------------------------------
 * primitive-level entry points (tests/test_warp_emul.py compares the CUDA device routines, compiled
 * for the host, against these).  out: 7 reals per contact = dist, pos[3], normal[3].
 * ------------------------------------------------------------------------------------------- */
static int prim_out(const RawCon* c, int n, real* out) {
  for (int i = 0; i < n; i++) {
    out[7*i] = c[i].dist;
    for (int k = 0; k < 3; k++) { out[7*i+1+k] = c[i].pos[k]; out[7*i+4+k] = c[i].frame[k]; }
  }
  return n;
}
int b2o_prim_sphere_box(const real* sp, real r, const real* bp, const real* bm, const real* h, real margin, real* out) {
  RawCon c[1];
  return prim_out(c, sphere_box(c, margin, sp, r, bp, bm, h), out);
}
int b2o_prim_capsule_box(const real* cp, const real* cm, const real* cs, const real* bp, const real* bm, const real* h,
                         real margin, real* out) {
  RawCon c[2];
  return prim_out(c, capsule_box(c, margin, cp, cm, cs, bp, bm, h), out);
}
int b2o_prim_box_box(const real* p1, const real* m1, const real* h1, const real* p2, const real* m2, const real* h2,
                     real margin, real* out) {
  RawCon c[8];
  return prim_out(c, box_box(c, margin, p1, m1, h1, p2, m2, h2), out);
}
/* convex routines: shapes given as (MuJoCo geom type, pos, mat, size, verts, nvert) */
int b2o_prim_convex(int t1, const real* p1, const real* m1, const real* s1, const real* v1, int n1,
                    int t2, const real* p2, const real* m2, const real* s2, const real* v2, int n2,
                    real margin, real scale, real* out) {
  B2CShape A, B; B2CCon c[1];
  real r1 = b2c_shape(&A, t1, p1, m1, s1, v1, n1), r2 = b2c_shape(&B, t2, p2, m2, s2, v2, n2);
  int n = b2c_pair(c, margin, &A, r1, &B, r2, p1, p2, scale);
  RawCon rc[1];
  return prim_out(rc, from_b2c(rc, c, n), out);
}
int b2o_prim_plane_mesh(const real* pp, const real* pn, const real* p2, const real* m2, const real* v2, int n2,
                        real margin, real* out) {
  B2CShape B; B2CCon c[4]; real sz[3] = {0, 0, 0};
  b2c_shape(&B, G_MESH, p2, m2, sz, v2, n2);
  RawCon rc[4];
  return prim_out(rc, from_b2c(rc, c, b2c_plane_mesh(c, margin, pp, pn, &B)), out);
}
/* plane against a cylinder (t2 = 5, up to 4 contacts) or an ellipsoid (t2 = 4, one contact) */
int b2o_prim_plane_smooth(const real* pp, const real* pn, int t2, const real* p2, const real* m2, const real* s2,
                          real margin, real* out) {
  B2CShape B; B2CCon c[4];
  b2c_shape(&B, t2, p2, m2, s2, NULL, 0);
  RawCon rc[4];
  int n = t2 == G_CYLINDER ? b2c_plane_cylinder(c, margin, pp, pn, p2, m2, s2) : b2c_plane_ellipsoid(c, margin, pp, pn, &B);
  return prim_out(rc, from_b2c(rc, c, n), out);
}
int b2o_prim_hfield(const real* hp, const real* hm, const real* hsize, int nrow, int ncol, const real* hdata,
                    int t2, const real* p2, const real* m2, const real* s2, const real* v2, int n2, real rbound,
                    real margin, real* out) {
  B2CShape B; B2CCon c[B2C_MAXOUT];
  real r2 = b2c_shape(&B, t2, p2, m2, s2, v2, n2);
  RawCon rc[B2C_MAXOUT];
  return prim_out(rc, from_b2c(rc, c, b2c_hfield(c, margin, hp, hm, hsize, nrow, ncol, hdata, &B, r2, p2, rbound)), out);
}
