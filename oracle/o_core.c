/* TEST INFRASTRUCTURE - CPU oracle, smooth dynamics (kinematics, CRB mass matrix, RNE bias, passive + fluid forces,
 * actuation, Euler integration).  Restates the stages listed in SURVEY.md section 8 rows a1/a7 for the calls
 * `robosuite/utils/binding_utils.py:1101-1107`.  Physics parity is unpinned (see b2s_oracle.h). */
#include "b2s_oracle.h"
#include "o_math.h"
#include <stdio.h>
#include <stdlib.h>

/* ------------------------------------------------------------------------------------------------ blob reader */
typedef struct {
  char name[48];
  int32_t dtype, ndim, shape[4];
  int64_t off, nbytes;
} BlobRec;

static const BlobRec* blob_find(const void* blob, const char* name) {
  const char* p = (const char*)blob;
  int64_t n;
  memcpy(&n, p + 8, 8);
  const BlobRec* r = (const BlobRec*)(p + 16);
  for (int64_t i = 0; i < n; i++)
    if (strcmp(r[i].name, name) == 0) return r + i;
  return NULL;
}
static const double* blob_f64(const void* blob, const char* name) {
  const BlobRec* r = blob_find(blob, name);
  if (!r || r->dtype != 0) { fprintf(stderr, "oracle: missing f64 field %s\n", name); abort(); }
  return (const double*)((const char*)blob + r->off);
}
static const int* blob_i32(const void* blob, const char* name) {
  const BlobRec* r = blob_find(blob, name);
  if (!r || r->dtype != 1) { fprintf(stderr, "oracle: missing i32 field %s\n", name); abort(); }
  return (const int*)((const char*)blob + r->off);
}

OModel* o_model_load(const void* blob_in, size_t nbytes) {
  if (nbytes < 16 || memcmp(blob_in, "B2SMODEL", 8) != 0) return NULL;
  OModel* m = (OModel*)calloc(1, sizeof(OModel));
  m->blob = malloc(nbytes);
  memcpy(m->blob, blob_in, nbytes);
  const void* b = m->blob;
#define I(name) m->name = blob_i32(b, #name)[0]
#define PI(name) m->name = blob_i32(b, #name)
#define PF(name) m->name = blob_f64(b, #name)
  I(nq); I(nv); I(nu); I(nbody); I(njnt); I(ngeom); I(nsite); I(nmesh); I(nM); I(npair); I(nmocap); I(nsensordata);
  I(nmeshvert);
  m->timestep = blob_f64(b, "opt_timestep")[0];
  m->impratio = blob_f64(b, "opt_impratio")[0];
  m->density = blob_f64(b, "opt_density")[0];
  m->viscosity = blob_f64(b, "opt_viscosity")[0];
  m->tolerance = blob_f64(b, "opt_tolerance")[0];
  m->ls_tolerance = blob_f64(b, "opt_ls_tolerance")[0];
  m->meaninertia = blob_f64(b, "stat_meaninertia")[0];
  m->iterations = blob_i32(b, "opt_iterations")[0];
  m->ls_iterations = blob_i32(b, "opt_ls_iterations")[0];
  m->cone = blob_i32(b, "opt_cone")[0];
  m->gravity = blob_f64(b, "opt_gravity");
  m->wind = blob_f64(b, "opt_wind");
  PI(body_parentid); PI(body_rootid); PI(body_weldid); PI(body_mocapid); PI(body_jntnum); PI(body_jntadr);
  PI(body_dofnum); PI(body_dofadr); PI(body_geomnum); PI(body_geomadr);
  PF(body_pos); PF(body_quat); PF(body_ipos); PF(body_iquat); PF(body_mass); PF(body_subtreemass); PF(body_inertia);
  PF(body_invweight0);
  PI(jnt_type); PI(jnt_qposadr); PI(jnt_dofadr); PI(jnt_bodyid); PI(jnt_limited);
  PF(jnt_pos); PF(jnt_axis); PF(jnt_range); PF(jnt_margin); PF(jnt_solref); PF(jnt_solimp); PF(jnt_stiffness);
  PI(dof_bodyid); PI(dof_jntid); PI(dof_parentid); PI(dof_Madr);
  PF(dof_armature); PF(dof_damping); PF(dof_frictionloss); PF(dof_solref); PF(dof_solimp); PF(dof_invweight0);
  PF(dof_M0); PF(qpos0); PF(qpos_spring);
  PI(geom_type); PI(geom_contype); PI(geom_conaffinity); PI(geom_condim); PI(geom_bodyid); PI(geom_dataid);
  PI(geom_priority);
  PF(geom_size); PF(geom_pos); PF(geom_quat); PF(geom_friction); PF(geom_solmix); PF(geom_solref); PF(geom_solimp);
  PF(geom_margin); PF(geom_gap); PF(geom_rbound); PF(geom_aabb);
  PI(pair_geom); PI(mesh_vertadr); PI(mesh_vertnum); PF(mesh_vert);
  PI(site_bodyid); PF(site_pos); PF(site_quat);
  PI(actuator_trnid); PI(actuator_ctrllimited); PI(actuator_forcelimited); PI(actuator_biastype);
  PF(actuator_ctrlrange); PF(actuator_forcerange); PF(actuator_gear); PF(actuator_gainprm); PF(actuator_biasprm);
#undef I
#undef PI
#undef PF
  return m;
}

void o_model_free(OModel* m) {
  if (!m) return;
  free(m->blob);
  free(m);
}

static double* zalloc(size_t n) { return (double*)calloc(n ? n : 1, sizeof(double)); }

OData* o_data_new(const OModel* m) {
  OData* d = (OData*)calloc(1, sizeof(OData));
  int nq = m->nq, nv = m->nv, nb = m->nbody;
  d->qpos = zalloc(nq); d->qvel = zalloc(nv); d->qacc = zalloc(nv); d->qacc_warmstart = zalloc(nv);
  d->ctrl = zalloc(m->nu); d->qfrc_applied = zalloc(nv);
  d->mocap_pos = zalloc(3 * m->nmocap); d->mocap_quat = zalloc(4 * m->nmocap);
  d->xpos = zalloc(3 * nb); d->xquat = zalloc(4 * nb); d->xmat = zalloc(9 * nb); d->xipos = zalloc(3 * nb);
  d->ximat = zalloc(9 * nb); d->xanchor = zalloc(3 * m->njnt); d->xaxis = zalloc(3 * m->njnt);
  d->geom_xpos = zalloc(3 * m->ngeom); d->geom_xmat = zalloc(9 * m->ngeom);
  d->site_xpos = zalloc(3 * m->nsite); d->site_xmat = zalloc(9 * m->nsite);
  d->cdof = zalloc(6 * nv); d->cinert = zalloc(10 * nb); d->crb = zalloc(10 * nb);
  d->qM = zalloc(m->nM); d->M = zalloc((size_t)nv * nv); d->L = zalloc((size_t)nv * nv);
  d->cvel = zalloc(6 * nb); d->cdof_dot = zalloc(6 * nv);
  d->qfrc_bias = zalloc(nv); d->qfrc_passive = zalloc(nv); d->qfrc_actuator = zalloc(nv);
  d->actuator_force = zalloc(m->nu); d->qfrc_smooth = zalloc(nv); d->qacc_smooth = zalloc(nv);
  d->qfrc_constraint = zalloc(nv); d->sensordata = zalloc(m->nsensordata);
  d->efc_J = zalloc((size_t)O_MAXEFC * nv);
  o_reset_data(m, d);
  return d;
}

void o_data_free(OData* d) {
  if (!d) return;
  double* ptrs[] = {d->qpos, d->qvel, d->qacc, d->qacc_warmstart, d->ctrl, d->qfrc_applied, d->mocap_pos,
                    d->mocap_quat, d->xpos, d->xquat, d->xmat, d->xipos, d->ximat, d->xanchor, d->xaxis, d->geom_xpos,
                    d->geom_xmat, d->site_xpos, d->site_xmat, d->cdof, d->cinert, d->crb, d->qM, d->M, d->L, d->cvel,
                    d->cdof_dot, d->qfrc_bias, d->qfrc_passive, d->qfrc_actuator, d->actuator_force, d->qfrc_smooth,
                    d->qacc_smooth, d->qfrc_constraint, d->sensordata, d->efc_J};
  for (size_t i = 0; i < sizeof(ptrs) / sizeof(ptrs[0]); i++) free(ptrs[i]);
  free(d);
}

double* o_data_field(OData* d, const char* name) {
#define F(n) if (strcmp(name, #n) == 0) return d->n
  F(qpos); F(qvel); F(qacc); F(qacc_warmstart); F(ctrl); F(qfrc_applied); F(mocap_pos); F(mocap_quat); F(xpos);
  F(xquat); F(xmat); F(xipos); F(ximat); F(xanchor); F(xaxis); F(geom_xpos); F(geom_xmat); F(site_xpos); F(site_xmat);
  F(cdof); F(cinert); F(crb); F(qM); F(M); F(L); F(cvel); F(cdof_dot); F(qfrc_bias); F(qfrc_passive);
  F(qfrc_actuator); F(actuator_force); F(qfrc_smooth); F(qacc_smooth); F(qfrc_constraint); F(sensordata); F(efc_J);
  F(efc_pos); F(efc_D); F(efc_R); F(efc_aref); F(efc_vel); F(efc_force); F(efc_frictionloss); F(efc_diagApprox);
  F(efc_margin);
#undef F
  if (strcmp(name, "time") == 0) return &d->time;
  return NULL;
}

void o_reset_data(const OModel* m, OData* d) {
  d->time = 0;
  memcpy(d->qpos, m->qpos0, sizeof(double) * m->nq);
  memset(d->qvel, 0, sizeof(double) * m->nv);
  memset(d->qacc, 0, sizeof(double) * m->nv);
  memset(d->qacc_warmstart, 0, sizeof(double) * m->nv);
  memset(d->qfrc_applied, 0, sizeof(double) * m->nv);
  memset(d->ctrl, 0, sizeof(double) * m->nu);
  for (int b = 0; b < m->nbody; b++)
    if (m->body_mocapid[b] >= 0) {
      memcpy(d->mocap_pos + 3 * m->body_mocapid[b], m->body_pos + 3 * b, 3 * sizeof(double));
      memcpy(d->mocap_quat + 4 * m->body_mocapid[b], m->body_quat + 4 * b, 4 * sizeof(double));
    }
  d->ncon = 0; d->nefc = 0; d->nf = 0; d->nl = 0;
  d->warn_flags = 0;
}

/* ------------------------------------------------------------------------------------------------ kinematics */
/* mj_checkPos / mj_checkVel / mj_checkAcc of the engine (first calls of mj_step, and after the solve): a non-finite or huge
 * coordinate resets the data to the model defaults (warn bit 32) instead of integrating garbage */
static int vec_bad(const double* x, int n) {
  for (int i = 0; i < n; i++) if (!(fabs(x[i]) <= 1e10)) return 1;
  return 0;
}
static void reset_defaults(const OModel* m, OData* d) {
  memcpy(d->qpos, m->qpos0, sizeof(double) * m->nq);
  for (int i = 0; i < m->nv; i++) { d->qvel[i] = 0; d->qacc[i] = 0; d->qacc_warmstart[i] = 0; }
  d->time = 0;
  d->warn_flags |= 32;
}

void o_kinematics(const OModel* m, OData* d) {
  if (vec_bad(d->qpos, m->nq) || vec_bad(d->qvel, m->nv)) reset_defaults(m, d);
  /* world body */
  v3_set(d->xpos, 0, 0, 0);
  d->xquat[0] = 1; d->xquat[1] = d->xquat[2] = d->xquat[3] = 0;
  quat2mat(d->xmat, d->xquat);
  v3_set(d->xipos, 0, 0, 0);
  quat2mat(d->ximat, d->xquat);
  for (int b = 1; b < m->nbody; b++) {
    double pos[3], quat[4], R[9];
    int p = m->body_parentid[b];
    if (m->body_mocapid[b] >= 0) {
      v3_copy(pos, d->mocap_pos + 3 * m->body_mocapid[b]);
      memcpy(quat, d->mocap_quat + 4 * m->body_mocapid[b], sizeof quat);
      quat_normalize(quat);
    } else {
      m3_mulv(pos, d->xmat + 9 * p, m->body_pos + 3 * b);
      v3_add(pos, pos, d->xpos + 3 * p);
      quat_mul(quat, d->xquat + 4 * p, m->body_quat + 4 * b);
    }
    for (int k = 0; k < m->body_jntnum[b]; k++) {
      int j = m->body_jntadr[b] + k, qa = m->jnt_qposadr[j], t = m->jnt_type[j];
      double* anchor = d->xanchor + 3 * j;
      double* axis = d->xaxis + 3 * j;
      if (t == O_JNT_FREE) {
        v3_copy(pos, d->qpos + qa);
        memcpy(quat, d->qpos + qa + 3, sizeof quat);
        quat_normalize(quat);
        v3_copy(anchor, pos);
        v3_set(axis, 0, 0, 1);
        continue;
      }
      quat2mat(R, quat);
      m3_mulv(anchor, R, m->jnt_pos + 3 * j);
      v3_add(anchor, anchor, pos);
      m3_mulv(axis, R, m->jnt_axis + 3 * j);
      if (t == O_JNT_SLIDE) {
        v3_addscl(pos, pos, axis, d->qpos[qa] - m->qpos0[qa]);
      } else {
        double ql[4], tmp[4], off[3];
        if (t == O_JNT_HINGE) axisangle2quat(ql, m->jnt_axis + 3 * j, d->qpos[qa] - m->qpos0[qa]);
        else { memcpy(ql, d->qpos + qa, sizeof ql); quat_normalize(ql); }
        quat_mul(tmp, quat, ql);
        memcpy(quat, tmp, sizeof quat);
        quat2mat(R, quat);
        m3_mulv(off, R, m->jnt_pos + 3 * j);
        v3_sub(pos, anchor, off);
      }
    }
    quat_normalize(quat);
    v3_copy(d->xpos + 3 * b, pos);
    memcpy(d->xquat + 4 * b, quat, sizeof quat);
    quat2mat(d->xmat + 9 * b, quat);
    m3_mulv(d->xipos + 3 * b, d->xmat + 9 * b, m->body_ipos + 3 * b);
    v3_add(d->xipos + 3 * b, d->xipos + 3 * b, pos);
    double qi[4];
    quat_mul(qi, quat, m->body_iquat + 4 * b);
    quat2mat(d->ximat + 9 * b, qi);
  }
  for (int g = 0; g < m->ngeom; g++) {
    int b = m->geom_bodyid[g];
    double q[4];
    m3_mulv(d->geom_xpos + 3 * g, d->xmat + 9 * b, m->geom_pos + 3 * g);
    v3_add(d->geom_xpos + 3 * g, d->geom_xpos + 3 * g, d->xpos + 3 * b);
    quat_mul(q, d->xquat + 4 * b, m->geom_quat + 4 * g);
    quat2mat(d->geom_xmat + 9 * g, q);
  }
  for (int s = 0; s < m->nsite; s++) {
    int b = m->site_bodyid[s];
    double q[4];
    m3_mulv(d->site_xpos + 3 * s, d->xmat + 9 * b, m->site_pos + 3 * s);
    v3_add(d->site_xpos + 3 * s, d->site_xpos + 3 * s, d->xpos + 3 * b);
    quat_mul(q, d->xquat + 4 * b, m->site_quat + 4 * s);
    quat2mat(d->site_xmat + 9 * s, q);
  }
  /* spatial motion axis of every dof about the world origin: [w; p x w] (revolute through p), [0; a] (prismatic) */
  for (int i = 0; i < m->nv; i++) {
    int j = m->dof_jntid[i], t = m->jnt_type[j], k = i - m->jnt_dofadr[j], b = m->jnt_bodyid[j];
    double* c = d->cdof + 6 * i;
    if (t == O_JNT_FREE && k < 3) {
      v3_set(c, 0, 0, 0); v3_set(c + 3, 0, 0, 0); c[3 + k] = 1;
    } else if (t == O_JNT_FREE || t == O_JNT_BALL) {
      int col = t == O_JNT_FREE ? k - 3 : k;
      const double* R = d->xmat + 9 * b;
      v3_set(c, R[col], R[3 + col], R[6 + col]);
      v3_cross(c + 3, t == O_JNT_FREE ? d->xpos + 3 * b : d->xanchor + 3 * j, c);
    } else if (t == O_JNT_SLIDE) {
      v3_set(c, 0, 0, 0); v3_copy(c + 3, d->xaxis + 3 * j);
    } else {
      v3_copy(c, d->xaxis + 3 * j);
      v3_cross(c + 3, d->xanchor + 3 * j, c);
    }
  }
  /* spatial inertia of each body about the world origin */
  for (int b = 0; b < m->nbody; b++) {
    double* ci = d->cinert + 10 * b;
    const double* Ri = d->ximat + 9 * b;
    const double* I = m->body_inertia + 3 * b;
    const double* c = d->xipos + 3 * b;
    double mass = m->body_mass[b];
    double Iw[9];
    for (int r = 0; r < 3; r++)
      for (int s = 0; s < 3; s++) Iw[3 * r + s] = Ri[3 * r] * I[0] * Ri[3 * s] + Ri[3 * r + 1] * I[1] * Ri[3 * s + 1] + Ri[3 * r + 2] * I[2] * Ri[3 * s + 2];
    double cc = v3_dot(c, c);
    ci[0] = Iw[0] + mass * (cc - c[0] * c[0]);
    ci[1] = Iw[4] + mass * (cc - c[1] * c[1]);
    ci[2] = Iw[8] + mass * (cc - c[2] * c[2]);
    ci[3] = Iw[1] - mass * c[0] * c[1];
    ci[4] = Iw[2] - mass * c[0] * c[2];
    ci[5] = Iw[5] - mass * c[1] * c[2];
    ci[6] = mass * c[0]; ci[7] = mass * c[1]; ci[8] = mass * c[2];
    ci[9] = mass;
  }
}

/* f = I * v for the 10-number spatial inertia; v = [w; vO], f = [torque about O; force] */
static void inert_mulv(double* f, const double* I, const double* v) {
  const double *w = v, *l = v + 3, *h = I + 6;
  double t[3];
  f[0] = I[0] * w[0] + I[3] * w[1] + I[4] * w[2];
  f[1] = I[3] * w[0] + I[1] * w[1] + I[5] * w[2];
  f[2] = I[4] * w[0] + I[5] * w[1] + I[2] * w[2];
  v3_cross(t, h, l);
  v3_add(f, f, t);
  v3_cross(t, w, h);
  f[3] = I[9] * l[0] + t[0]; f[4] = I[9] * l[1] + t[1]; f[5] = I[9] * l[2] + t[2];
}
static double dot6(const double* a, const double* b) {
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5];
}
/* motion cross product r = v x s */
static void cross_motion(double* r, const double* v, const double* s) {
  double a[3], b[3];
  v3_cross(r, v, s);
  v3_cross(a, v, s + 3);
  v3_cross(b, v + 3, s);
  v3_add(r + 3, a, b);
}
/* force cross product r = v x* f */
static void cross_force(double* r, const double* v, const double* f) {
  double a[3], b[3];
  v3_cross(a, v, f);
  v3_cross(b, v + 3, f + 3);
  v3_add(r, a, b);
  v3_cross(r + 3, v, f + 3);
}

/* ------------------------------------------------------------------------------------------------ CRB -> M */
void o_crb(const OModel* m, OData* d) {
  int nv = m->nv;
  memcpy(d->crb, d->cinert, sizeof(double) * 10 * m->nbody);
  for (int b = m->nbody - 1; b > 0; b--) {
    int p = m->body_parentid[b];
    for (int k = 0; k < 10; k++) d->crb[10 * p + k] += d->crb[10 * b + k];
  }
  memset(d->M, 0, sizeof(double) * nv * nv);
  for (int i = 0; i < nv; i++) {
    double f[6];
    inert_mulv(f, d->crb + 10 * m->dof_bodyid[i], d->cdof + 6 * i);
    int adr = m->dof_Madr[i];
    for (int j = i; j >= 0; j = m->dof_parentid[j]) {
      double v = dot6(d->cdof + 6 * j, f);
      if (j == i) v += m->dof_armature[i];
      d->M[i * nv + j] = d->M[j * nv + i] = v;
      d->qM[adr++] = v;
    }
  }
}

void o_full_m(const OModel* m, const OData* d, double* dst) { memcpy(dst, d->M, sizeof(double) * m->nv * m->nv); }

/* dense Cholesky M = L L^T (lower) */
static int chol(double* L, const double* A, int n) {
  memcpy(L, A, sizeof(double) * n * n);
  for (int j = 0; j < n; j++) {
    double s = L[j * n + j];
    for (int k = 0; k < j; k++) s -= L[j * n + k] * L[j * n + k];
    if (s < 1e-300) return -1;
    s = sqrt(s);
    L[j * n + j] = s;
    for (int i = j + 1; i < n; i++) {
      double t = L[i * n + j];
      for (int k = 0; k < j; k++) t -= L[i * n + k] * L[j * n + k];
      L[i * n + j] = t / s;
    }
    for (int i = 0; i < j; i++) L[i * n + j] = 0;
  }
  return 0;
}
static void chol_solve(const double* L, double* x, int n) {
  for (int i = 0; i < n; i++) {
    double s = x[i];
    for (int k = 0; k < i; k++) s -= L[i * n + k] * x[k];
    x[i] = s / L[i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    double s = x[i];
    for (int k = i + 1; k < n; k++) s -= L[k * n + i] * x[k];
    x[i] = s / L[i * n + i];
  }
}
int o_chol(double* L, const double* A, int n) { return chol(L, A, n); }
void o_chol_solve(const double* L, double* x, int n) { chol_solve(L, x, n); }

void o_factor_m(const OModel* m, OData* d) {
  if (chol(d->L, d->M, m->nv) != 0) d->warn_flags |= 1;
}
void o_solve_m(const OModel* m, const OData* d, double* x, int n) {
  for (int r = 0; r < n; r++) chol_solve(d->L, x + (size_t)r * m->nv, m->nv);
}

/* ------------------------------------------------------------------------------------------------ Jacobian */
void o_jac(const OModel* m, const OData* d, double* jacp, double* jacr, const double point[3], int body) {
  int nv = m->nv;
  if (jacp) memset(jacp, 0, sizeof(double) * 3 * nv);
  if (jacr) memset(jacr, 0, sizeof(double) * 3 * nv);
  while (body > 0 && m->body_dofnum[body] == 0) body = m->body_parentid[body];
  if (body == 0) return;
  for (int i = m->body_dofadr[body] + m->body_dofnum[body] - 1; i >= 0; i = m->dof_parentid[i]) {
    const double* c = d->cdof + 6 * i;
    if (jacr) { jacr[i] = c[0]; jacr[nv + i] = c[1]; jacr[2 * nv + i] = c[2]; }
    if (jacp) {
      double t[3];
      v3_cross(t, c, point);
      jacp[i] = c[3] + t[0]; jacp[nv + i] = c[4] + t[1]; jacp[2 * nv + i] = c[5] + t[2];
    }
  }
}

/* ------------------------------------------------------------------------------------------------ velocity */
void o_com_vel(const OModel* m, OData* d) {
  memset(d->cvel, 0, sizeof(double) * 6);
  for (int b = 1; b < m->nbody; b++) {
    double v[6];
    memcpy(v, d->cvel + 6 * m->body_parentid[b], sizeof v);
    for (int k = 0; k < m->body_jntnum[b]; k++) {
      int j = m->body_jntadr[b] + k, da = m->jnt_dofadr[j], t = m->jnt_type[j];
      if (t == O_JNT_FREE) {
        /* translational axes are world-fixed: zero derivative; add their velocity first */
        memset(d->cdof_dot + 6 * da, 0, sizeof(double) * 18);
        for (int c = 0; c < 3; c++)
          for (int e = 0; e < 6; e++) v[e] += d->cdof[6 * (da + c) + e] * d->qvel[da + c];
        da += 3;
      }
      if (t == O_JNT_FREE || t == O_JNT_BALL) {
        for (int c = 0; c < 3; c++) cross_motion(d->cdof_dot + 6 * (da + c), v, d->cdof + 6 * (da + c));
        for (int c = 0; c < 3; c++)
          for (int e = 0; e < 6; e++) v[e] += d->cdof[6 * (da + c) + e] * d->qvel[da + c];
      } else {
        cross_motion(d->cdof_dot + 6 * da, v, d->cdof + 6 * da);
        for (int e = 0; e < 6; e++) v[e] += d->cdof[6 * da + e] * d->qvel[da];
      }
    }
    memcpy(d->cvel + 6 * b, v, sizeof v);
  }
}

void o_rne_bias(const OModel* m, OData* d) {
  int nb = m->nbody;
  double* acc = (double*)calloc(6 * nb, sizeof(double));
  double* frc = (double*)calloc(6 * nb, sizeof(double));
  acc[3] = -m->gravity[0]; acc[4] = -m->gravity[1]; acc[5] = -m->gravity[2];
  for (int b = 1; b < nb; b++) {
    double* a = acc + 6 * b;
    memcpy(a, acc + 6 * m->body_parentid[b], 6 * sizeof(double));
    for (int i = m->body_dofadr[b]; i < m->body_dofadr[b] + m->body_dofnum[b]; i++)
      for (int e = 0; e < 6; e++) a[e] += d->cdof_dot[6 * i + e] * d->qvel[i];
    double Iv[6], Ia[6], vxIv[6];
    inert_mulv(Ia, d->cinert + 10 * b, a);
    inert_mulv(Iv, d->cinert + 10 * b, d->cvel + 6 * b);
    cross_force(vxIv, d->cvel + 6 * b, Iv);
    for (int e = 0; e < 6; e++) frc[6 * b + e] = Ia[e] + vxIv[e];
  }
  for (int b = nb - 1; b > 0; b--)
    for (int e = 0; e < 6; e++) frc[6 * m->body_parentid[b] + e] += frc[6 * b + e];
  for (int i = 0; i < m->nv; i++) d->qfrc_bias[i] = dot6(d->cdof + 6 * i, frc + 6 * m->dof_bodyid[i]);
  free(acc);
  free(frc);
}

/* ------------------------------------------------------------------------------------------------ passive */
void o_passive(const OModel* m, OData* d) {
  int nv = m->nv;
  for (int i = 0; i < nv; i++) d->qfrc_passive[i] = -m->dof_damping[i] * d->qvel[i];
  /* joint springs on slide and hinge joints, about the spring reference (springref), not the joint's zero (ref) */
  for (int j = 0; j < m->njnt; j++)
    if (m->jnt_stiffness[j] != 0 && (m->jnt_type[j] == O_JNT_SLIDE || m->jnt_type[j] == O_JNT_HINGE))
      d->qfrc_passive[m->jnt_dofadr[j]] -= m->jnt_stiffness[j] * (d->qpos[m->jnt_qposadr[j]] - m->qpos_spring[m->jnt_qposadr[j]]);
  if (m->density <= 0 && m->viscosity <= 0) return;
  /* fluid forces, inertia-box model (option density / viscosity are non-zero in models/assets/base.xml:3-5) */
  double* jp = (double*)malloc(sizeof(double) * 3 * nv);
  double* jr = (double*)malloc(sizeof(double) * 3 * nv);
  for (int b = 1; b < m->nbody; b++) {
    double mass = m->body_mass[b];
    if (mass < O_MINVAL) continue;
    const double* I = m->body_inertia + 3 * b;
    double box[3];
    box[0] = sqrt(fmax(O_MINVAL, (I[1] + I[2] - I[0])) / mass * 6.0);
    box[1] = sqrt(fmax(O_MINVAL, (I[0] + I[2] - I[1])) / mass * 6.0);
    box[2] = sqrt(fmax(O_MINVAL, (I[0] + I[1] - I[2])) / mass * 6.0);
    /* 6D velocity at the inertial frame origin, in inertial-frame axes */
    const double* cv = d->cvel + 6 * b;
    double lin[3], t[3], lvel[6], lfrc[6] = {0, 0, 0, 0, 0, 0};
    v3_cross(t, cv, d->xipos + 3 * b);
    v3_add(lin, cv + 3, t);
    v3_sub(lin, lin, m->wind);
    m3_mulTv(lvel, d->ximat + 9 * b, cv);
    m3_mulTv(lvel + 3, d->ximat + 9 * b, lin);
    if (m->viscosity > 0) {
      double diam = (box[0] + box[1] + box[2]) / 3.0;
      double kr = -M_PI * diam * diam * diam * m->viscosity, kl = -3.0 * M_PI * diam * m->viscosity;
      for (int k = 0; k < 3; k++) { lfrc[k] = kr * lvel[k]; lfrc[3 + k] = kl * lvel[3 + k]; }
    }
    if (m->density > 0) {
      double rho = m->density;
      lfrc[3] -= 0.5 * rho * box[1] * box[2] * fabs(lvel[3]) * lvel[3];
      lfrc[4] -= 0.5 * rho * box[0] * box[2] * fabs(lvel[4]) * lvel[4];
      lfrc[5] -= 0.5 * rho * box[0] * box[1] * fabs(lvel[5]) * lvel[5];
      lfrc[0] -= rho * box[0] * (pow(box[1], 4) + pow(box[2], 4)) * fabs(lvel[0]) * lvel[0] / 64.0;
      lfrc[1] -= rho * box[1] * (pow(box[0], 4) + pow(box[2], 4)) * fabs(lvel[1]) * lvel[1] / 64.0;
      lfrc[2] -= rho * box[2] * (pow(box[0], 4) + pow(box[1], 4)) * fabs(lvel[2]) * lvel[2] / 64.0;
    }
    double torque[3], force[3];
    m3_mulv(torque, d->ximat + 9 * b, lfrc);
    m3_mulv(force, d->ximat + 9 * b, lfrc + 3);
    o_jac(m, d, jp, jr, d->xipos + 3 * b, b);
    for (int i = 0; i < nv; i++)
      d->qfrc_passive[i] += jp[i] * force[0] + jp[nv + i] * force[1] + jp[2 * nv + i] * force[2] +
                            jr[i] * torque[0] + jr[nv + i] * torque[1] + jr[2 * nv + i] * torque[2];
  }
  free(jp);
  free(jr);
}

/* ------------------------------------------------------------------------------------------------ actuation */
void o_fwd_actuation(const OModel* m, OData* d) {
  memset(d->qfrc_actuator, 0, sizeof(double) * m->nv);
  for (int i = 0; i < m->nu; i++) {
    double ctrl = d->ctrl[i];
    if (m->actuator_ctrllimited[i]) ctrl = fmin(fmax(ctrl, m->actuator_ctrlrange[2 * i]), m->actuator_ctrlrange[2 * i + 1]);
    int j = m->actuator_trnid[i], qa = m->jnt_qposadr[j], da = m->jnt_dofadr[j];
    double gear = m->actuator_gear[6 * i];
    double length = d->qpos[qa] * gear, velocity = d->qvel[da] * gear;
    double f = m->actuator_gainprm[3 * i] * ctrl;
    if (m->actuator_biastype[i])
      f += m->actuator_biasprm[3 * i] + m->actuator_biasprm[3 * i + 1] * length + m->actuator_biasprm[3 * i + 2] * velocity;
    if (m->actuator_forcelimited[i]) f = fmin(fmax(f, m->actuator_forcerange[2 * i]), m->actuator_forcerange[2 * i + 1]);
    d->actuator_force[i] = f;
    d->qfrc_actuator[da] += gear * f;
  }
}

void o_fwd_acceleration(const OModel* m, OData* d) {
  for (int i = 0; i < m->nv; i++) {
    d->qfrc_smooth[i] = d->qfrc_passive[i] - d->qfrc_bias[i] + d->qfrc_applied[i] + d->qfrc_actuator[i];
    d->qacc_smooth[i] = d->qfrc_smooth[i];
  }
  chol_solve(d->L, d->qacc_smooth, m->nv);
}

/* ------------------------------------------------------------------------------------------------ integrator */
void o_euler(const OModel* m, OData* d) {
  int nv = m->nv;
  double h = m->timestep;
  if (vec_bad(d->qacc, nv)) { reset_defaults(m, d); return; }
  double* qacc = (double*)malloc(sizeof(double) * nv);
  int damped = 0;
  for (int i = 0; i < nv; i++) damped |= m->dof_damping[i] > 0;
  if (damped) {
    /* implicit-in-velocity joint damping: (M + h D) a = qfrc_smooth + qfrc_constraint */
    double* A = (double*)malloc(sizeof(double) * nv * nv);
    double* L = (double*)malloc(sizeof(double) * nv * nv);
    memcpy(A, d->M, sizeof(double) * nv * nv);
    for (int i = 0; i < nv; i++) {
      A[i * nv + i] += h * m->dof_damping[i];
      qacc[i] = d->qfrc_smooth[i] + d->qfrc_constraint[i];
    }
    if (chol(L, A, nv) != 0) d->warn_flags |= 2;
    chol_solve(L, qacc, nv);
    free(A);
    free(L);
  } else {
    memcpy(qacc, d->qacc, sizeof(double) * nv);
  }
  for (int i = 0; i < nv; i++) d->qvel[i] += h * qacc[i];
  for (int j = 0; j < m->njnt; j++) {
    int qa = m->jnt_qposadr[j], da = m->jnt_dofadr[j], t = m->jnt_type[j];
    if (t == O_JNT_FREE) {
      for (int k = 0; k < 3; k++) d->qpos[qa + k] += h * d->qvel[da + k];
      qa += 3; da += 3;
    }
    if (t == O_JNT_FREE || t == O_JNT_BALL) {
      double w[3] = {d->qvel[da], d->qvel[da + 1], d->qvel[da + 2]};
      double ang = v3_normalize(w) * h;
      double dq[4], r[4];
      axisangle2quat(dq, w, ang);
      quat_mul(r, d->qpos + qa, dq);
      quat_normalize(r);
      memcpy(d->qpos + qa, r, sizeof r);
    } else {
      d->qpos[qa] += h * d->qvel[da];
    }
  }
  memcpy(d->qacc_warmstart, d->qacc, sizeof(double) * nv);
  d->time += h;
  free(qacc);
}
