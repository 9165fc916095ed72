/* TEST INFRASTRUCTURE - CPU oracle, soft-constraint assembly (friction-loss dofs, joint limits, elliptic-cone
 * contacts) and the primal Newton solver with exact line search.  Restates SURVEY.md Appendix C for the engine call
 * behind `robosuite/utils/binding_utils.py:1101-1107`; the reference leaves <option> at defaults apart from
 * `impratio=20 cone=elliptic` (`robosuite/models/assets/base.xml:3-5`).  Parity unpinned (see b2s_oracle.h). */
#include "b2s_oracle.h"
#include "o_math.h"
#include <stdlib.h>

int o_chol(double* L, const double* A, int n);
void o_chol_solve(const double* L, double* x, int n);

#define MINIMP 0.0001
#define MAXIMP 0.9999

static double clampd(double x, double lo, double hi) { return x < lo ? lo : x > hi ? hi : x; }

static double impedance(const double* solimp, double pos, double margin) {
  double dmin = clampd(solimp[0], MINIMP, MAXIMP), dmax = clampd(solimp[1], MINIMP, MAXIMP);
  double width = fmax(0.0, solimp[2]), mid = clampd(solimp[3], MINIMP, MAXIMP), power = fmax(1.0, solimp[4]);
  if (dmin == dmax || width <= O_MINVAL) return 0.5 * (dmin + dmax);
  double x = fabs(pos - margin) / width;
  if (x >= 1) return dmax;
  if (x <= 0) return dmin;
  double y;
  if (power == 1) y = x;
  else if (x <= mid) y = pow(x, power) / pow(mid, power - 1);
  else y = 1 - pow(1 - x, power) / pow(1 - mid, power - 1);
  return dmin + y * (dmax - dmin);
}

static int add_row(OData* d, int nv, int type, int id, double pos, double margin, double frictionloss) {
  int i = d->nefc;
  if (i >= O_MAXEFC) { d->warn_flags |= 8; return -1; }
  memset(d->efc_J + (size_t)i * nv, 0, sizeof(double) * nv);
  d->efc_type[i] = type;
  d->efc_id[i] = id;
  d->efc_pos[i] = pos;
  d->efc_margin[i] = margin;
  d->efc_frictionloss[i] = frictionloss;
  d->nefc++;
  return i;
}

void o_make_constraint(const OModel* m, OData* d) {
  int nv = m->nv;
  d->nefc = d->nf = d->nl = 0;
  /* --- friction-loss dofs */
  for (int i = 0; i < nv; i++)
    if (m->dof_frictionloss[i] > 0) {
      int r = add_row(d, nv, O_CNSTR_FRICTION_DOF, i, 0, 0, m->dof_frictionloss[i]);
      if (r < 0) break;
      d->efc_J[(size_t)r * nv + i] = 1;
      d->nf++;
    }
  /* --- joint limits (slide / hinge): a side is active within the joint's margin (both sides when the range is narrower than
   * twice the margin) */
  for (int j = 0; j < m->njnt; j++) {
    if (!m->jnt_limited[j]) continue;
    int t = m->jnt_type[j];
    if (t != O_JNT_SLIDE && t != O_JNT_HINGE) continue;
    double value = d->qpos[m->jnt_qposadr[j]], margin = m->jnt_margin[j];
    for (int side = -1; side <= 1; side += 2) {
      double dist = side * (m->jnt_range[2 * j + (side + 1) / 2] - value);
      if (dist < margin) {
        int r = add_row(d, nv, O_CNSTR_LIMIT_JOINT, j, dist, margin, 0);
        if (r < 0) break;
        d->efc_J[(size_t)r * nv + m->jnt_dofadr[j]] = -side;
        d->nl++;
      }
    }
  }
  /* --- contacts */
  double* jp1 = (double*)malloc(sizeof(double) * 12 * nv);
  double *jr1 = jp1 + 3 * nv, *jp2 = jp1 + 6 * nv, *jr2 = jp1 + 9 * nv;
  for (int c = 0; c < d->ncon; c++) {
    OContact* con = d->contact + c;
    con->efc_address = -1;
    if (con->dist >= 0) continue; /* includemargin = 0 */
    int b1 = m->geom_bodyid[con->geom1], b2 = m->geom_bodyid[con->geom2];
    o_jac(m, d, jp1, jr1, con->pos, b1);
    o_jac(m, d, jp2, jr2, con->pos, b2);
    int dim = con->dim;
    int type = dim == 1 ? O_CNSTR_CONTACT_FRICTIONLESS : O_CNSTR_CONTACT_ELLIPTIC;
    if (d->nefc + dim > O_MAXEFC) { d->warn_flags |= 8; break; } /* a contact enters with all of its rows or not at all */
    for (int k = 0; k < dim; k++) {
      int r = add_row(d, nv, type, c, k == 0 ? con->dist : 0.0, 0, 0);
      if (r < 0) break;
      if (k == 0) con->efc_address = r;
      const double* ax = con->frame + 3 * (k < 3 ? k : k - 3);
      const double *a = k < 3 ? jp1 : jr1, *b = k < 3 ? jp2 : jr2;
      for (int i = 0; i < nv; i++)
        d->efc_J[(size_t)r * nv + i] = ax[0] * (b[i] - a[i]) + ax[1] * (b[nv + i] - a[nv + i]) + ax[2] * (b[2 * nv + i] - a[2 * nv + i]);
    }
  }
  free(jp1);
  /* --- efc_vel, diagApprox, impedance, R/D, aref */
  for (int i = 0; i < d->nefc; i++) {
    double v = 0;
    for (int k = 0; k < nv; k++) v += d->efc_J[(size_t)i * nv + k] * d->qvel[k];
    d->efc_vel[i] = v;
  }
  for (int i = 0; i < d->nefc; i++) {
    int type = d->efc_type[i], id = d->efc_id[i];
    const double *solref, *solimp;
    int first = 1; /* first row of its constraint */
    double diag;
    if (type == O_CNSTR_FRICTION_DOF) {
      solref = m->dof_solref + 2 * id; solimp = m->dof_solimp + 5 * id; diag = m->dof_invweight0[id];
    } else if (type == O_CNSTR_LIMIT_JOINT) {
      solref = m->jnt_solref + 2 * id; solimp = m->jnt_solimp + 5 * id; diag = m->dof_invweight0[m->jnt_dofadr[id]];
    } else {
      const OContact* con = d->contact + id;
      int k = i - con->efc_address;
      first = k == 0;
      solref = con->solref; solimp = con->solimp;
      int b1 = m->geom_bodyid[con->geom1], b2 = m->geom_bodyid[con->geom2];
      diag = k < 3 ? m->body_invweight0[2 * b1] + m->body_invweight0[2 * b2]
                   : m->body_invweight0[2 * b1 + 1] + m->body_invweight0[2 * b2 + 1];
    }
    d->efc_diagApprox[i] = diag;
    double pos = d->efc_pos[i], margin = d->efc_margin[i];
    double imp = first ? impedance(solimp, pos, margin) : d->efc_KBIP[4 * (i - 1) + 2];
    double dmax = clampd(solimp[1], MINIMP, MAXIMP);
    double K, B;
    if (solref[0] > 0) {
      double tc = fmax(solref[0], 2 * m->timestep), dr = solref[1];
      K = 1.0 / fmax(O_MINVAL, dmax * dmax * tc * tc * dr * dr);
      B = 2.0 / fmax(O_MINVAL, dmax * tc);
    } else {
      K = -solref[0] / fmax(O_MINVAL, dmax * dmax);
      B = -solref[1] / fmax(O_MINVAL, dmax);
    }
    if (type == O_CNSTR_FRICTION_DOF || (type == O_CNSTR_CONTACT_ELLIPTIC && !first)) K = 0;
    d->efc_KBIP[4 * i] = K; d->efc_KBIP[4 * i + 1] = B; d->efc_KBIP[4 * i + 2] = imp; d->efc_KBIP[4 * i + 3] = 0;
    d->efc_R[i] = fmax(O_MINVAL, (1 - imp) * diag / imp);
    d->efc_aref[i] = -B * d->efc_vel[i] - K * imp * (pos - margin);
  }
  /* elliptic cones: friction-row regularisation tied to the normal row through impratio; cone friction `mu` */
  for (int c = 0; c < d->ncon; c++) {
    OContact* con = d->contact + c;
    if (con->efc_address < 0 || con->dim < 3) continue;
    double* R = d->efc_R + con->efc_address;
    R[1] = R[0] / fmax(O_MINVAL, m->impratio);
    for (int k = 2; k < con->dim; k++)
      R[k] = R[1] * con->friction[0] * con->friction[0] / (con->friction[k - 1] * con->friction[k - 1]);
    con->mu = con->friction[0] * sqrt(R[1] / R[0]);
  }
  for (int i = 0; i < d->nefc; i++) d->efc_D[i] = 1.0 / d->efc_R[i];
}

/* ------------------------------------------------------------------------------------------------ primal solver */
typedef struct {
  const OModel* m;
  OData* d;
  int nv, nefc;
  double *jar, *Ma, *grad, *search, *Mv, *jv, *H, *L;
  double cost;
} Ctx;

/* per-constraint cost, force and state at jar; optionally accumulate the Hessian J^T (d2s) J into H */
static double update_constraint(Ctx* c, const double* jar, double* force, int* state, double* H) {
  OData* d = c->d;
  int nv = c->nv;
  double cost = 0;
  for (int i = 0; i < c->nefc; i++) {
    int type = d->efc_type[i];
    double D = d->efc_D[i], R = d->efc_R[i];
    const double* Ji = d->efc_J + (size_t)i * nv;
    if (type == O_CNSTR_FRICTION_DOF) {
      double f = d->efc_frictionloss[i];
      if (jar[i] <= -R * f) { force[i] = f; state[i] = O_STATE_LINEARNEG; cost += -0.5 * R * f * f - f * jar[i]; }
      else if (jar[i] >= R * f) { force[i] = -f; state[i] = O_STATE_LINEARPOS; cost += -0.5 * R * f * f + f * jar[i]; }
      else { force[i] = -D * jar[i]; state[i] = O_STATE_QUADRATIC; cost += 0.5 * D * jar[i] * jar[i]; }
    } else if (type == O_CNSTR_LIMIT_JOINT || type == O_CNSTR_CONTACT_FRICTIONLESS) {
      if (jar[i] < 0) { force[i] = -D * jar[i]; state[i] = O_STATE_QUADRATIC; cost += 0.5 * D * jar[i] * jar[i]; }
      else { force[i] = 0; state[i] = O_STATE_SATISFIED; }
    } else { /* elliptic contact block */
      const OContact* con = d->contact + d->efc_id[i];
      int dim = con->dim;
      double mu = con->mu, U[6];
      U[0] = jar[i] * mu;
      double TT = 0;
      for (int k = 1; k < dim; k++) { U[k] = jar[i + k] * con->friction[k - 1]; TT += U[k] * U[k]; }
      double N = U[0], T = sqrt(TT);
      if (N >= mu * T || (T <= 0 && N >= 0)) {
        for (int k = 0; k < dim; k++) { force[i + k] = 0; state[i + k] = O_STATE_SATISFIED; }
      } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
        for (int k = 0; k < dim; k++) {
          force[i + k] = -d->efc_D[i + k] * jar[i + k];
          state[i + k] = O_STATE_QUADRATIC;
          cost += 0.5 * d->efc_D[i + k] * jar[i + k] * jar[i + k];
        }
        if (H)
          for (int k = 0; k < dim; k++) {
            const double* Jk = Ji + (size_t)k * nv;
            double Dk = d->efc_D[i + k];
            for (int a = 0; a < nv; a++) {
              if (Jk[a] == 0) continue;
              double s = Dk * Jk[a];
              for (int b = 0; b <= a; b++) H[a * nv + b] += s * Jk[b];
            }
          }
      } else {
        double Dm = D / fmax(mu * mu * (1 + mu * mu), O_MINVAL);
        double NT = N - mu * T;
        cost += 0.5 * Dm * NT * NT;
        force[i] = -Dm * NT * mu;
        for (int k = 1; k < dim; k++) force[i + k] = -force[i] / T * U[k] * con->friction[k - 1];
        for (int k = 0; k < dim; k++) state[i + k] = O_STATE_CONE;
        if (H) {
          /* block Hessian in constraint space, then J^T Hc J */
          double Hc[36], sc[6];
          sc[0] = mu;
          for (int k = 1; k < dim; k++) sc[k] = con->friction[k - 1];
          Hc[0] = Dm;
          for (int k = 1; k < dim; k++) Hc[k] = Hc[k * dim] = -Dm * mu * U[k] / T;
          for (int a = 1; a < dim; a++)
            for (int b = 1; b < dim; b++)
              Hc[a * dim + b] = Dm * mu * mu * U[a] * U[b] / (T * T) - Dm * NT * mu * ((a == b ? 1.0 / T : 0.0) - U[a] * U[b] / (T * T * T));
          for (int a = 0; a < dim; a++)
            for (int b = 0; b < dim; b++) Hc[a * dim + b] *= sc[a] * sc[b];
          /* tmp = Hc J (dim x nv) */
          double tmp[6 * 64];
          double* tp = nv <= 64 ? tmp : (double*)malloc(sizeof(double) * 6 * nv);
          for (int a = 0; a < dim; a++)
            for (int x = 0; x < nv; x++) {
              double s = 0;
              for (int b = 0; b < dim; b++) s += Hc[a * dim + b] * Ji[(size_t)b * nv + x];
              tp[a * nv + x] = s;
            }
          for (int x = 0; x < nv; x++)
            for (int y = 0; y <= x; y++) {
              double s = 0;
              for (int a = 0; a < dim; a++) s += Ji[(size_t)a * nv + x] * tp[a * nv + y];
              H[x * nv + y] += s;
            }
          if (tp != tmp) free(tp);
        }
      }
      i += dim - 1;
      continue;
    }
    if (H && state[i] == O_STATE_QUADRATIC)
      for (int a = 0; a < nv; a++) {
        if (Ji[a] == 0) continue;
        double s = D * Ji[a];
        for (int b = 0; b <= a; b++) H[a * nv + b] += s * Ji[b];
      }
  }
  return cost;
}

/* first and second derivative of the total cost along the search direction at step alpha */
static void ls_eval(Ctx* c, double alpha, double quad1, double quad2, double* d1, double* d2) {
  OData* d = c->d;
  double g = quad1 + alpha * quad2, h = quad2;
  for (int i = 0; i < c->nefc; i++) {
    int type = d->efc_type[i];
    double D = d->efc_D[i], R = d->efc_R[i];
    double x = c->jar[i] + alpha * c->jv[i], v = c->jv[i];
    if (type == O_CNSTR_FRICTION_DOF) {
      double f = d->efc_frictionloss[i];
      if (x <= -R * f) g += -f * v;
      else if (x >= R * f) g += f * v;
      else { g += D * x * v; h += D * v * v; }
    } else if (type == O_CNSTR_LIMIT_JOINT || type == O_CNSTR_CONTACT_FRICTIONLESS) {
      if (x < 0) { g += D * x * v; h += D * v * v; }
    } else {
      const OContact* con = d->contact + d->efc_id[i];
      int dim = con->dim;
      double mu = con->mu;
      double N = x * mu, Nd = v * mu, TT = 0, UV = 0, VV = 0;
      for (int k = 1; k < dim; k++) {
        double fk = con->friction[k - 1];
        double u = (c->jar[i + k] + alpha * c->jv[i + k]) * fk, w = c->jv[i + k] * fk;
        TT += u * u; UV += u * w; VV += w * w;
      }
      double T = sqrt(TT);
      if (N >= mu * T || (T <= 0 && N >= 0)) {
        /* satisfied */
      } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
        for (int k = 0; k < dim; k++) {
          double xk = c->jar[i + k] + alpha * c->jv[i + k], vk = c->jv[i + k], Dk = d->efc_D[i + k];
          g += Dk * xk * vk; h += Dk * vk * vk;
        }
      } else {
        double Dm = D / fmax(mu * mu * (1 + mu * mu), O_MINVAL);
        double NT = N - mu * T;
        double Td = UV / T, Tdd = VV / T - UV * UV / (T * T * T);
        double NTd = Nd - mu * Td;
        g += Dm * NT * NTd;
        h += Dm * (NTd * NTd + NT * (-mu * Tdd));
      }
      i += dim - 1;
    }
  }
  *d1 = g;
  *d2 = h;
}

void o_fwd_constraint(const OModel* m, OData* d) {
  int nv = m->nv, nefc = d->nefc;
  memset(d->qfrc_constraint, 0, sizeof(double) * nv);
  d->solver_niter = 0;
  if (nefc == 0) { memcpy(d->qacc, d->qacc_smooth, sizeof(double) * nv); return; }
  Ctx c;
  c.m = m; c.d = d; c.nv = nv; c.nefc = nefc;
  double* buf = (double*)calloc((size_t)2 * nefc + 5 * nv + 2 * nv * nv, sizeof(double));
  c.jar = buf; c.jv = buf + nefc; c.Ma = c.jv + nefc; c.grad = c.Ma + nv; c.search = c.grad + nv; c.Mv = c.search + nv;
  double* tmpv = c.Mv + nv;
  c.H = tmpv + nv; c.L = c.H + nv * nv;
  double* qacc = d->qacc;
  const double* J = d->efc_J;
  double scale = 1.0 / (m->meaninertia * (nv > 1 ? nv : 1));

  /* --- warm start: previous qacc unless the unconstrained acceleration is cheaper */
  double cost_ws, cost_sm;
  for (int pass = 0; pass < 2; pass++) {
    const double* q = pass == 0 ? d->qacc_warmstart : d->qacc_smooth;
    for (int i = 0; i < nefc; i++) {
      double s = -d->efc_aref[i];
      for (int k = 0; k < nv; k++) s += J[(size_t)i * nv + k] * q[k];
      c.jar[i] = s;
    }
    double cc = update_constraint(&c, c.jar, d->efc_force, d->efc_state, NULL);
    if (pass == 0) {
      double gauss = 0;
      for (int i = 0; i < nv; i++) {
        double s = 0;
        for (int k = 0; k < nv; k++) s += d->M[i * nv + k] * q[k];
        gauss += 0.5 * (s - d->qfrc_smooth[i]) * (q[i] - d->qacc_smooth[i]);
      }
      cost_ws = cc + gauss;
    } else cost_sm = cc;
  }
  memcpy(qacc, cost_ws < cost_sm ? d->qacc_warmstart : d->qacc_smooth, sizeof(double) * nv);

  double prev_cost = 0;
  for (int iter = 0; iter <= m->iterations; iter++) {
    /* Ma, jar, cost, gradient, Hessian */
    for (int i = 0; i < nv; i++) {
      double s = 0;
      for (int k = 0; k < nv; k++) s += d->M[i * nv + k] * qacc[k];
      c.Ma[i] = s;
    }
    for (int i = 0; i < nefc; i++) {
      double s = -d->efc_aref[i];
      for (int k = 0; k < nv; k++) s += J[(size_t)i * nv + k] * qacc[k];
      c.jar[i] = s;
    }
    memcpy(c.H, d->M, sizeof(double) * nv * nv);
    double cost = update_constraint(&c, c.jar, d->efc_force, d->efc_state, c.H);
    for (int i = 0; i < nv; i++) cost += 0.5 * (c.Ma[i] - d->qfrc_smooth[i]) * (qacc[i] - d->qacc_smooth[i]);
    double gnorm = 0;
    for (int i = 0; i < nv; i++) {
      double s = c.Ma[i] - d->qfrc_smooth[i];
      for (int r = 0; r < nefc; r++) s -= J[(size_t)r * nv + i] * d->efc_force[r];
      c.grad[i] = s;
      gnorm += s * s;
    }
    gnorm = sqrt(gnorm);
    if (iter > 0) {
      double improvement = scale * (prev_cost - cost);
      if (improvement < m->tolerance || scale * gnorm < m->tolerance) break;
    } else if (scale * gnorm < m->tolerance) break;
    if (iter == m->iterations) break;
    prev_cost = cost;
    d->solver_niter = iter + 1;
    for (int a = 0; a < nv; a++)
      for (int b = a + 1; b < nv; b++) c.H[a * nv + b] = c.H[b * nv + a];
    if (o_chol(c.L, c.H, nv) != 0) { d->warn_flags |= 16; break; }
    for (int i = 0; i < nv; i++) c.search[i] = -c.grad[i];
    o_chol_solve(c.L, c.search, nv);
    /* --- exact line search on the convex 1-D restriction */
    double quad1 = 0, quad2 = 0;
    for (int i = 0; i < nv; i++) {
      double s = 0;
      for (int k = 0; k < nv; k++) s += d->M[i * nv + k] * c.search[k];
      c.Mv[i] = s;
      quad1 += c.search[i] * (c.Ma[i] - d->qfrc_smooth[i]);
      quad2 += c.search[i] * s;
    }
    for (int i = 0; i < nefc; i++) {
      double s = 0;
      for (int k = 0; k < nv; k++) s += J[(size_t)i * nv + k] * c.search[k];
      c.jv[i] = s;
    }
    double d1, d2, alpha = 0, lo = 0, hi = -1, dlo;
    ls_eval(&c, 0, quad1, quad2, &d1, &d2);
    if (d1 >= 0) break; /* not a descent direction: converged to numerical precision */
    dlo = d1;
    double gtol = 1e-12 * fabs(d1);
    alpha = -d1 / d2;
    for (int ls = 0; ls < 100; ls++) {
      ls_eval(&c, alpha, quad1, quad2, &d1, &d2);
      if (fabs(d1) <= gtol) break;
      if (d1 < 0) { lo = alpha; dlo = d1; } else { hi = alpha; }
      double next = alpha - d1 / d2;
      if (hi < 0) { if (next <= lo) next = 2 * alpha + 1e-12; }
      else if (next <= lo || next >= hi) next = 0.5 * (lo + hi);
      if (hi >= 0 && hi - lo < 1e-15 * fmax(1.0, hi)) break;
      alpha = next;
    }
    (void)dlo;
    for (int i = 0; i < nv; i++) qacc[i] += alpha * c.search[i];
  }
  /* final forces at the solution */
  for (int i = 0; i < nefc; i++) {
    double s = -d->efc_aref[i];
    for (int k = 0; k < nv; k++) s += J[(size_t)i * nv + k] * qacc[k];
    c.jar[i] = s;
  }
  update_constraint(&c, c.jar, d->efc_force, d->efc_state, NULL);
  for (int i = 0; i < nv; i++) {
    double s = 0;
    for (int r = 0; r < nefc; r++) s += J[(size_t)r * nv + i] * d->efc_force[r];
    d->qfrc_constraint[i] = s;
  }
  free(buf);
}
