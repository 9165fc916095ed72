/* TEST INFRASTRUCTURE - CPU oracle, collision detection: static pair list + bounding-sphere cull, analytic narrow
 * phase for plane/sphere/box/cylinder pairs, plane-capsule / plane-ellipsoid, sphere-capsule and capsule-capsule (closest
 * points of the cores), box-box by separating axes + face clipping, everything else by
 * GJK + EPA on convex supports (one contact per convex pair: the reference models run with multiccd off,
 * `robosuite/models/world.py:11,18`).  Restates SURVEY.md section 8 row a1 "collision"; parity unpinned. */
#include "b2s_oracle.h"
#include "o_math.h"
#include <float.h>
#include <stdio.h>
#include <stdlib.h>

/* ------------------------------------------------------------------------------------------------ shape access */
typedef struct {
  int type;
  const double* pos;
  const double* mat; /* row-major 3x3, columns are the local axes in world */
  const double* size;
  const double* vert; /* mesh hull vertices (local) */
  int nvert;
} Shape;

static void shape_get(const OModel* m, const OData* d, int g, Shape* s) {
  s->type = m->geom_type[g];
  s->pos = d->geom_xpos + 3 * g;
  s->mat = d->geom_xmat + 9 * g;
  s->size = m->geom_size + 3 * g;
  s->vert = NULL;
  s->nvert = 0;
  if (s->type == O_GEOM_MESH) {
    int id = m->geom_dataid[g];
    s->vert = m->mesh_vert + 3 * m->mesh_vertadr[id];
    s->nvert = m->mesh_vertnum[id];
  }
}

/* support point of the (un-inflated) shape in world direction dir */
static void support(const Shape* s, const double* dir, double* out) {
  double l[3], p[3] = {0, 0, 0};
  m3_mulTv(l, s->mat, dir);
  switch (s->type) {
    case O_GEOM_SPHERE: break; /* core = centre point; radius handled by caller */
    case O_GEOM_BOX:
      p[0] = l[0] >= 0 ? s->size[0] : -s->size[0];
      p[1] = l[1] >= 0 ? s->size[1] : -s->size[1];
      p[2] = l[2] >= 0 ? s->size[2] : -s->size[2];
      break;
    case O_GEOM_CYLINDER: {
      double n = sqrt(l[0] * l[0] + l[1] * l[1]);
      if (n > 1e-12) { p[0] = l[0] / n * s->size[0]; p[1] = l[1] / n * s->size[0]; }
      p[2] = l[2] >= 0 ? s->size[1] : -s->size[1];
      break;
    }
    case O_GEOM_CAPSULE: p[2] = l[2] >= 0 ? s->size[1] : -s->size[1]; break; /* core = segment */
    case O_GEOM_ELLIPSOID: {
      double t[3] = {l[0] * s->size[0], l[1] * s->size[1], l[2] * s->size[2]};
      double n = v3_norm(t);
      if (n > 1e-12) { p[0] = t[0] * s->size[0] / n; p[1] = t[1] * s->size[1] / n; p[2] = t[2] * s->size[2] / n; }
      break;
    }
    case O_GEOM_MESH: {
      double best = -DBL_MAX;
      int bi = 0;
      for (int i = 0; i < s->nvert; i++) {
        double v = s->vert[3 * i] * l[0] + s->vert[3 * i + 1] * l[1] + s->vert[3 * i + 2] * l[2];
        if (v > best) { best = v; bi = i; }
      }
      v3_copy(p, s->vert + 3 * bi);
      break;
    }
    default: break;
  }
  m3_mulv(out, s->mat, p);
  v3_add(out, out, s->pos);
}
static double shape_radius(const Shape* s) {
  return (s->type == O_GEOM_SPHERE || s->type == O_GEOM_CAPSULE) ? s->size[0] : 0.0;
}

/* ------------------------------------------------------------------------------------------------ contact out */
static void make_frame(double* frame) {
  /* frame[0..2] holds the normal; complete to an orthonormal right-handed triad */
  double* x = frame;
  double* y = frame + 3;
  double* z = frame + 6;
  v3_normalize(x);
  v3_set(y, 0, 0, 0);
  if (x[1] < 0.5 && x[1] > -0.5) y[1] = 1; else y[2] = 1;
  double dt = v3_dot(x, y);
  v3_addscl(y, y, x, -dt);
  v3_normalize(y);
  v3_cross(z, x, y);
}
static int add_contact(OContact* out, int n, int maxout, const double* pos, const double* normal, double dist) {
  if (n >= maxout) return n;
  OContact* c = out + n;
  c->dist = dist;
  v3_copy(c->pos, pos);
  v3_copy(c->frame, normal);
  make_frame(c->frame);
  return n + 1;
}
#define COL(R, k) {(R)[k], (R)[3 + (k)], (R)[6 + (k)]}

/* ------------------------------------------------------------------------------------------------ plane pairs */
static int plane_sphere(const Shape* p, const Shape* s, OContact* out, int maxout) {
  double n[3] = COL(p->mat, 2), df[3], pos[3];
  v3_sub(df, s->pos, p->pos);
  double dist = v3_dot(df, n) - s->size[0];
  if (dist > 0) return 0;
  v3_addscl(pos, s->pos, n, -(s->size[0] + 0.5 * dist));
  return add_contact(out, 0, maxout, pos, n, dist);
}
static int plane_box(const Shape* p, const Shape* b, OContact* out, int maxout) {
  double n[3] = COL(p->mat, 2), df[3];
  v3_sub(df, b->pos, p->pos);
  double dist = v3_dot(df, n);
  int cnt = 0;
  for (int i = 0; i < 8 && cnt < 4; i++) {
    double vec[3] = {(i & 1 ? 1 : -1) * b->size[0], (i & 2 ? 1 : -1) * b->size[1], (i & 4 ? 1 : -1) * b->size[2]};
    double corner[3], pos[3];
    m3_mulv(corner, b->mat, vec);
    double ld = v3_dot(n, corner);
    if (dist + ld > 0 || ld > 0) continue;
    double cd = dist + ld;
    v3_add(pos, b->pos, corner);
    v3_addscl(pos, pos, n, -0.5 * cd);
    cnt = add_contact(out, cnt, maxout, pos, n, cd);
  }
  return cnt;
}
static int plane_cylinder(const Shape* p, const Shape* c, OContact* out, int maxout) {
  double n[3] = COL(p->mat, 2), axis[3] = COL(c->mat, 2), df[3], vec[3], pos[3];
  double r = c->size[0], h = c->size[1];
  v3_sub(df, c->pos, p->pos);
  double dist0 = v3_dot(df, n);
  double prjaxis = v3_dot(n, axis);
  if (prjaxis > 0) { v3_scl(axis, axis, -1); prjaxis = -prjaxis; } /* axis now points toward the plane */
  /* direction in the cap plane pointing most toward the plane: -(n - axis (n.axis)) */
  v3_scl(vec, n, -1);
  v3_addscl(vec, vec, axis, prjaxis); /* -(n - axis (n.axis)) */
  double len = v3_norm(vec);
  if (len < 1e-12) { double x[3] = COL(c->mat, 0); v3_scl(vec, x, r); }
  else v3_scl(vec, vec, r / len);
  double prjvec = v3_dot(vec, n); /* <= 0 */
  int cnt = 0;
  /* 1: rim point of the near cap closest to the plane */
  double d1 = dist0 + h * prjaxis + prjvec;
  if (d1 > 0) return 0;
  v3_addscl(pos, c->pos, axis, h);
  v3_add(pos, pos, vec);
  v3_addscl(pos, pos, n, -0.5 * d1);
  cnt = add_contact(out, cnt, maxout, pos, n, d1);
  /* 2: same generator line, far cap (cylinder lying on its side) */
  double d2 = dist0 - h * prjaxis + prjvec;
  if (d2 <= 0) {
    v3_addscl(pos, c->pos, axis, -h);
    v3_add(pos, pos, vec);
    v3_addscl(pos, pos, n, -0.5 * d2);
    cnt = add_contact(out, cnt, maxout, pos, n, d2);
  }
  /* 3,4: two more rim points of the near cap at +-120 degrees (cylinder standing on its cap) */
  double side[3];
  v3_cross(side, vec, axis);
  v3_normalize(side);
  v3_scl(side, side, r * sqrt(3.0) / 2.0);
  for (int k = 0; k < 2; k++) {
    double off[3];
    v3_scl(off, vec, -0.5);
    v3_addscl(off, off, side, k ? -1.0 : 1.0);
    double d3 = dist0 + h * prjaxis + v3_dot(off, n);
    if (d3 > 0) continue;
    v3_addscl(pos, c->pos, axis, h);
    v3_add(pos, pos, off);
    v3_addscl(pos, pos, n, -0.5 * d3);
    cnt = add_contact(out, cnt, maxout, pos, n, d3);
  }
  return cnt;
}
static int plane_capsule(const Shape* p, const Shape* c, OContact* out, int maxout) {
  /* one contact per penetrating end sphere of the segment, + end first */
  double n[3] = COL(p->mat, 2), axis[3] = COL(c->mat, 2), df[3], pos[3];
  double r = c->size[0], h = c->size[1];
  v3_sub(df, c->pos, p->pos);
  double dist0 = v3_dot(df, n), prj = h * v3_dot(n, axis);
  int cnt = 0;
  for (int k = 0; k < 2; k++) {
    double sg = k ? -1.0 : 1.0, dist = dist0 + sg * prj - r;
    if (dist > 0) continue;
    v3_addscl(pos, c->pos, axis, sg * h);
    v3_addscl(pos, pos, n, -(r + 0.5 * dist));
    cnt = add_contact(out, cnt, maxout, pos, n, dist);
  }
  return cnt;
}
static int plane_ellipsoid(const Shape* p, const Shape* e, OContact* out, int maxout) {
  /* support point of the ellipsoid along -n: local -S^2 nl / |S nl| */
  double n[3] = COL(p->mat, 2), nl[3], df[3], sp[3], w[3], pos[3];
  m3_mulTv(nl, e->mat, n);
  double t[3] = {nl[0] * e->size[0], nl[1] * e->size[1], nl[2] * e->size[2]};
  double len = v3_norm(t);
  for (int k = 0; k < 3; k++) sp[k] = -t[k] * e->size[k] / len;
  m3_mulv(w, e->mat, sp);
  v3_add(w, w, e->pos);
  v3_sub(df, w, p->pos);
  double dist = v3_dot(df, n);
  if (dist > 0) return 0;
  v3_addscl(pos, w, n, -0.5 * dist);
  return add_contact(out, 0, maxout, pos, n, dist);
}
static int plane_mesh(const Shape* p, const Shape* s, OContact* out, int maxout) {
  /* deepest hull vertex first, then up to three more penetrating vertices chosen greedily far from those taken */
  double n[3] = COL(p->mat, 2), nl[3];
  m3_mulTv(nl, s->mat, n);
  double df[3];
  v3_sub(df, s->pos, p->pos);
  double base = v3_dot(df, n);
  int chosen[4], cnt = 0, nc = 0;
  for (int round = 0; round < 4; round++) {
    int best = -1;
    double bestscore = -DBL_MAX;
    for (int i = 0; i < s->nvert; i++) {
      double dist = base + v3_dot(s->vert + 3 * i, nl);
      if (dist > 0) continue;
      double score;
      if (round == 0) score = -dist;
      else {
        score = DBL_MAX;
        int dup = 0;
        for (int k = 0; k < nc; k++) {
          double e[3];
          v3_sub(e, s->vert + 3 * i, s->vert + 3 * chosen[k]);
          double dd = v3_dot(e, e);
          if (chosen[k] == i) dup = 1;
          if (dd < score) score = dd;
        }
        if (dup || score < 1e-10) continue;
      }
      if (score > bestscore) { bestscore = score; best = i; }
    }
    if (best < 0) break;
    chosen[nc++] = best;
    double w[3], pos[3];
    m3_mulv(w, s->mat, s->vert + 3 * best);
    v3_add(w, w, s->pos);
    double dist = base + v3_dot(s->vert + 3 * best, nl);
    v3_addscl(pos, w, n, -0.5 * dist);
    cnt = add_contact(out, cnt, maxout, pos, n, dist);
  }
  return cnt;
}

/* ------------------------------------------------------------------------------------------------ sphere pairs */
static int sphere_sphere(const Shape* a, const Shape* b, OContact* out, int maxout) {
  double n[3], pos[3];
  v3_sub(n, b->pos, a->pos);
  double len = v3_norm(n), dist = len - a->size[0] - b->size[0];
  if (dist > 0) return 0;
  if (len < 1e-12) v3_set(n, 1, 0, 0); else v3_scl(n, n, 1.0 / len);
  v3_addscl(pos, a->pos, n, a->size[0] + 0.5 * dist);
  return add_contact(out, 0, maxout, pos, n, dist);
}
static int sphere_box(const Shape* s, const Shape* b, OContact* out, int maxout) {
  double df[3], c[3], cl[3], n[3], pos[3];
  v3_sub(df, s->pos, b->pos);
  m3_mulTv(c, b->mat, df);
  int inside = 1;
  for (int k = 0; k < 3; k++) {
    cl[k] = fmin(fmax(c[k], -b->size[k]), b->size[k]);
    if (cl[k] != c[k]) inside = 0;
  }
  double dist, r = s->size[0];
  if (inside) {
    int ax = 0;
    double best = DBL_MAX;
    for (int k = 0; k < 3; k++) {
      double dd = b->size[k] - fabs(c[k]);
      if (dd < best) { best = dd; ax = k; }
    }
    double nl[3] = {0, 0, 0};
    nl[ax] = c[ax] >= 0 ? -1 : 1; /* from sphere (geom1) into the box (geom2) */
    m3_mulv(n, b->mat, nl);
    dist = -best - r;
  } else {
    double e[3], el[3];
    v3_sub(el, cl, c);
    double len = v3_norm(el);
    dist = len - r;
    if (dist > 0) return 0;
    v3_scl(el, el, 1.0 / len);
    m3_mulv(e, b->mat, el);
    v3_copy(n, e);
  }
  v3_addscl(pos, s->pos, n, r + 0.5 * dist);
  return add_contact(out, 0, maxout, pos, n, dist);
}
static int sphere_cylinder(const Shape* s, const Shape* c, OContact* out, int maxout) {
  double df[3], p[3], q[3], n[3], pos[3];
  double R = c->size[0], h = c->size[1], r = s->size[0];
  v3_sub(df, s->pos, c->pos);
  m3_mulTv(p, c->mat, df);
  double rho = sqrt(p[0] * p[0] + p[1] * p[1]);
  double dist;
  if (rho <= R && fabs(p[2]) <= h) { /* centre inside the solid cylinder */
    double dside = R - rho, dcap = h - fabs(p[2]);
    double nl[3] = {0, 0, 0};
    if (dcap < dside) { nl[2] = p[2] >= 0 ? -1 : 1; dist = -dcap - r; }
    else if (rho < 1e-12) { nl[0] = 1; dist = -dside - r; } /* on the axis, nearer the side: a fixed perpendicular */
    else { nl[0] = -p[0] / rho; nl[1] = -p[1] / rho; dist = -dside - r; }
    m3_mulv(n, c->mat, nl);
  } else {
    double sc = rho > R ? R / rho : 1.0;
    q[0] = p[0] * sc; q[1] = p[1] * sc; q[2] = fmin(fmax(p[2], -h), h);
    double el[3];
    v3_sub(el, q, p);
    double len = v3_norm(el);
    dist = len - r;
    if (dist > 0) return 0;
    v3_scl(el, el, 1.0 / len);
    m3_mulv(n, c->mat, el);
  }
  v3_addscl(pos, s->pos, n, r + 0.5 * dist);
  return add_contact(out, 0, maxout, pos, n, dist);
}

/* ------------------------------------------------------------------------------------------------ capsule pairs */
/* closest points of the segments a + s u (|s| <= ha) and b + t v (|t| <= hb), u and v unit; parallel segments take s = 0 */
static void seg_seg(const double* a, const double* u, double ha, const double* b, const double* v, double hb, double* p, double* q) {
  double r[3];
  v3_sub(r, a, b);
  double uv = v3_dot(u, v), c = v3_dot(u, r), f = v3_dot(v, r), den = 1 - uv * uv;
  double s = den > 1e-12 ? fmin(fmax((uv * f - c) / den, -ha), ha) : 0.0;
  double t = uv * s + f;
  if (t < -hb || t > hb) {
    t = fmin(fmax(t, -hb), hb);
    s = fmin(fmax(uv * t - c, -ha), ha);
  }
  v3_addscl(p, a, u, s);
  v3_addscl(q, b, v, t);
}
/* contact of two inflated cores with closest points p (on A's core) and q (on B's); nfb: normal when p == q */
static int core_contact(const double* p, const double* q, double ra, double rb, const double* nfb, OContact* out, int maxout) {
  double n[3], pos[3];
  v3_sub(n, q, p);
  double len = v3_norm(n), dist = len - ra - rb;
  if (dist > 0) return 0;
  if (len < 1e-12) v3_copy(n, nfb); else v3_scl(n, n, 1.0 / len);
  v3_addscl(pos, p, n, ra + 0.5 * dist);
  return add_contact(out, 0, maxout, pos, n, dist);
}
static int sphere_capsule(const Shape* s, const Shape* c, OContact* out, int maxout) {
  double axis[3] = COL(c->mat, 2), nfb[3] = COL(c->mat, 0), df[3], q[3];
  v3_sub(df, s->pos, c->pos);
  v3_addscl(q, c->pos, axis, fmin(fmax(v3_dot(df, axis), -c->size[1]), c->size[1]));
  return core_contact(s->pos, q, s->size[0], c->size[0], nfb, out, maxout); /* centre on the segment: a fixed perpendicular */
}
static int capsule_capsule(const Shape* A, const Shape* B, OContact* out, int maxout) {
  double u[3] = COL(A->mat, 2), v[3] = COL(B->mat, 2), p[3], q[3], nfb[3], df[3];
  seg_seg(A->pos, u, A->size[1], B->pos, v, B->size[1], p, q);
  /* intersecting cores: crossing axes take their common perpendicular, pointing along the centre difference; collinear ones a
   * fixed perpendicular of A's axis */
  v3_cross(nfb, u, v);
  double len = v3_norm(nfb);
  if (len > 1e-6) {
    v3_sub(df, B->pos, A->pos);
    v3_scl(nfb, nfb, (v3_dot(nfb, df) < 0 ? -1.0 : 1.0) / len);
  } else v3_set(nfb, A->mat[0], A->mat[3], A->mat[6]);
  return core_contact(p, q, A->size[0], B->size[0], nfb, out, maxout);
}

/* ------------------------------------------------------------------------------------------------ box - box */
static int clip_poly(double (*poly)[2], int n, int axis, double lim, double sign) {
  /* keep the part of the polygon with sign*coord[axis] <= lim (Sutherland-Hodgman, in place) */
  double outp[16][2];
  int no = 0;
  for (int i = 0; i < n; i++) {
    const double* a = poly[i];
    const double* b = poly[(i + 1) % n];
    double da = sign * a[axis] - lim, db = sign * b[axis] - lim;
    if (da <= 0) { outp[no][0] = a[0]; outp[no][1] = a[1]; no++; }
    if ((da < 0 && db > 0) || (da > 0 && db < 0)) {
      double t = da / (da - db);
      outp[no][0] = a[0] + t * (b[0] - a[0]);
      outp[no][1] = a[1] + t * (b[1] - a[1]);
      no++;
    }
    if (no >= 15) break;
  }
  for (int i = 0; i < no; i++) { poly[i][0] = outp[i][0]; poly[i][1] = outp[i][1]; }
  return no;
}

static int box_box(const Shape* A, const Shape* B, OContact* out, int maxout) {
  double Aax[3][3], Bax[3][3], T[3];
  for (int k = 0; k < 3; k++) {
    double a[3] = COL(A->mat, k), b[3] = COL(B->mat, k);
    v3_copy(Aax[k], a);
    v3_copy(Bax[k], b);
  }
  v3_sub(T, B->pos, A->pos);
  double best = DBL_MAX, bestn[3] = {0, 0, 0};
  int code = -1;
  /* face axes */
  for (int k = 0; k < 6; k++) {
    const double* L = k < 3 ? Aax[k] : Bax[k - 3];
    double ra = 0, rb = 0;
    for (int i = 0; i < 3; i++) { ra += A->size[i] * fabs(v3_dot(Aax[i], L)); rb += B->size[i] * fabs(v3_dot(Bax[i], L)); }
    double tl = v3_dot(T, L), ov = ra + rb - fabs(tl);
    if (ov < 0) return 0;
    if (ov + 1e-5 < best) { best = ov; code = k; v3_scl(bestn, L, tl >= 0 ? 1 : -1); }
  }
  /* edge-edge axes (fudge so that faces win near ties) */
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double L[3];
      v3_cross(L, Aax[i], Bax[j]);
      double len = v3_norm(L);
      if (len < 1e-6) continue;
      v3_scl(L, L, 1.0 / len);
      double ra = 0, rb = 0;
      for (int k = 0; k < 3; k++) { ra += A->size[k] * fabs(v3_dot(Aax[k], L)); rb += B->size[k] * fabs(v3_dot(Bax[k], L)); }
      double tl = v3_dot(T, L), ov = ra + rb - fabs(tl);
      if (ov < 0) return 0;
      if (ov * 1.05 + 1e-5 < best) { best = ov * 1.05 + 1e-5; code = 6 + 3 * i + j; v3_scl(bestn, L, tl >= 0 ? 1 : -1); }
    }
  if (code < 0) return 0;
  double n[3];
  v3_copy(n, bestn); /* points from A (geom1) to B (geom2) */
  if (code >= 6) {
    int i = (code - 6) / 3, j = (code - 6) % 3;
    double pa[3], pb[3];
    v3_copy(pa, A->pos);
    v3_copy(pb, B->pos);
    for (int k = 0; k < 3; k++) {
      if (k != i) v3_addscl(pa, pa, Aax[k], (v3_dot(Aax[k], n) > 0 ? 1 : -1) * A->size[k]);
      if (k != j) v3_addscl(pb, pb, Bax[k], (v3_dot(Bax[k], n) > 0 ? -1 : 1) * B->size[k]);
    }
    /* closest points of lines pa + s u, pb + t v */
    const double* u = Aax[i];
    const double* v = Bax[j];
    double w[3];
    v3_sub(w, pa, pb);
    double uv = v3_dot(u, v), uw = v3_dot(u, w), vw = v3_dot(v, w), den = 1 - uv * uv;
    double s = den > 1e-12 ? (uv * vw - uw) / den : 0, t = den > 1e-12 ? (vw - uv * uw) / den : 0;
    s = fmin(fmax(s, -A->size[i]), A->size[i]);
    t = fmin(fmax(t, -B->size[j]), B->size[j]);
    double qa[3], qb[3], pos[3];
    v3_addscl(qa, pa, u, s);
    v3_addscl(qb, pb, v, t);
    v3_add(pos, qa, qb);
    v3_scl(pos, pos, 0.5);
    double dv[3];
    v3_sub(dv, qb, qa);
    double dist = v3_dot(dv, n);
    if (dist > 0) return 0;
    return add_contact(out, 0, maxout, pos, n, dist);
  }
  /* face contact: reference box R (face along axis `ax`), incident box Ic */
  const Shape* Rf = code < 3 ? A : B;
  const Shape* Ic = code < 3 ? B : A;
  double (*Rax)[3] = code < 3 ? Aax : Bax;
  double (*Iax)[3] = code < 3 ? Bax : Aax;
  int ax = code < 3 ? code : code - 3;
  double nr[3]; /* outward normal of the reference face */
  v3_scl(nr, n, code < 3 ? 1 : -1);
  int iu = (ax + 1) % 3, iv = (ax + 2) % 3;
  /* incident face: most anti-parallel to nr */
  int ia = 0;
  double bestd = -1;
  for (int k = 0; k < 3; k++) {
    double dd = fabs(v3_dot(Iax[k], nr));
    if (dd > bestd) { bestd = dd; ia = k; }
  }
  double sgn = v3_dot(Iax[ia], nr) > 0 ? -1 : 1;
  double fc[3];
  v3_addscl(fc, Ic->pos, Iax[ia], sgn * Ic->size[ia]);
  int ju = (ia + 1) % 3, jv = (ia + 2) % 3;
  double rc[3]; /* reference face centre */
  v3_addscl(rc, Rf->pos, nr, Rf->size[ax]);
  double poly[16][2], hgt[4];
  double corners[4][3];
  static const int sg[4][2] = {{1, 1}, {-1, 1}, {-1, -1}, {1, -1}};
  for (int k = 0; k < 4; k++) {
    v3_copy(corners[k], fc);
    v3_addscl(corners[k], corners[k], Iax[ju], sg[k][0] * Ic->size[ju]);
    v3_addscl(corners[k], corners[k], Iax[jv], sg[k][1] * Ic->size[jv]);
    double rel[3];
    v3_sub(rel, corners[k], rc);
    poly[k][0] = v3_dot(rel, Rax[iu]);
    poly[k][1] = v3_dot(rel, Rax[iv]);
    hgt[k] = v3_dot(rel, nr);
  }
  /* height is affine in the 2-D coordinates of the incident face: h = h0 + g . (x - x0) */
  double e1[2] = {poly[1][0] - poly[0][0], poly[1][1] - poly[0][1]}, e2[2] = {poly[3][0] - poly[0][0], poly[3][1] - poly[0][1]};
  double det = e1[0] * e2[1] - e1[1] * e2[0];
  double x0[2] = {poly[0][0], poly[0][1]};
  double h0 = hgt[0], dh1 = hgt[1] - hgt[0], dh2 = hgt[3] - hgt[0];
  int np = 4;
  np = clip_poly(poly, np, 0, Rf->size[iu], 1);
  np = clip_poly(poly, np, 0, Rf->size[iu], -1);
  np = clip_poly(poly, np, 1, Rf->size[iv], 1);
  np = clip_poly(poly, np, 1, Rf->size[iv], -1);
  int cnt = 0;
  for (int k = 0; k < np && cnt < 8; k++) {
    double hh;
    if (fabs(det) > 1e-14) {
      double dx = poly[k][0] - x0[0], dy = poly[k][1] - x0[1];
      double a = (dx * e2[1] - dy * e2[0]) / det, b = (e1[0] * dy - e1[1] * dx) / det;
      hh = h0 + a * dh1 + b * dh2;
    } else hh = h0;
    if (hh > 0) continue; /* above the reference face: not penetrating */
    /* point on incident face (world) and its projection on the reference face */
    double p[3], pos[3];
    v3_copy(p, rc);
    v3_addscl(p, p, Rax[iu], poly[k][0]);
    v3_addscl(p, p, Rax[iv], poly[k][1]);
    v3_addscl(p, p, nr, hh);
    v3_addscl(pos, p, nr, -0.5 * hh); /* midway between p and the reference face */
    cnt = add_contact(out, cnt, maxout, pos, n, hh);
  }
  return cnt;
}

/* ------------------------------------------------------------------------------------------------ GJK + EPA */
typedef struct { double w[3], a[3], b[3]; } SV; /* Minkowski-difference vertex with witnesses */

static void sv_support(const Shape* A, const Shape* B, const double* dir, SV* o) {
  double nd[3] = {-dir[0], -dir[1], -dir[2]};
  support(A, dir, o->a);
  support(B, nd, o->b);
  v3_sub(o->w, o->a, o->b);
}

/* closest point to the origin on a simplex; reduces the simplex to the supporting sub-simplex and returns
 * barycentric weights.  Returns 1 if the origin is inside a tetrahedron. */
static void closest_seg(SV* s, int* n, double* lam) {
  double ab[3];
  v3_sub(ab, s[1].w, s[0].w);
  double den = v3_dot(ab, ab);
  double t = den > 0 ? -v3_dot(s[0].w, ab) / den : 0;
  if (t <= 0) { *n = 1; lam[0] = 1; }
  else if (t >= 1) { s[0] = s[1]; *n = 1; lam[0] = 1; }
  else { lam[0] = 1 - t; lam[1] = t; }
}
static void closest_tri(SV* s, int* n, double* lam) {
  const double *a = s[0].w, *b = s[1].w, *c = s[2].w;
  double ab[3], ac[3], ap[3], bp[3], cp[3];
  v3_sub(ab, b, a); v3_sub(ac, c, a);
  v3_scl(ap, a, -1);
  double d1 = v3_dot(ab, ap), d2 = v3_dot(ac, ap);
  if (d1 <= 0 && d2 <= 0) { *n = 1; lam[0] = 1; return; }
  v3_scl(bp, b, -1);
  double d3 = v3_dot(ab, bp), d4 = v3_dot(ac, bp);
  if (d3 >= 0 && d4 <= d3) { s[0] = s[1]; *n = 1; lam[0] = 1; return; }
  double vc = d1 * d4 - d3 * d2;
  if (vc <= 0 && d1 >= 0 && d3 <= 0) { double v = d1 / (d1 - d3); *n = 2; lam[0] = 1 - v; lam[1] = v; return; }
  v3_scl(cp, c, -1);
  double d5 = v3_dot(ab, cp), d6 = v3_dot(ac, cp);
  if (d6 >= 0 && d5 <= d6) { s[0] = s[2]; *n = 1; lam[0] = 1; return; }
  double vb = d5 * d2 - d1 * d6;
  if (vb <= 0 && d2 >= 0 && d6 <= 0) { double w = d2 / (d2 - d6); s[1] = s[2]; *n = 2; lam[0] = 1 - w; lam[1] = w; return; }
  double va = d3 * d6 - d5 * d4;
  if (va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0) {
    double w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
    s[0] = s[1]; s[1] = s[2]; *n = 2; lam[0] = 1 - w; lam[1] = w; return;
  }
  double den = 1.0 / (va + vb + vc);
  lam[1] = vb * den; lam[2] = vc * den; lam[0] = 1 - lam[1] - lam[2];
}
static double orient(const double* a, const double* b, const double* c, const double* d) {
  double ab[3], ac[3], ad[3], cr[3];
  v3_sub(ab, b, a); v3_sub(ac, c, a); v3_sub(ad, d, a);
  v3_cross(cr, ab, ac);
  return v3_dot(cr, ad);
}
static int closest_tet(SV* s, int* n, double* lam) {
  /* test the four faces; if the origin is on the inner side of all -> inside */
  static const int F[4][3] = {{0, 1, 2}, {0, 1, 3}, {0, 2, 3}, {1, 2, 3}};
  static const int O[4] = {3, 2, 1, 0};
  double zero[3] = {0, 0, 0};
  double bestd = DBL_MAX;
  SV bests[3];
  double bestlam[3];
  int bestn = 0, outside = 0;
  for (int f = 0; f < 4; f++) {
    double so = orient(s[F[f][0]].w, s[F[f][1]].w, s[F[f][2]].w, zero);
    double sd = orient(s[F[f][0]].w, s[F[f][1]].w, s[F[f][2]].w, s[O[f]].w);
    if (fabs(sd) < 1e-30) { outside = 1; } /* degenerate tetra: treat every face as candidate */
    if (fabs(sd) >= 1e-30 && so * sd > 0) continue; /* origin on the same side as the opposite vertex */
    outside = 1;
    SV t[3] = {s[F[f][0]], s[F[f][1]], s[F[f][2]]};
    int tn = 3;
    double tl[3] = {0, 0, 0};
    closest_tri(t, &tn, tl);
    double p[3] = {0, 0, 0};
    for (int k = 0; k < tn; k++) v3_addscl(p, p, t[k].w, tl[k]);
    double dd = v3_dot(p, p);
    if (dd < bestd) { bestd = dd; bestn = tn; for (int k = 0; k < tn; k++) { bests[k] = t[k]; bestlam[k] = tl[k]; } }
  }
  if (!outside) return 1;
  *n = bestn;
  for (int k = 0; k < bestn; k++) { s[k] = bests[k]; lam[k] = bestlam[k]; }
  return 0;
}

/* GJK on the cores.  Returns: 0 separated (dist, witnesses wa/wb valid), 1 overlapping (simplex valid for EPA).
 * If `cutoff` >= 0 the search stops as soon as the cores are proven further apart than cutoff (returns 0, dist=cutoff+1). */
static int gjk(const Shape* A, const Shape* B, SV* simplex, int* ns, double* dist, double* wa, double* wb, double cutoff) {
  double v[3];
  v3_sub(v, A->pos, B->pos);
  if (v3_dot(v, v) < 1e-20) v3_set(v, 1, 0, 0);
  int n = 0;
  double lam[4] = {1, 0, 0, 0};
  double nv[3];
  v3_scl(nv, v, -1);
  sv_support(A, B, nv, &simplex[0]);
  n = 1;
  v3_copy(v, simplex[0].w);
  for (int it = 0; it < 64; it++) {
    double vv = v3_dot(v, v);
    if (vv < 1e-24) { *ns = n; return 1; }
    SV w;
    v3_scl(nv, v, -1);
    sv_support(A, B, nv, &w);
    double vw = v3_dot(v, w.w);
    /* lower bound on the distance: vw / |v| */
    if (cutoff >= 0 && vw > 0 && vw * vw > cutoff * cutoff * vv) { *dist = cutoff + 1; *ns = n; return 0; }
    if (vv - vw <= 1e-12 * vv) break; /* no progress possible: v is the closest point */
    int dup = 0;
    for (int k = 0; k < n; k++) {
      double e[3];
      v3_sub(e, simplex[k].w, w.w);
      if (v3_dot(e, e) < 1e-24) dup = 1;
    }
    if (dup) break;
    simplex[n++] = w;
    if (n == 2) closest_seg(simplex, &n, lam);
    else if (n == 3) closest_tri(simplex, &n, lam);
    else if (closest_tet(simplex, &n, lam)) { *ns = 4; return 1; }
    v3_set(v, 0, 0, 0);
    for (int k = 0; k < n; k++) v3_addscl(v, v, simplex[k].w, lam[k]);
  }
  *ns = n;
  *dist = v3_norm(v);
  v3_set(wa, 0, 0, 0);
  v3_set(wb, 0, 0, 0);
  for (int k = 0; k < n; k++) { v3_addscl(wa, wa, simplex[k].a, lam[k]); v3_addscl(wb, wb, simplex[k].b, lam[k]); }
  return 0;
}

#define EPA_MAXV 96   /* same polytope capacity, iteration cap and stopping rule as the device (csrc/b2s_collide.cuh) */
#define EPA_MAXF 192
typedef struct { int v[3]; double n[3]; double d; int alive; } EFace;

static int epa_face(EFace* f, const SV* V, int a, int b, int c) {
  f->v[0] = a; f->v[1] = b; f->v[2] = c;
  double ab[3], ac[3];
  v3_sub(ab, V[b].w, V[a].w);
  v3_sub(ac, V[c].w, V[a].w);
  v3_cross(f->n, ab, ac);
  double len = v3_norm(f->n);
  f->alive = 1;
  if (len < 1e-30) { f->d = DBL_MAX; return -1; }
  v3_scl(f->n, f->n, 1.0 / len);
  f->d = v3_dot(f->n, V[a].w);
  return 0;
}

/* EPA from an enclosing simplex.  Output: penetration depth (>0), normal (A -> B), witnesses. */
static int epa(const Shape* A, const Shape* B, SV* simplex, int ns, double* depth, double* normal, double* wa, double* wb) {
  SV V[EPA_MAXV];
  EFace F[EPA_MAXF];
  static int epa_trace = -1; /* B2S_EPA_TRACE=1: print the expansion steps (tools/debug_epa.py) */
  if (epa_trace < 0) epa_trace = getenv("B2S_EPA_TRACE") != NULL;
  int nV = 0, nF = 0;
  for (int k = 0; k < ns; k++) V[nV++] = simplex[k];
  /* grow a degenerate simplex into a tetrahedron (acceptance thresholds relative to the simplex's size, as on the device) */
  static const double dirs[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
  if (nV == 1) {
    for (int k = 0; k < 6 && nV < 2; k++) {
      SV w;
      sv_support(A, B, dirs[k], &w);
      double e[3];
      v3_sub(e, w.w, V[0].w);
      if (v3_dot(e, e) > 1e-12) V[nV++] = w;
    }
  }
  if (nV == 2) {
    double ab[3];
    v3_sub(ab, V[1].w, V[0].w);
    for (int k = 0; k < 6 && nV < 3; k++) {
      double dir[3];
      v3_cross(dir, ab, dirs[k]);
      if (v3_dot(dir, dir) < 1e-12 * v3_dot(ab, ab)) continue;
      SV w;
      sv_support(A, B, dir, &w);
      double e[3], cr[3];
      v3_sub(e, w.w, V[0].w);
      v3_cross(cr, ab, e);
      if (v3_dot(cr, cr) > 1e-12 * v3_dot(ab, ab) * v3_dot(ab, ab)) V[nV++] = w;
    }
  }
  if (nV == 3) {
    double ab[3], ac[3], nrm[3];
    v3_sub(ab, V[1].w, V[0].w);
    v3_sub(ac, V[2].w, V[0].w);
    v3_cross(nrm, ab, ac);
    for (int s = 0; s < 2 && nV < 4; s++) {
      double dir[3];
      v3_scl(dir, nrm, s ? -1 : 1);
      SV w;
      sv_support(A, B, dir, &w);
      double e[3];
      v3_sub(e, w.w, V[0].w);
      if (fabs(v3_dot(e, nrm)) > 1e-7 * v3_dot(nrm, nrm)) V[nV++] = w;
    }
  }
  if (nV < 4) return -1;
  /* orient so that face normals point outward */
  if (orient(V[0].w, V[1].w, V[2].w, V[3].w) > 0) { SV t = V[0]; V[0] = V[1]; V[1] = t; }
  epa_face(&F[nF++], V, 0, 1, 2);
  epa_face(&F[nF++], V, 0, 3, 1);
  epa_face(&F[nF++], V, 0, 2, 3);
  epa_face(&F[nF++], V, 1, 3, 2);
  int bestf = -1;
  for (int it = 0; it < 100; it++) {
    double bd = DBL_MAX;
    bestf = -1;
    for (int f = 0; f < nF; f++)
      if (F[f].alive && F[f].d < bd) { bd = F[f].d; bestf = f; }
    if (bestf < 0) return -1;
    SV w;
    sv_support(A, B, F[bestf].n, &w);
    double dw = v3_dot(w.w, F[bestf].n);
    if (epa_trace) fprintf(stderr, "ora it %d bf %d bd %.9g dw %.9g nV %d nF %d n %.4f %.4f %.4f\n", it, bestf, bd, dw, nV, nF, F[bestf].n[0], F[bestf].n[1], F[bestf].n[2]);
    if (dw - bd < 1e-7 || nV >= EPA_MAXV - 1 || nF >= EPA_MAXF - 16) break;
    /* remove faces visible from w, collect horizon */
    int edges[64][2], ne = 0;
    for (int f = 0; f < nF; f++) {
      if (!F[f].alive) continue;
      double e[3];
      v3_sub(e, w.w, V[F[f].v[0]].w);
      if (v3_dot(F[f].n, e) > 1e-12) {
        F[f].alive = 0;
        for (int k = 0; k < 3; k++) {
          int a = F[f].v[k], b = F[f].v[(k + 1) % 3], found = 0;
          for (int q = 0; q < ne; q++)
            if (edges[q][0] == b && edges[q][1] == a) { edges[q][0] = edges[ne - 1][0]; edges[q][1] = edges[ne - 1][1]; ne--; found = 1; break; }
          if (!found && ne < 64) { edges[ne][0] = a; edges[ne][1] = b; ne++; }
        }
      }
    }
    if (epa_trace) fprintf(stderr, "ora    ne %d\n", ne);
    if (ne == 0) break;
    int vi = nV;
    V[nV++] = w;
    for (int q = 0; q < ne && nF < EPA_MAXF; q++) epa_face(&F[nF++], V, edges[q][0], edges[q][1], vi);
  }
  if (bestf < 0) return -1;
  const EFace* f = &F[bestf];
  *depth = f->d;
  v3_copy(normal, f->n);
  /* barycentric coordinates of the projection of the origin onto the face */
  double p[3];
  v3_scl(p, f->n, f->d);
  const double *a = V[f->v[0]].w, *b = V[f->v[1]].w, *c = V[f->v[2]].w;
  double v0[3], v1[3], v2[3];
  v3_sub(v0, b, a); v3_sub(v1, c, a); v3_sub(v2, p, a);
  double d00 = v3_dot(v0, v0), d01 = v3_dot(v0, v1), d11 = v3_dot(v1, v1), d20 = v3_dot(v2, v0), d21 = v3_dot(v2, v1);
  double den = d00 * d11 - d01 * d01;
  double bv = den != 0 ? (d11 * d20 - d01 * d21) / den : 0, bw = den != 0 ? (d00 * d21 - d01 * d20) / den : 0;
  double bu = 1 - bv - bw;
  for (int k = 0; k < 3; k++) {
    wa[k] = bu * V[f->v[0]].a[k] + bv * V[f->v[1]].a[k] + bw * V[f->v[2]].a[k];
    wb[k] = bu * V[f->v[0]].b[k] + bv * V[f->v[1]].b[k] + bw * V[f->v[2]].b[k];
  }
  return 0;
}

static int convex_convex(const Shape* A, const Shape* B, OContact* out, int maxout) {
  SV simplex[4];
  int ns = 0;
  double dist = 0, wa[3], wb[3], n[3], pos[3];
  double ra = shape_radius(A), rb = shape_radius(B);
  int hit = gjk(A, B, simplex, &ns, &dist, wa, wb, ra + rb);
  if (!hit) {
    if (ra + rb <= 0 || dist > ra + rb) return 0;
    /* cores separated but inflated shapes overlap: analytic from the witness points */
    v3_sub(n, wb, wa);
    v3_scl(n, n, 1.0 / dist);
    double pa[3], pb[3];
    v3_addscl(pa, wa, n, ra);
    v3_addscl(pb, wb, n, -rb);
    v3_add(pos, pa, pb);
    v3_scl(pos, pos, 0.5);
    return add_contact(out, 0, maxout, pos, n, dist - ra - rb);
  }
  double depth;
  if (epa(A, B, simplex, ns, &depth, n, wa, wb) != 0) return 0;
  double pa[3], pb[3];
  v3_addscl(pa, wa, n, ra);
  v3_addscl(pb, wb, n, -rb);
  v3_add(pos, pa, pb);
  v3_scl(pos, pos, 0.5);
  return add_contact(out, 0, maxout, pos, n, -depth - ra - rb);
}

/* ------------------------------------------------------------------------------------------------ dispatch */
static void mix_params(const OModel* m, int g1, int g2, OContact* c) {
  /* equal priority everywhere in scope: condim = max, friction = element-wise max, solref/solimp = solmix-weighted */
  int p1 = m->geom_priority[g1], p2 = m->geom_priority[g2];
  double mix;
  if (p1 != p2) {
    int g = p1 > p2 ? g1 : g2;
    c->dim = m->geom_condim[g];
    const double* f = m->geom_friction + 3 * g;
    c->friction[0] = c->friction[1] = f[0]; c->friction[2] = f[1]; c->friction[3] = c->friction[4] = f[2];
    memcpy(c->solref, m->geom_solref + 2 * g, sizeof c->solref);
    memcpy(c->solimp, m->geom_solimp + 5 * g, sizeof c->solimp);
    return;
  }
  c->dim = m->geom_condim[g1] > m->geom_condim[g2] ? m->geom_condim[g1] : m->geom_condim[g2];
  double s1 = m->geom_solmix[g1], s2 = m->geom_solmix[g2];
  if (s1 >= O_MINVAL && s2 >= O_MINVAL) mix = s1 / (s1 + s2);
  else if (s1 < O_MINVAL && s2 < O_MINVAL) mix = 0.5;
  else mix = s1 < O_MINVAL ? 0.0 : 1.0;
  const double *f1 = m->geom_friction + 3 * g1, *f2 = m->geom_friction + 3 * g2;
  double f[3];
  for (int k = 0; k < 3; k++) f[k] = fmax(f1[k], f2[k]);
  c->friction[0] = c->friction[1] = f[0]; c->friction[2] = f[1]; c->friction[3] = c->friction[4] = f[2];
  const double *r1 = m->geom_solref + 2 * g1, *r2 = m->geom_solref + 2 * g2;
  if (r1[0] > 0 && r2[0] > 0)
    for (int k = 0; k < 2; k++) c->solref[k] = mix * r1[k] + (1 - mix) * r2[k];
  else
    for (int k = 0; k < 2; k++) c->solref[k] = fmin(r1[k], r2[k]);
  for (int k = 0; k < 5; k++) c->solimp[k] = mix * m->geom_solimp[5 * g1 + k] + (1 - mix) * m->geom_solimp[5 * g2 + k];
}

int o_collide_pair(const OModel* m, const OData* d, int g1, int g2, OContact* out, int maxout) {
  if (m->geom_type[g1] > m->geom_type[g2]) { int t = g1; g1 = g2; g2 = t; }
  Shape A, B;
  shape_get(m, d, g1, &A);
  shape_get(m, d, g2, &B);
  int t1 = A.type, t2 = B.type, n = 0;
  if (t1 == O_GEOM_PLANE) {
    if (t2 == O_GEOM_SPHERE) n = plane_sphere(&A, &B, out, maxout);
    else if (t2 == O_GEOM_BOX) n = plane_box(&A, &B, out, maxout);
    else if (t2 == O_GEOM_CYLINDER) n = plane_cylinder(&A, &B, out, maxout);
    else if (t2 == O_GEOM_MESH) n = plane_mesh(&A, &B, out, maxout);
    else if (t2 == O_GEOM_CAPSULE) n = plane_capsule(&A, &B, out, maxout);
    else if (t2 == O_GEOM_ELLIPSOID) n = plane_ellipsoid(&A, &B, out, maxout);
    else n = 0;
  } else if (t1 == O_GEOM_SPHERE && t2 == O_GEOM_SPHERE) n = sphere_sphere(&A, &B, out, maxout);
  else if (t1 == O_GEOM_SPHERE && t2 == O_GEOM_BOX) n = sphere_box(&A, &B, out, maxout);
  else if (t1 == O_GEOM_SPHERE && t2 == O_GEOM_CYLINDER) n = sphere_cylinder(&A, &B, out, maxout);
  else if (t1 == O_GEOM_SPHERE && t2 == O_GEOM_CAPSULE) n = sphere_capsule(&A, &B, out, maxout);
  else if (t1 == O_GEOM_CAPSULE && t2 == O_GEOM_CAPSULE) n = capsule_capsule(&A, &B, out, maxout);
  else if (t1 == O_GEOM_BOX && t2 == O_GEOM_BOX) n = box_box(&A, &B, out, maxout);
  else n = convex_convex(&A, &B, out, maxout);
  for (int k = 0; k < n; k++) {
    out[k].geom1 = g1;
    out[k].geom2 = g2;
    mix_params(m, g1, g2, out + k);
    out[k].mu = 0;
    out[k].efc_address = -1;
  }
  return n;
}

void o_collision(const OModel* m, OData* d) {
  d->ncon = 0;
  for (int p = 0; p < m->npair; p++) {
    int g1 = m->pair_geom[2 * p], g2 = m->pair_geom[2 * p + 1];
    int t1 = m->geom_type[g1], t2 = m->geom_type[g2];
    /* bounding-sphere cull (margin = 0 everywhere in scope) */
    if (t1 != O_GEOM_PLANE && t2 != O_GEOM_PLANE) {
      double df[3];
      v3_sub(df, d->geom_xpos + 3 * g1, d->geom_xpos + 3 * g2);
      double bound = m->geom_rbound[g1] + m->geom_rbound[g2];
      if (v3_dot(df, df) > bound * bound) continue;
    } else {
      int gp = t1 == O_GEOM_PLANE ? g1 : g2, go = t1 == O_GEOM_PLANE ? g2 : g1;
      double nrm[3] = COL(d->geom_xmat + 9 * gp, 2), df[3];
      v3_sub(df, d->geom_xpos + 3 * go, d->geom_xpos + 3 * gp);
      if (v3_dot(df, nrm) > m->geom_rbound[go]) continue;
    }
    int room = O_MAXCON - d->ncon;
    if (room <= 0) { d->warn_flags |= 4; break; }
    d->ncon += o_collide_pair(m, d, g1, g2, d->contact + d->ncon, room);
  }
}
