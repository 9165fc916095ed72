// Per-warp collision detection: lane-per-pair bounding-sphere + oriented-box culling over the static pair list,
// lane-per-candidate analytic narrow phase (plane / sphere / box / cylinder, plane_capsule and plane_ellipsoid, sphere_capsule and
// capsule_capsule from the closest points of the cores), warp-cooperative GJK + EPA for
// convex pairs (mesh support scans are split across the 32 lanes).  Contacts come out ordered by pair index.
// Replaces the collision stage of mj_step1 (robosuite/utils/binding_utils.py:1101-1103), SURVEY.md section 8 a1.
#pragma once
#include <cstdio>
#include "b2s_engine.cuh"

template <typename R>
struct Shape {
  int type;
  const R* pos;   // shared memory
  const R* mat;   // shared memory, row-major
  R size[3];
  const R* vert;  // global memory (hull vertices, local frame)
  int nvert;
};

template <typename R>
DEV void shape_from(const DModel<R>& m, const DState<R>& st, int env, int g, const R* gpos, const R* gmat, Shape<R>& s) {
  int k = m.geom_cgid[g];
  s.type = m.geom_type[g];
  s.pos = gpos + 3 * k;
  s.mat = gmat + 9 * k;
  const R* sz = geom_size_of(m, st, g, env);
  s.size[0] = sz[0]; s.size[1] = sz[1]; s.size[2] = sz[2];
  s.vert = nullptr; s.nvert = 0;
  if (s.type == G_MESH) {
    int id = m.geom_dataid[g];
    s.vert = m.mesh_vert + 3 * m.mesh_vertadr[id];
    s.nvert = m.mesh_vertnum[id];
  }
}

template <typename R> DEV void make_frame(R* f) {
  R* x = f; R* y = f + 3; R* z = f + 6;
  v3normalize(x);
  y[0] = 0; y[1] = 0; y[2] = 0;
  if (x[1] < R(0.5) && x[1] > R(-0.5)) y[1] = 1; else y[2] = 1;
  R dt = v3dot(x, y);
  v3addscl(y, y, x, -dt);
  v3normalize(y);
  v3cross(z, x, y);
}

// local contact record: pos(3) normal(3) dist
#define CREC 7
template <typename R> DEV int put(R* out, int n, int maxn, const R* pos, const R* nrm, R dist) {
  if (n >= maxn) return n;
  R* c = out + CREC * n;
  c[0] = pos[0]; c[1] = pos[1]; c[2] = pos[2]; c[3] = nrm[0]; c[4] = nrm[1]; c[5] = nrm[2]; c[6] = dist;
  return n + 1;
}
#define COLV(M, k) {(M)[k], (M)[3 + (k)], (M)[6 + (k)]}

// ---------------------------------------------------------------------------------------------- analytic pairs
template <typename R> DEVN int plane_sphere(const Shape<R>& p, const Shape<R>& s, R* out, int maxn) {
  R n[3] = COLV(p.mat, 2), df[3], pos[3];
  v3sub(df, s.pos, p.pos);
  R dist = v3dot(df, n) - s.size[0];
  if (dist > 0) return 0;
  v3addscl(pos, s.pos, n, -(s.size[0] + R(0.5) * dist));
  return put(out, 0, maxn, pos, n, dist);
}
template <typename R> DEVN int plane_box(const Shape<R>& p, const Shape<R>& b, R* out, int maxn) {
  R n[3] = COLV(p.mat, 2), df[3];
  v3sub(df, b.pos, p.pos);
  R dist = v3dot(df, n);
  int cnt = 0;
  for (int i = 0; i < 8 && cnt < 4; i++) {
    R vec[3] = {(i & 1 ? 1 : -1) * b.size[0], (i & 2 ? 1 : -1) * b.size[1], (i & 4 ? 1 : -1) * b.size[2]};
    R corner[3], pos[3];
    m3mulv(corner, b.mat, vec);
    R ld = v3dot(n, corner);
    if (dist + ld > 0 || ld > 0) continue;
    R cd = dist + ld;
    v3add(pos, b.pos, corner);
    v3addscl(pos, pos, n, -R(0.5) * cd);
    cnt = put(out, cnt, maxn, pos, n, cd);
  }
  return cnt;
}
template <typename R> DEVN int plane_cylinder(const Shape<R>& p, const Shape<R>& c, R* out, int maxn) {
  R n[3] = COLV(p.mat, 2), axis[3] = COLV(c.mat, 2), df[3], vec[3], pos[3];
  R r = c.size[0], h = c.size[1];
  v3sub(df, c.pos, p.pos);
  R dist0 = v3dot(df, n);
  R prjaxis = v3dot(n, axis);
  if (prjaxis > 0) { v3scl(axis, axis, R(-1)); prjaxis = -prjaxis; }
  v3scl(vec, n, R(-1));
  v3addscl(vec, vec, axis, prjaxis);
  R len = v3norm(vec);
  if (len < R(1e-12)) { R x[3] = COLV(c.mat, 0); v3scl(vec, x, r); }
  else v3scl(vec, vec, r / len);
  R prjvec = v3dot(vec, n);
  int cnt = 0;
  R d1 = dist0 + h * prjaxis + prjvec;
  if (d1 > 0) return 0;
  v3addscl(pos, c.pos, axis, h);
  v3add(pos, pos, vec);
  v3addscl(pos, pos, n, -R(0.5) * d1);
  cnt = put(out, cnt, maxn, pos, n, d1);
  R d2 = dist0 - h * prjaxis + prjvec;
  if (d2 <= 0) {
    v3addscl(pos, c.pos, axis, -h);
    v3add(pos, pos, vec);
    v3addscl(pos, pos, n, -R(0.5) * d2);
    cnt = put(out, cnt, maxn, pos, n, d2);
  }
  R side[3];
  v3cross(side, vec, axis);
  v3normalize(side);
  v3scl(side, side, r * R(0.8660254037844386));
  for (int k = 0; k < 2; k++) {
    R off[3];
    v3scl(off, vec, R(-0.5));
    v3addscl(off, off, side, k ? R(-1) : R(1));
    R d3 = dist0 + h * prjaxis + v3dot(off, n);
    if (d3 > 0) continue;
    v3addscl(pos, c.pos, axis, h);
    v3add(pos, pos, off);
    v3addscl(pos, pos, n, -R(0.5) * d3);
    cnt = put(out, cnt, maxn, pos, n, d3);
  }
  return cnt;
}
// one contact per penetrating end sphere of the segment, + end first
template <typename R> DEVN int plane_capsule(const Shape<R>& p, const Shape<R>& c, R* out, int maxn) {
  R n[3] = COLV(p.mat, 2), axis[3] = COLV(c.mat, 2), df[3], pos[3];
  R r = c.size[0], h = c.size[1];
  v3sub(df, c.pos, p.pos);
  R dist0 = v3dot(df, n), prj = h * v3dot(n, axis);
  int cnt = 0;
  for (int k = 0; k < 2; k++) {
    R sg = k ? R(-1) : R(1), dist = dist0 + sg * prj - r;
    if (dist > 0) continue;
    v3addscl(pos, c.pos, axis, sg * h);
    v3addscl(pos, pos, n, -(r + R(0.5) * dist));
    cnt = put(out, cnt, maxn, pos, n, dist);
  }
  return cnt;
}
// support point of the ellipsoid along -n: local -S^2 nl / |S nl|
template <typename R> DEVN int plane_ellipsoid(const Shape<R>& p, const Shape<R>& e, R* out, int maxn) {
  R n[3] = COLV(p.mat, 2), nl[3], df[3], sp[3], w[3], pos[3];
  m3mulTv(nl, e.mat, n);
  R t[3] = {nl[0] * e.size[0], nl[1] * e.size[1], nl[2] * e.size[2]};
  R len = v3norm(t);
  for (int k = 0; k < 3; k++) sp[k] = -t[k] * e.size[k] / len;
  m3mulv(w, e.mat, sp);
  v3add(w, w, e.pos);
  v3sub(df, w, p.pos);
  R dist = v3dot(df, n);
  if (dist > 0) return 0;
  v3addscl(pos, w, n, -R(0.5) * dist);
  return put(out, 0, maxn, pos, n, dist);
}
template <typename R> DEVN int plane_mesh(const Shape<R>& p, const Shape<R>& s, R* out, int maxn) {
  R n[3] = COLV(p.mat, 2), nl[3], df[3];
  m3mulTv(nl, s.mat, n);
  v3sub(df, s.pos, p.pos);
  R base = v3dot(df, n);
  int chosen[4], cnt = 0, nc = 0;
  for (int round = 0; round < 4; round++) {
    int best = -1;
    R bestscore = -Lim<R>::big();
    for (int i = 0; i < s.nvert; i++) {
      R v[3] = {s.vert[3 * i], s.vert[3 * i + 1], s.vert[3 * i + 2]};
      R dist = base + v3dot(v, nl);
      if (dist > 0) continue;
      R score;
      if (round == 0) score = -dist;
      else {
        score = Lim<R>::big();
        int dup = 0;
        for (int k = 0; k < nc; k++) {
          R u[3] = {s.vert[3 * chosen[k]], s.vert[3 * chosen[k] + 1], s.vert[3 * chosen[k] + 2]}, d3[3];
          v3sub(d3, v, u);
          R dd = v3dot(d3, d3);
          if (chosen[k] == i) dup = 1;
          if (dd < score) score = dd;
        }
        if (dup || score < R(1e-10)) continue;
      }
      if (score > bestscore) { bestscore = score; best = i; }
    }
    if (best < 0) break;
    chosen[nc++] = best;
    R v[3] = {s.vert[3 * best], s.vert[3 * best + 1], s.vert[3 * best + 2]}, w[3], pos[3];
    m3mulv(w, s.mat, v);
    v3add(w, w, s.pos);
    R dist = base + v3dot(v, nl);
    v3addscl(pos, w, n, -R(0.5) * dist);
    cnt = put(out, cnt, maxn, pos, n, dist);
  }
  return cnt;
}
template <typename R> DEVN int sphere_sphere(const Shape<R>& a, const Shape<R>& b, R* out, int maxn) {
  R n[3], pos[3];
  v3sub(n, b.pos, a.pos);
  R len = v3norm(n), dist = len - a.size[0] - b.size[0];
  if (dist > 0) return 0;
  if (len < R(1e-12)) v3set(n, R(1), R(0), R(0)); else v3scl(n, n, R(1) / len);
  v3addscl(pos, a.pos, n, a.size[0] + R(0.5) * dist);
  return put(out, 0, maxn, pos, n, dist);
}
template <typename R> DEVN int sphere_box(const Shape<R>& s, const Shape<R>& b, R* out, int maxn) {
  R df[3], c[3], cl[3], n[3], pos[3];
  v3sub(df, s.pos, b.pos);
  m3mulTv(c, b.mat, df);
  int inside = 1;
  for (int k = 0; k < 3; k++) {
    cl[k] = r_min(r_max(c[k], -b.size[k]), b.size[k]);
    if (cl[k] != c[k]) inside = 0;
  }
  R dist, r = s.size[0];
  if (inside) {
    int ax = 0;
    R best = Lim<R>::big();
    for (int k = 0; k < 3; k++) {
      R dd = b.size[k] - r_abs(c[k]);
      if (dd < best) { best = dd; ax = k; }
    }
    R nl[3] = {0, 0, 0};
    nl[ax] = c[ax] >= 0 ? R(-1) : R(1);
    m3mulv(n, b.mat, nl);
    dist = -best - r;
  } else {
    R el[3];
    v3sub(el, cl, c);
    R len = v3norm(el);
    dist = len - r;
    if (dist > 0) return 0;
    v3scl(el, el, R(1) / len);
    m3mulv(n, b.mat, el);
  }
  v3addscl(pos, s.pos, n, r + R(0.5) * dist);
  return put(out, 0, maxn, pos, n, dist);
}
template <typename R> DEVN int sphere_cylinder(const Shape<R>& s, const Shape<R>& c, R* out, int maxn) {
  R df[3], p[3], q[3], n[3], pos[3];
  R Rc = c.size[0], h = c.size[1], r = s.size[0];
  v3sub(df, s.pos, c.pos);
  m3mulTv(p, c.mat, df);
  R rho = r_sqrt(p[0] * p[0] + p[1] * p[1]);
  R dist;
  if (rho <= Rc && r_abs(p[2]) <= h) {
    R dside = Rc - rho, dcap = h - r_abs(p[2]);
    R nl[3] = {0, 0, 0};
    if (dcap < dside) { nl[2] = p[2] >= 0 ? R(-1) : R(1); dist = -dcap - r; }
    else if (rho < R(1e-12)) { nl[0] = R(1); dist = -dside - r; }  // on the axis, nearer the side: a fixed perpendicular
    else { nl[0] = -p[0] / rho; nl[1] = -p[1] / rho; dist = -dside - r; }
    m3mulv(n, c.mat, nl);
  } else {
    R sc = rho > Rc ? Rc / rho : R(1);
    q[0] = p[0] * sc; q[1] = p[1] * sc; q[2] = r_min(r_max(p[2], -h), h);
    R el[3];
    v3sub(el, q, p);
    R len = v3norm(el);
    dist = len - r;
    if (dist > 0) return 0;
    v3scl(el, el, R(1) / len);
    m3mulv(n, c.mat, el);
  }
  v3addscl(pos, s.pos, n, r + R(0.5) * dist);
  return put(out, 0, maxn, pos, n, dist);
}

// closest points of the segments a + s u (|s| <= ha) and b + t v (|t| <= hb), u and v unit; parallel segments take s = 0
template <typename R> DEV void seg_seg(const R* a, const R* u, R ha, const R* b, const R* v, R hb, R* p, R* q) {
  R r[3];
  v3sub(r, a, b);
  R uv = v3dot(u, v), c = v3dot(u, r), f = v3dot(v, r), den = 1 - uv * uv;
  R s = den > R(1e-12) ? r_min(r_max((uv * f - c) / den, -ha), ha) : R(0);
  R t = uv * s + f;
  if (t < -hb || t > hb) {
    t = r_min(r_max(t, -hb), hb);
    s = r_min(r_max(uv * t - c, -ha), ha);
  }
  v3addscl(p, a, u, s);
  v3addscl(q, b, v, t);
}
// contact of two inflated cores with closest points p (on A's core) and q (on B's); nfb: the normal where the cores meet.  fp32 takes
// core distances below 1e-5 as meeting: at metre-scale coordinates the rounding of p - q is ~1e-7 and its direction is noise
template <typename R> DEV int core_contact(const R* p, const R* q, R ra, R rb, const R* nfb, R* out, int maxn) {
  R n[3], pos[3];
  v3sub(n, q, p);
  R len = v3norm(n), dist = len - ra - rb;
  if (dist > 0) return 0;
  if (len < (sizeof(R) == 4 ? R(1e-5) : R(1e-12))) v3copy(n, nfb); else v3scl(n, n, R(1) / len);
  v3addscl(pos, p, n, ra + R(0.5) * dist);
  return put(out, 0, maxn, pos, n, dist);
}
template <typename R> DEVN int sphere_capsule(const Shape<R>& s, const Shape<R>& c, R* out, int maxn) {
  R axis[3] = COLV(c.mat, 2), nfb[3] = COLV(c.mat, 0), df[3], q[3];
  v3sub(df, s.pos, c.pos);
  v3addscl(q, c.pos, axis, r_min(r_max(v3dot(df, axis), -c.size[1]), c.size[1]));
  return core_contact(s.pos, q, s.size[0], c.size[0], nfb, out, maxn);  // centre on the segment: a fixed perpendicular
}
template <typename R> DEVN int capsule_capsule(const Shape<R>& A, const Shape<R>& B, R* out, int maxn) {
  R u[3] = COLV(A.mat, 2), v[3] = COLV(B.mat, 2), p[3], q[3], nfb[3], df[3];
  seg_seg(A.pos, u, A.size[1], B.pos, v, B.size[1], p, q);
  // intersecting cores: crossing axes take their common perpendicular, pointing along the centre difference; collinear ones a fixed
  // perpendicular of A's axis
  v3cross(nfb, u, v);
  R len = v3norm(nfb);
  if (len > R(1e-6)) {
    v3sub(df, B.pos, A.pos);
    v3scl(nfb, nfb, (v3dot(nfb, df) < 0 ? R(-1) : R(1)) / len);
  } else v3set(nfb, A.mat[0], A.mat[3], A.mat[6]);
  return core_contact(p, q, A.size[0], B.size[0], nfb, out, maxn);
}

// keep the part of the polygon with sign*coord[axis] <= lim
template <typename R> DEV int clip_poly(R (*poly)[2], int n, int axis, R lim, R sign) {
  R outp[16][2];
  int no = 0;
  for (int i = 0; i < n; i++) {
    const R* a = poly[i];
    const R* b = poly[(i + 1) % n];
    R da = sign * a[axis] - lim, db = sign * b[axis] - lim;
    if (da <= 0) { outp[no][0] = a[0]; outp[no][1] = a[1]; no++; }
    if ((da < 0 && db > 0) || (da > 0 && db < 0)) {
      R t = da / (da - db);
      outp[no][0] = a[0] + t * (b[0] - a[0]);
      outp[no][1] = a[1] + t * (b[1] - a[1]);
      no++;
    }
    if (no >= 15) break;
  }
  for (int i = 0; i < no; i++) { poly[i][0] = outp[i][0]; poly[i][1] = outp[i][1]; }
  return no;
}

template <typename R> DEVN int box_box(const Shape<R>& A, const Shape<R>& B, R* out, int maxn) {
  R Aax[3][3], Bax[3][3], T[3];
  for (int k = 0; k < 3; k++) {
    Aax[k][0] = A.mat[k]; Aax[k][1] = A.mat[3 + k]; Aax[k][2] = A.mat[6 + k];
    Bax[k][0] = B.mat[k]; Bax[k][1] = B.mat[3 + k]; Bax[k][2] = B.mat[6 + k];
  }
  v3sub(T, B.pos, A.pos);
  R best = Lim<R>::big(), n[3] = {0, 0, 0};
  int code = -1;
  for (int k = 0; k < 6; k++) {
    const R* Lx = k < 3 ? Aax[k] : Bax[k - 3];
    R ra = 0, rb = 0;
    for (int i = 0; i < 3; i++) { ra += A.size[i] * r_abs(v3dot(Aax[i], Lx)); rb += B.size[i] * r_abs(v3dot(Bax[i], Lx)); }
    R tl = v3dot(T, Lx), ov = ra + rb - r_abs(tl);
    if (ov < 0) return 0;
    if (ov + R(1e-5) < best) { best = ov; code = k; v3scl(n, Lx, tl >= 0 ? R(1) : R(-1)); }
  }
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      R Lx[3];
      v3cross(Lx, Aax[i], Bax[j]);
      R len = v3norm(Lx);
      if (len < R(1e-6)) continue;
      v3scl(Lx, Lx, R(1) / len);
      R ra = 0, rb = 0;
      for (int k = 0; k < 3; k++) { ra += A.size[k] * r_abs(v3dot(Aax[k], Lx)); rb += B.size[k] * r_abs(v3dot(Bax[k], Lx)); }
      R tl = v3dot(T, Lx), ov = ra + rb - r_abs(tl);
      if (ov < 0) return 0;
      if (ov * R(1.05) + R(1e-5) < best) { best = ov * R(1.05) + R(1e-5); code = 6 + 3 * i + j; v3scl(n, Lx, tl >= 0 ? R(1) : R(-1)); }
    }
  if (code < 0) return 0;
  if (code >= 6) {
    int i = (code - 6) / 3, j = (code - 6) % 3;
    R pa[3], pb[3];
    v3copy(pa, A.pos);
    v3copy(pb, B.pos);
    for (int k = 0; k < 3; k++) {
      if (k != i) v3addscl(pa, pa, Aax[k], (v3dot(Aax[k], n) > 0 ? R(1) : R(-1)) * A.size[k]);
      if (k != j) v3addscl(pb, pb, Bax[k], (v3dot(Bax[k], n) > 0 ? R(-1) : R(1)) * B.size[k]);
    }
    const R* u = Aax[i];
    const R* v = Bax[j];
    R w[3];
    v3sub(w, pa, pb);
    R uv = v3dot(u, v), uw = v3dot(u, w), vw = v3dot(v, w), den = 1 - uv * uv;
    R s = den > R(1e-12) ? (uv * vw - uw) / den : R(0), t = den > R(1e-12) ? (vw - uv * uw) / den : R(0);
    s = r_min(r_max(s, -A.size[i]), A.size[i]);
    t = r_min(r_max(t, -B.size[j]), B.size[j]);
    R qa[3], qb[3], pos[3], dv[3];
    v3addscl(qa, pa, u, s);
    v3addscl(qb, pb, v, t);
    v3add(pos, qa, qb);
    v3scl(pos, pos, R(0.5));
    v3sub(dv, qb, qa);
    R dist = v3dot(dv, n);
    if (dist > 0) return 0;
    return put(out, 0, maxn, pos, n, dist);
  }
  const Shape<R>& Rf = code < 3 ? A : B;
  const Shape<R>& Ic = code < 3 ? B : A;
  R (*Rax)[3] = code < 3 ? Aax : Bax;
  R (*Iax)[3] = code < 3 ? Bax : Aax;
  int ax = code < 3 ? code : code - 3;
  R nr[3];
  v3scl(nr, n, code < 3 ? R(1) : R(-1));
  int iu = (ax + 1) % 3, iv = (ax + 2) % 3;
  int ia = 0;
  R bestd = -1;
  for (int k = 0; k < 3; k++) {
    R dd = r_abs(v3dot(Iax[k], nr));
    if (dd > bestd) { bestd = dd; ia = k; }
  }
  R sgn = v3dot(Iax[ia], nr) > 0 ? R(-1) : R(1);
  R fc[3], rc[3];
  v3addscl(fc, Ic.pos, Iax[ia], sgn * Ic.size[ia]);
  int ju = (ia + 1) % 3, jv = (ia + 2) % 3;
  v3addscl(rc, Rf.pos, nr, Rf.size[ax]);
  R poly[16][2], hgt[4];
  const int sg[4][2] = {{1, 1}, {-1, 1}, {-1, -1}, {1, -1}};
  for (int k = 0; k < 4; k++) {
    R cn[3], rel[3];
    v3copy(cn, fc);
    v3addscl(cn, cn, Iax[ju], R(sg[k][0]) * Ic.size[ju]);
    v3addscl(cn, cn, Iax[jv], R(sg[k][1]) * Ic.size[jv]);
    v3sub(rel, cn, rc);
    poly[k][0] = v3dot(rel, Rax[iu]);
    poly[k][1] = v3dot(rel, Rax[iv]);
    hgt[k] = v3dot(rel, nr);
  }
  R e1[2] = {poly[1][0] - poly[0][0], poly[1][1] - poly[0][1]}, e2[2] = {poly[3][0] - poly[0][0], poly[3][1] - poly[0][1]};
  R det = e1[0] * e2[1] - e1[1] * e2[0];
  R x0[2] = {poly[0][0], poly[0][1]};
  R h0 = hgt[0], dh1 = hgt[1] - hgt[0], dh2 = hgt[3] - hgt[0];
  int np = 4;
  np = clip_poly(poly, np, 0, Rf.size[iu], R(1));
  np = clip_poly(poly, np, 0, Rf.size[iu], R(-1));
  np = clip_poly(poly, np, 1, Rf.size[iv], R(1));
  np = clip_poly(poly, np, 1, Rf.size[iv], R(-1));
  int cnt = 0;
  for (int k = 0; k < np && cnt < 8; k++) {
    R hh;
    if (r_abs(det) > R(1e-14)) {
      R dx = poly[k][0] - x0[0], dy = poly[k][1] - x0[1];
      R a = (dx * e2[1] - dy * e2[0]) / det, b = (e1[0] * dy - e1[1] * dx) / det;
      hh = h0 + a * dh1 + b * dh2;
    } else hh = h0;
    if (hh > 0) continue;
    R pnt[3], pos[3];
    v3copy(pnt, rc);
    v3addscl(pnt, pnt, Rax[iu], poly[k][0]);
    v3addscl(pnt, pnt, Rax[iv], poly[k][1]);
    v3addscl(pnt, pnt, nr, hh);
    v3addscl(pos, pnt, nr, -R(0.5) * hh);
    cnt = put(out, cnt, maxn, pos, n, hh);
  }
  return cnt;
}

// ---------------------------------------------------------------------------------------------- GJK / EPA (warp)
// support point of the core shape in world direction dir; mesh scans are split across lanes, result warp-uniform
// (the direction travels by value: with a pointer to a caller-side local array nvcc 12.9 merged the stack slots of the
//  direction and of its negation inside epa(), so one of the two supports was evaluated in the wrong direction)
template <typename R> DEVN void support_w(const Shape<R>& s, R dx, R dy, R dz, R* out, int lane) {
  R l[3], pnt[3] = {0, 0, 0};
  const R dir[3] = {dx, dy, dz};
  m3mulTv(l, s.mat, dir);
  switch (s.type) {
    case G_BOX:
      pnt[0] = l[0] >= 0 ? s.size[0] : -s.size[0];
      pnt[1] = l[1] >= 0 ? s.size[1] : -s.size[1];
      pnt[2] = l[2] >= 0 ? s.size[2] : -s.size[2];
      break;
    case G_CYLINDER: {
      R nn = r_sqrt(l[0] * l[0] + l[1] * l[1]);
      if (nn > R(1e-12)) { pnt[0] = l[0] / nn * s.size[0]; pnt[1] = l[1] / nn * s.size[0]; }
      pnt[2] = l[2] >= 0 ? s.size[1] : -s.size[1];
      break;
    }
    case G_CAPSULE: pnt[2] = l[2] >= 0 ? s.size[1] : -s.size[1]; break;
    case G_ELLIPSOID: {
      R t[3] = {l[0] * s.size[0], l[1] * s.size[1], l[2] * s.size[2]};
      R nn = v3norm(t);
      if (nn > R(1e-12)) { pnt[0] = t[0] * s.size[0] / nn; pnt[1] = t[1] * s.size[1] / nn; pnt[2] = t[2] * s.size[2] / nn; }
      break;
    }
    case G_MESH: {
      R best = -Lim<R>::big();
      int bi = 0;  // vertex 0 when no comparison succeeds (a NaN direction), never an index past the hull
      // generic loads: the work-list convex kernel stages the hull vertices of a pair that needs real GJK / EPA work in shared memory
      const R* vt = s.vert;
      for (int i = lane; i < s.nvert; i += 32) {
        R v = vt[3 * i] * l[0] + vt[3 * i + 1] * l[1] + vt[3 * i + 2] * l[2];
        if (v > best) { best = v; bi = i; }
      }
      warp_argmax(best, bi);
      pnt[0] = vt[3 * bi]; pnt[1] = vt[3 * bi + 1]; pnt[2] = vt[3 * bi + 2];
      break;
    }
    default: break;  // sphere: core = centre
  }
  m3mulv(out, s.mat, pnt);
  v3add(out, out, s.pos);
}
template <typename R> DEV R shape_radius(const Shape<R>& s) { return (s.type == G_SPHERE || s.type == G_CAPSULE) ? s.size[0] : R(0); }

template <typename R> struct SV { R w[3], a[3], b[3]; };

template <typename R> DEV void sv_support(const Shape<R>& A, const Shape<R>& B, const R* dir, SV<R>& o, int lane) {
  const R dx = dir[0], dy = dir[1], dz = dir[2];
  support_w(A, dx, dy, dz, o.a, lane);
  support_w(B, -dx, -dy, -dz, o.b, lane);
  v3sub(o.w, o.a, o.b);
}

// ---- GJK simplex in SHARED memory ----------------------------------------------------------------------------------------------
// 4 entries x 9 reals (w = a - b, a, b).  Every lane of the warp runs the same scalar code on the same values; as per-thread arrays
// the simplex (dynamically indexed) lived in local memory - 32 redundant copies behind an L1 that is a few KB beside the phase
// kernels' shared memory - and a 64-iteration GJK on a curved shape took up to 0.9 ms (tools/probe_instr.py "slow_items").  One copy
// per warp in shared memory: loads are broadcasts, stores go through lane 0.
template <typename R> DEV void sx_load(const R* sx, int k, SV<R>& o) {
  const R* p = sx + 9 * k;
#pragma unroll
  for (int e = 0; e < 3; e++) { o.w[e] = p[e]; o.a[e] = p[3 + e]; o.b[e] = p[6 + e]; }
}
template <typename R> DEV void sx_store(R* sx, int k, const SV<R>& v, int lane) {
  __syncwarp();
  if (lane == 0) {
    R* p = sx + 9 * k;
#pragma unroll
    for (int e = 0; e < 3; e++) { p[e] = v.w[e]; p[3 + e] = v.a[e]; p[6 + e] = v.b[e]; }
  }
  __syncwarp();
}
// keep entries i0, i1, i2 (the first n of them) as the new entries 0..n-1
template <typename R> DEV void sx_select(R* sx, int n, int i0, int i1, int i2, int lane) {
  SV<R> t0, t1, t2;
  sx_load(sx, i0, t0);
  if (n > 1) sx_load(sx, i1, t1);
  if (n > 2) sx_load(sx, i2, t2);
  if (i0 != 0) sx_store(sx, 0, t0, lane);
  if (n > 1 && i1 != 1) sx_store(sx, 1, t1, lane);
  if (n > 2 && i2 != 2) sx_store(sx, 2, t2, lane);
}

// closest point of the triangle (a, b, c) to the origin: which of the three vertices support it (idx, n of them) and their weights
template <typename R> DEV void tri_closest(const R* a, const R* b, const R* c, int& n, int* idx, R* lam) {
  R ab[3], ac[3];
  v3sub(ab, b, a); v3sub(ac, c, a);
  idx[0] = 0; idx[1] = 1; idx[2] = 2; lam[0] = 1; lam[1] = 0; lam[2] = 0;
  R d1 = -v3dot(ab, a), d2 = -v3dot(ac, a);
  if (d1 <= 0 && d2 <= 0) { n = 1; return; }
  R d3 = -v3dot(ab, b), d4 = -v3dot(ac, b);
  if (d3 >= 0 && d4 <= d3) { idx[0] = 1; n = 1; return; }
  R vc = d1 * d4 - d3 * d2;
  if (vc <= 0 && d1 >= 0 && d3 <= 0) { R v = d1 / (d1 - d3); n = 2; lam[0] = 1 - v; lam[1] = v; return; }
  R d5 = -v3dot(ab, c), d6 = -v3dot(ac, c);
  if (d6 >= 0 && d5 <= d6) { idx[0] = 2; n = 1; return; }
  R vb = d5 * d2 - d1 * d6;
  if (vb <= 0 && d2 >= 0 && d6 <= 0) { R w = d2 / (d2 - d6); idx[1] = 2; n = 2; lam[0] = 1 - w; lam[1] = w; return; }
  R va = d3 * d6 - d5 * d4;
  if (va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0) {
    R w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
    idx[0] = 1; idx[1] = 2; n = 2; lam[0] = 1 - w; lam[1] = w; return;
  }
  R den = R(1) / (va + vb + vc);
  n = 3;
  lam[1] = vb * den; lam[2] = vc * den; lam[0] = 1 - lam[1] - lam[2];
}

template <typename R> DEV void closest_seg(R* sx, int& n, R* lam, int lane) {
  R ab[3];
  const R *s0 = sx, *s1 = sx + 9;
  v3sub(ab, s1, s0);
  R den = v3dot(ab, ab);
  R t = den > 0 ? -v3dot(s0, ab) / den : R(0);
  if (t <= 0) { n = 1; lam[0] = 1; }
  else if (t >= 1) { sx_select(sx, 1, 1, 0, 0, lane); n = 1; lam[0] = 1; }
  else { lam[0] = 1 - t; lam[1] = t; }
}
template <typename R> DEV void closest_tri(R* sx, int& n, R* lam, int lane) {
  R a[3] = {sx[0], sx[1], sx[2]}, b[3] = {sx[9], sx[10], sx[11]}, c[3] = {sx[18], sx[19], sx[20]};
  int idx[3];
  R l3[3];
  tri_closest(a, b, c, n, idx, l3);
  sx_select(sx, n, idx[0], idx[1], idx[2], lane);
  for (int k = 0; k < n; k++) lam[k] = l3[k];
}
template <typename R> DEV R orient3(const R* a, const R* b, const R* c, const R* d) {
  R ab[3], ac[3], ad[3], cr[3];
  v3sub(ab, b, a); v3sub(ac, c, a); v3sub(ad, d, a);
  v3cross(cr, ab, ac);
  return v3dot(cr, ad);
}
template <typename R> DEVN int closest_tet(R* sx, int& n, R* lam, int lane) {
  R w4[4][3];
#pragma unroll
  for (int k = 0; k < 4; k++) { w4[k][0] = sx[9 * k]; w4[k][1] = sx[9 * k + 1]; w4[k][2] = sx[9 * k + 2]; }
  R zero[3] = {0, 0, 0};
  R bestd = Lim<R>::big();
  R bestlam[3] = {0, 0, 0};
  int bestn = 0, outside = 0, bi0 = 0, bi1 = 0, bi2 = 0;
  const R tiny = R(1e-30);
#pragma unroll
  for (int f = 0; f < 4; f++) {
    // faces (0,1,2) (0,1,3) (0,2,3) (1,2,3), opposite vertices 3 2 1 0
    const int f0 = f == 3 ? 1 : 0, f1 = f < 2 ? 1 : 2, f2 = f == 0 ? 2 : 3, op = 3 - f;
    R so = orient3(w4[f0], w4[f1], w4[f2], zero);
    R sd = orient3(w4[f0], w4[f1], w4[f2], w4[op]);
    if (r_abs(sd) < tiny) outside = 1;
    if (r_abs(sd) >= tiny && so * sd > 0) continue;
    outside = 1;
    int tn, idx[3];
    R tl[3];
    tri_closest(w4[f0], w4[f1], w4[f2], tn, idx, tl);
    // (selects instead of indexing by idx[]: the vertex array stays in registers)
    R pp[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 3; k++)
      if (k < tn) {
        const int j = idx[k];
#pragma unroll
        for (int e = 0; e < 3; e++) pp[e] += (j == 0 ? w4[f0][e] : (j == 1 ? w4[f1][e] : w4[f2][e])) * tl[k];
      }
    R dd = v3dot(pp, pp);
    if (dd < bestd) {
      bestd = dd; bestn = tn;
      bi0 = idx[0] == 0 ? f0 : (idx[0] == 1 ? f1 : f2);
      bi1 = tn > 1 ? (idx[1] == 0 ? f0 : (idx[1] == 1 ? f1 : f2)) : 0;
      bi2 = tn > 2 ? (idx[2] == 0 ? f0 : (idx[2] == 1 ? f1 : f2)) : 0;
#pragma unroll
      for (int k = 0; k < 3; k++) bestlam[k] = tl[k];
    }
  }
  if (!outside) return 1;
  n = bestn;
  sx_select(sx, bestn, bi0, bi1, bi2, lane);
  for (int k = 0; k < bestn; k++) lam[k] = bestlam[k];
  return 0;
}

// the pair's remembered separating direction into cv, or false when there is none: a zero entry, or one that is not a direction -
// the cache travels in snapshot rows, which may come from a file, and an infinite component would make every support comparison
// fail (0 * inf).  |c|^2 finite also keeps M^T c and the support products finite.
template <typename R> DEV bool warm_direction(const R* cache, R* cv) {
  cv[0] = cache[0]; cv[1] = cache[1]; cv[2] = cache[2];
  const R c2 = v3dot(cv, cv);
  return c2 > R(1e-12) && isfinite(c2);
}

// returns 1 if the cores overlap (simplex valid), else 0 with dist / witnesses.  sx: the warp's simplex area in shared memory (36 reals)
template <typename R>
DEVN int gjk(const Shape<R>& A, const Shape<R>& B, R* sx, int& ns, R& dist, R* wa, R* wb, R cutoff, int lane, R* cache = nullptr) {
  const R tol_vv = sizeof(R) == 4 ? R(1e-16) : R(1e-24);
  const R tol_rel = sizeof(R) == 4 ? R(1e-6) : R(1e-12);
  R v[3], nv[3];
  v3sub(v, A.pos, B.pos);
  if (v3dot(v, v) < R(1e-20)) v3set(v, R(1), R(0), R(0));
  if (cache) {  // separating direction found for this pair on the previous substep (temporal coherence)
    R cv[3];
    if (warm_direction(cache, cv)) v3copy(v, cv);
  }
  int n = 0;
  R lam[4] = {1, 0, 0, 0};
  v3scl(nv, v, R(-1));
  SV<R> w;
  sv_support(A, B, nv, w, lane);
  sx_store(sx, 0, w, lane);
  n = 1;
  if (cache && cutoff >= 0) {  // does the remembered direction still separate the pair?  (one support pair, no iteration)
    R vv0 = v3dot(v, v), vw0 = v3dot(v, w.w);
    if (vw0 > 0 && vw0 * vw0 > cutoff * cutoff * vv0) { dist = cutoff + 1; ns = 1; return 0; }
  }
  v3copy(v, w.w);
  // iteration cap: 64 in fp64 (the oracle's); the fp32 build stops at 32 - its relative convergence test (1e-6) sits at the edge of
  // fp32 resolution, so touching / grazing pairs of curved shapes never pass it and churned through all 64 iterations at their
  // rounding floor (the 300-400 us work items that set the length of half of the narrow-phase launches: profiles/r02_summary.md)
  const int max_it = sizeof(R) == 4 ? 32 : 64;
  for (int it = 0; it < max_it; it++) {
    R vv = v3dot(v, v);
    if (vv < tol_vv) { ns = n; if (cache && lane == 0) { cache[0] = 0; cache[1] = 0; cache[2] = 0; } return 1; }
    v3scl(nv, v, R(-1));
    sv_support(A, B, nv, w, lane);
    R vw = v3dot(v, w.w);
    if (cutoff >= 0 && vw > 0 && vw * vw > cutoff * cutoff * vv) {
      dist = cutoff + 1; ns = n;
      if (cache && lane == 0) { cache[0] = v[0]; cache[1] = v[1]; cache[2] = v[2]; }
      return 0;
    }
    if (vv - vw <= tol_rel * vv) break;
    int dup = 0;
    for (int k = 0; k < n; k++) {
      R e3[3];
      v3sub(e3, sx + 9 * k, w.w);
      if (v3dot(e3, e3) < tol_vv) dup = 1;
    }
    if (dup) break;
    sx_store(sx, n, w, lane);
    n++;
    if (n == 2) closest_seg(sx, n, lam, lane);
    else if (n == 3) closest_tri(sx, n, lam, lane);
    else if (closest_tet(sx, n, lam, lane)) { ns = 4; if (cache && lane == 0) { cache[0] = 0; cache[1] = 0; cache[2] = 0; } return 1; }
    v3set(v, R(0), R(0), R(0));
    for (int k = 0; k < n; k++) v3addscl(v, v, sx + 9 * k, lam[k]);
  }
  ns = n;
  dist = v3norm(v);
  if (cache && lane == 0) { cache[0] = v[0]; cache[1] = v[1]; cache[2] = v[2]; }
  v3set(wa, R(0), R(0), R(0));
  v3set(wb, R(0), R(0), R(0));
  for (int k = 0; k < n; k++) { v3addscl(wa, wa, sx + 9 * k + 3, lam[k]); v3addscl(wb, wb, sx + 9 * k + 6, lam[k]); }
  return 0;
}

#define EPA_MAXV 96   // polytope capacity (same numbers in the oracle: oracle/o_collide.c)
#define EPA_MAXF 192
// words of the EPA work area: vertices 9 x maxv, face planes 4 x maxf, packed face ids maxf, horizon edge list 64, spare 8, and - its
// last 40 words - the GJK simplex (4 x 9)
#define EPA_AREA_WORDS(maxv, maxf) ((9 * (maxv) + 5 * (maxf) + 64 + 8 + 40 + 3) & ~3)
#define EPA_SIMPLEX(scratch, maxv, maxf) ((scratch) + EPA_AREA_WORDS(maxv, maxf) - 40)
// EPA polytope lives in this warp's scratch: V[EPA_MAXV][9], Fn[EPA_MAXF][4] (normal, dist), Fi[EPA_MAXF] packed ids
template <typename R>
DEVN int epa(const Shape<R>& A, const Shape<R>& B, R* sx, int ns, R& depth, R* normal, R* wa, R* wb, R* scratch, int lane,
             int maxv = EPA_MAXV, int maxf = EPA_MAXF) {
  // polytope capacity: (EPA_MAXV, EPA_MAXF) inside the fused kernel's scratch, larger in the work-list convex kernel
  R* V = scratch;
  R* Fn = V + 9 * maxv;
  int* Fi = reinterpret_cast<int*>(Fn + 4 * maxf);
  int* edges = Fi + maxf;  // horizon edge list (64 entries) - in the work area, NOT a per-thread array: a dynamically indexed local
                           // array lives in local memory, and the serial edge search on it was most of a deep EPA's 300 us
  int nV = 0, nF = 0;
  nV = ns;  // the simplex (shared memory, sx) is completed to a tetrahedron in place
  const R dirs[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
  if (nV == 1) {
    for (int k = 0; k < 6 && nV < 2; k++) {
      SV<R> w;
      sv_support(A, B, dirs[k], w, lane);
      R e3[3];
      v3sub(e3, w.w, sx);
      if (v3dot(e3, e3) > R(1e-12)) { sx_store(sx, nV, w, lane); nV++; }
    }
  }
  if (nV == 2) {
    R ab[3];
    v3sub(ab, sx + 9, sx);
    for (int k = 0; k < 6 && nV < 3; k++) {
      R dir[3];
      v3cross(dir, ab, dirs[k]);
      if (v3dot(dir, dir) < R(1e-12) * v3dot(ab, ab)) continue;
      SV<R> w;
      sv_support(A, B, dir, w, lane);
      R e3[3], cr[3];
      v3sub(e3, w.w, sx);
      v3cross(cr, ab, e3);
      if (v3dot(cr, cr) > R(1e-12) * v3dot(ab, ab) * v3dot(ab, ab)) { sx_store(sx, nV, w, lane); nV++; }
    }
  }
  if (nV == 3) {
    R ab[3], ac[3], nrm[3];
    v3sub(ab, sx + 9, sx);
    v3sub(ac, sx + 18, sx);
    v3cross(nrm, ab, ac);
    for (int s = 0; s < 2 && nV < 4; s++) {
      R dir[3];
      v3scl(dir, nrm, s ? R(-1) : R(1));
      SV<R> w;
      sv_support(A, B, dir, w, lane);
      R e3[3];
      v3sub(e3, w.w, sx);
      if (r_abs(v3dot(e3, nrm)) > R(1e-7) * v3dot(nrm, nrm)) { sx_store(sx, nV, w, lane); nV++; }
    }
  }
  if (nV < 4) return -1;
  const bool flip = orient3(sx, sx + 9, sx + 18, sx + 27) > 0;  // entries 0 and 1 swap
  __syncwarp();
  if (lane == 0)
    for (int k = 0; k < 4; k++) {
      const R* src = sx + 9 * (flip && k < 2 ? 1 - k : k);
      for (int e = 0; e < 9; e++) V[9 * k + e] = src[e];
    }
  __syncwarp();
  auto mkface = [&](int f, int a, int b, int c) {
    // all lanes compute the same values; lane 0 stores
    R ab[3], ac[3], nn[3];
    v3sub(ab, V + 9 * b, V + 9 * a);
    v3sub(ac, V + 9 * c, V + 9 * a);
    v3cross(nn, ab, ac);
    R len = v3norm(nn), d;
    if (len < R(1e-30)) { d = Lim<R>::big(); nn[0] = 1; nn[1] = 0; nn[2] = 0; }
    else { v3scl(nn, nn, R(1) / len); d = v3dot(nn, V + 9 * a); }
    if (lane == 0) { Fn[4 * f] = nn[0]; Fn[4 * f + 1] = nn[1]; Fn[4 * f + 2] = nn[2]; Fn[4 * f + 3] = d; Fi[f] = a | (b << 8) | (c << 16) | (1 << 24); }
  };
  mkface(0, 0, 1, 2); mkface(1, 0, 3, 1); mkface(2, 0, 2, 3); mkface(3, 1, 3, 2);
  nF = 4;
  __syncwarp();
  int bestf = -1;
  // fp32: 1e-6 - at 2e-6 the depth error of resting mesh contacts moved loose objects by 2-8e-4 per control step
  const R epa_tol = sizeof(R) == 4 ? R(1e-6) : R(1e-7);
  const R vis_tol = sizeof(R) == 4 ? R(2e-7) : R(1e-12);  // fp32: above the rounding noise of the plane distances
  for (int it = 0; it < 100; it++) {
    // closest alive face (lane-parallel scan)
    R bd = Lim<R>::big();
    int bf = 0x7fffffff;
    for (int f = lane; f < nF; f += 32)
      if ((Fi[f] >> 24) && Fn[4 * f + 3] < bd) { bd = Fn[4 * f + 3]; bf = f; }
    R nbd = -bd;
    warp_argmax(nbd, bf);
    bd = -nbd;
    if (bf == 0x7fffffff) return -1;
    bestf = bf;
    R fn[3] = {Fn[4 * bf], Fn[4 * bf + 1], Fn[4 * bf + 2]};
    SV<R> w;
    sv_support(A, B, fn, w, lane);
    R dw = v3dot(w.w, fn);
#ifdef B2S_EPA_TRACE
    if (lane == 0) printf("dev it %d bf %d bd %.9g dw %.9g nV %d nF %d n %.4f %.4f %.4f\n", it, bf, (double)bd, (double)dw, nV, nF, (double)fn[0], (double)fn[1], (double)fn[2]);
#endif
    if (dw - bd < epa_tol || nV >= maxv - 1 || nF >= maxf - 16) break;
    // remove the faces visible from w and build the horizon.  Visibility is tested lane-parallel (32 faces at a time);
    // the few visible faces are then processed in increasing face order by the whole warp (same order as a serial scan).
    int ne = 0;
    for (int base = 0; base < nF; base += 32) {
      int f = base + lane, fi = 0;
      bool vis = false;
      if (f < nF) {
        fi = Fi[f];
        if (fi >> 24) {
          const R* va = V + 9 * (fi & 255);
          vis = Fn[4 * f] * (w.w[0] - va[0]) + Fn[4 * f + 1] * (w.w[1] - va[1]) + Fn[4 * f + 2] * (w.w[2] - va[2]) > vis_tol;
        }
      }
      unsigned mask = __ballot_sync(B2S_FULL, vis);
      while (mask) {
        int l = __ffs(mask) - 1;
        mask &= mask - 1;
        int fv = __shfl_sync(B2S_FULL, fi, l);
        if (lane == 0) Fi[base + l] = fv & 0xffffff;
        int vs[3] = {fv & 255, (fv >> 8) & 255, (fv >> 16) & 255};
#pragma unroll
        for (int k = 0; k < 3; k++) {
          // toggle the directed edge (a, b): it cancels against its reverse if that is in the list (swap-remove, same list order as
          // the serial search of the oracle), otherwise it is appended.  The search is lane-parallel; at most one entry matches.
          int a = vs[k], b = vs[(k + 1) % 3], key = b | (a << 8), hit = -1;
          for (int q = lane; q < ne; q += 32)
            if (edges[q] == key) hit = q;
          unsigned hm = __ballot_sync(B2S_FULL, hit >= 0);
          if (hm) {
            int idx = __shfl_sync(B2S_FULL, hit, __ffs(hm) - 1);
            if (lane == 0) edges[idx] = edges[ne - 1];
            ne--;
          } else if (ne < 64) {
            if (lane == 0) edges[ne] = a | (b << 8);
            ne++;
          }
          __syncwarp();
        }
      }
    }
    __syncwarp();
#ifdef B2S_EPA_TRACE
    if (lane == 0) printf("dev    ne %d\n", ne);
#endif
    if (ne == 0) break;
    int vi = nV;
    if (lane == 0)
      for (int e = 0; e < 3; e++) { V[9 * vi + e] = w.w[e]; V[9 * vi + 3 + e] = w.a[e]; V[9 * vi + 6 + e] = w.b[e]; }
    nV++;
    __syncwarp();
    // new faces (horizon edge, w): one lane per face
    int nnew = ne < maxf - nF ? ne : maxf - nF;
    for (int q = lane; q < nnew; q += 32) {
      int a = edges[q] & 255, b = edges[q] >> 8, f = nF + q;
      R ab[3], ac[3], nn[3];
      v3sub(ab, V + 9 * b, V + 9 * a);
      v3sub(ac, V + 9 * vi, V + 9 * a);
      v3cross(nn, ab, ac);
      R len = v3norm(nn), d;
      if (len < R(1e-30)) { d = Lim<R>::big(); nn[0] = 1; nn[1] = 0; nn[2] = 0; }
      else { v3scl(nn, nn, R(1) / len); d = v3dot(nn, V + 9 * a); }
      Fn[4 * f] = nn[0]; Fn[4 * f + 1] = nn[1]; Fn[4 * f + 2] = nn[2]; Fn[4 * f + 3] = d;
      Fi[f] = a | (b << 8) | (vi << 16) | (1 << 24);
    }
    nF += nnew;
    __syncwarp();
  }
#ifdef B2S_INSTR
  if (lane == 0) { edges[64] = nV; edges[65] = nF; }
#endif
  if (bestf < 0) return -1;
  int fi = Fi[bestf];
  int ia = fi & 255, ib = (fi >> 8) & 255, ic = (fi >> 16) & 255;
  depth = Fn[4 * bestf + 3];
  normal[0] = Fn[4 * bestf]; normal[1] = Fn[4 * bestf + 1]; normal[2] = Fn[4 * bestf + 2];
  R pp[3], v0[3], v1[3], v2[3];
  v3scl(pp, normal, depth);
  const R *a = V + 9 * ia, *b = V + 9 * ib, *c = V + 9 * ic;
  v3sub(v0, b, a); v3sub(v1, c, a); v3sub(v2, pp, a);
  R d00 = v3dot(v0, v0), d01 = v3dot(v0, v1), d11 = v3dot(v1, v1), d20 = v3dot(v2, v0), d21 = v3dot(v2, v1);
  R den = d00 * d11 - d01 * d01;
  R bv = den != 0 ? (d11 * d20 - d01 * d21) / den : R(0), bw = den != 0 ? (d00 * d21 - d01 * d20) / den : R(0);
  R bu = 1 - bv - bw;
  for (int k = 0; k < 3; k++) {
    wa[k] = bu * a[3 + k] + bv * b[3 + k] + bw * c[3 + k];
    wb[k] = bu * a[6 + k] + bv * b[6 + k] + bw * c[6 + k];
  }
  __syncwarp();
  return 0;
}

// `stage` (work-list convex kernel only): shared-memory area of `stage_cap` reals for the hull vertices of the pair.  The mesh support
// scans are L2-latency bound when they read the model's vertex array (L1 is a few KB beside 200+ KB of shared memory): a pair
// that the remembered separating direction does not dismiss at once gets its vertices copied in first (one coalesced pass, the
// cost of a single support scan) and all later scans - tens in GJK, up to ~190 in a deep EPA - run from shared memory.  Same
// vertex values, same arithmetic, same results.
template <typename R>
DEVN int convex_convex(const Shape<R>& A0, const Shape<R>& B0, R* out, int maxn, R* scratch, int lane, R* cache = nullptr,
                       int maxv = EPA_MAXV, int maxf = EPA_MAXF, R* stage = nullptr, int stage_cap = 0) {
  R* simplex = EPA_SIMPLEX(scratch, maxv, maxf);  // shared memory
  int ns = 0;
  R dist = 0, wa[3], wb[3], n[3], pos[3], pa[3], pb[3];
  Shape<R> A = A0, B = B0;
  R ra = shape_radius(A), rb = shape_radius(B);
  if (stage != nullptr) {
    // the two poses first (24 reals, one load per lane): support_w reads them on every call - through pointers into the global
    // workspace row that is four dependent L2 latencies per support pair (ncu: long-scoreboard stalls on the first use of `mat` and
    // on `pos` were ~45 % of support_w's samples), and the dismissal test below is one support pair
    __syncwarp();
    if (lane < 12) stage[lane] = lane < 3 ? A.pos[lane] : A.mat[lane - 3];
    else if (lane < 24) stage[lane] = lane < 15 ? B.pos[lane - 12] : B.mat[lane - 15];
    A.pos = stage; A.mat = stage + 3; B.pos = stage + 12; B.mat = stage + 15;
    stage += 24; stage_cap -= 24;
    __syncwarp();
    if (cache != nullptr) {  // gjk()'s own first test, made here so that dismissed pairs (the common case) never pay for staging the hulls
      R cv[3];
      if (warm_direction(cache, cv)) {
        R nv[3] = {-cv[0], -cv[1], -cv[2]};
        SV<R> w0;
        sv_support(A, B, nv, w0, lane);
        R vv0 = v3dot(cv, cv), vw0 = v3dot(cv, w0.w), cut = ra + rb;
        if (vw0 > 0 && vw0 * vw0 > cut * cut * vv0) return 0;
      }
    }
    __syncwarp();
    int used = 0;
    if (A.nvert > 0 && 3 * A.nvert <= stage_cap) {
      for (int i = lane; i < 3 * A.nvert; i += 32) stage[i] = A.vert[i];
      A.vert = stage; used = (3 * A.nvert + 3) & ~3;
    }
    if (B.nvert > 0 && used + 3 * B.nvert <= stage_cap) {
      if (B.vert == A0.vert && A.vert == stage) B.vert = stage;  // the same hull twice (two instances of one mesh)
      else { for (int i = lane; i < 3 * B.nvert; i += 32) stage[used + i] = B.vert[i]; B.vert = stage + used; }
    }
    __syncwarp();
  }
#ifdef B2S_INSTR
  long long tg0 = clock64();
#endif
  int hit = gjk(A, B, simplex, ns, dist, wa, wb, ra + rb, lane, cache);
#ifdef B2S_INSTR
  if (stage != nullptr && lane == 0) {
    int* sp = reinterpret_cast<int*>(scratch + 9 * maxv + 4 * maxf) + maxf + 64;
    sp[2] = (int)(clock64() - tg0); sp[3] = hit; sp[0] = 0; sp[1] = 0; sp[4] = (A.vert == stage) | ((B.vert != B0.vert) << 1);
  }
#endif
  if (!hit) {
    if (ra + rb <= 0 || dist > ra + rb) return 0;
    v3sub(n, wb, wa);
    v3scl(n, n, R(1) / dist);
    v3addscl(pa, wa, n, ra);
    v3addscl(pb, wb, n, -rb);
    v3add(pos, pa, pb);
    v3scl(pos, pos, R(0.5));
    return put(out, 0, maxn, pos, n, dist - ra - rb);
  }
  R depth;
  if (epa(A, B, simplex, ns, depth, n, wa, wb, scratch, lane, maxv, maxf) != 0) return 0;
  v3addscl(pa, wa, n, ra);
  v3addscl(pb, wb, n, -rb);
  v3add(pos, pa, pb);
  v3scl(pos, pos, R(0.5));
  return put(out, 0, maxn, pos, n, -depth - ra - rb);
}

// ---------------------------------------------------------------------------------------------- driver
// oriented-box overlap of the two geoms' local AABBs (15-axis separating test); planes use the box/plane distance
template <typename R> DEVN bool obb_overlap(const Eng<R> e, int g1, int g2) {
  const DModel<R>& m = e.model();
  int k1 = m.geom_cgid[g1], k2 = m.geom_cgid[g2];
  const R* M1 = e.p(e.lay().gmat) + 9 * k1; const R* M2 = e.p(e.lay().gmat) + 9 * k2;
  const R* a1 = geom_aabb_of(m, e.state(), g1, e.env); const R* a2 = geom_aabb_of(m, e.state(), g2, e.env);
  R c1[3], c2[3], t[3];
  R o1[3] = {a1[0], a1[1], a1[2]}, o2[3] = {a2[0], a2[1], a2[2]};
  m3mulv(t, M1, o1); v3add(c1, t, e.p(e.lay().gpos) + 3 * k1);
  m3mulv(t, M2, o2); v3add(c2, t, e.p(e.lay().gpos) + 3 * k2);
  R ha[3] = {a1[3], a1[4], a1[5]}, hb[3] = {a2[3], a2[4], a2[5]};
  int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  if (t1 == G_PLANE || t2 == G_PLANE) {
    const R* Mp = t1 == G_PLANE ? M1 : M2; const R* Mo = t1 == G_PLANE ? M2 : M1;
    const R* pp = e.p(e.lay().gpos) + 3 * (t1 == G_PLANE ? k1 : k2);
    const R* co = t1 == G_PLANE ? c2 : c1; const R* ho = t1 == G_PLANE ? hb : ha;
    R n[3] = COLV(Mp, 2), df[3];
    v3sub(df, co, pp);
    R d = v3dot(df, n);
    for (int k = 0; k < 3; k++) { R ax[3] = COLV(Mo, k); d -= ho[k] * r_abs(v3dot(n, ax)); }
    return d <= 0;
  }
  R T[3];
  v3sub(T, c2, c1);
  R A[3][3], B[3][3];
  for (int k = 0; k < 3; k++) { A[k][0] = M1[k]; A[k][1] = M1[3 + k]; A[k][2] = M1[6 + k]; B[k][0] = M2[k]; B[k][1] = M2[3 + k]; B[k][2] = M2[6 + k]; }
  R Rm[3][3], AR[3][3], ta[3];
  const R eps = sizeof(R) == 4 ? R(1e-5) : R(1e-9);
  for (int i = 0; i < 3; i++) {
    ta[i] = v3dot(T, A[i]);
    for (int j = 0; j < 3; j++) { Rm[i][j] = v3dot(A[i], B[j]); AR[i][j] = r_abs(Rm[i][j]) + eps; }
  }
  for (int i = 0; i < 3; i++)
    if (r_abs(ta[i]) > ha[i] + hb[0] * AR[i][0] + hb[1] * AR[i][1] + hb[2] * AR[i][2]) return false;
  for (int j = 0; j < 3; j++) {
    R tb = ta[0] * Rm[0][j] + ta[1] * Rm[1][j] + ta[2] * Rm[2][j];
    if (r_abs(tb) > ha[0] * AR[0][j] + ha[1] * AR[1][j] + ha[2] * AR[2][j] + hb[j]) return false;
  }
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      R ra = ha[i1] * AR[i2][j] + ha[i2] * AR[i1][j];
      R rb = hb[j1] * AR[i][j2] + hb[j2] * AR[i][j1];
      if (r_abs(ta[i2] * Rm[i1][j] - ta[i1] * Rm[i2][j]) > ra + rb) return false;
    }
  return true;
}

template <typename R> DEV bool is_gjk_pair(int t1, int t2) {
  if (t1 > t2) { int t = t1; t1 = t2; t2 = t; }
  if (t1 == G_PLANE) return false;
  if (t1 == G_SPHERE && (t2 == G_SPHERE || t2 == G_CAPSULE || t2 == G_BOX || t2 == G_CYLINDER)) return false;
  if ((t1 == G_BOX && t2 == G_BOX) || (t1 == G_CAPSULE && t2 == G_CAPSULE)) return false;
  return true;
}

// friction / condim mixing (equal priority: max; otherwise the higher-priority geom)
template <typename R> DEV void mix_contact(const DModel<R>& m, const DState<R>& s, int env, int g1, int g2, R* fric3, int& dim) {
  int p1 = m.geom_priority[g1], p2 = m.geom_priority[g2];
  const R* f1 = geom_friction_of(m, s, g1, env); const R* f2 = geom_friction_of(m, s, g2, env);
  if (p1 != p2) {
    const R* f = p1 > p2 ? f1 : f2;
    dim = m.geom_condim[p1 > p2 ? g1 : g2];
    fric3[0] = f[0]; fric3[1] = f[1]; fric3[2] = f[2];
    return;
  }
  dim = max(m.geom_condim[g1], m.geom_condim[g2]);
  for (int k = 0; k < 3; k++) fric3[k] = r_max(f1[k], f2[k]);
}

template <typename R> DEV int narrow_analytic(const Shape<R>& A, const Shape<R>& B, R* buf) {
  int t1 = A.type, t2 = B.type, n = 0;
  if (t1 == G_PLANE) {
    if (t2 == G_SPHERE) n = plane_sphere(A, B, buf, 8);
    else if (t2 == G_BOX) n = plane_box(A, B, buf, 8);
    else if (t2 == G_CYLINDER) n = plane_cylinder(A, B, buf, 8);
    else if (t2 == G_MESH) n = plane_mesh(A, B, buf, 8);
    else if (t2 == G_CAPSULE) n = plane_capsule(A, B, buf, 8);
    else if (t2 == G_ELLIPSOID) n = plane_ellipsoid(A, B, buf, 8);
  } else if (t1 == G_SPHERE && t2 == G_SPHERE) n = sphere_sphere(A, B, buf, 8);
  else if (t1 == G_SPHERE && t2 == G_BOX) n = sphere_box(A, B, buf, 8);
  else if (t1 == G_SPHERE && t2 == G_CYLINDER) n = sphere_cylinder(A, B, buf, 8);
  else if (t1 == G_SPHERE && t2 == G_CAPSULE) n = sphere_capsule(A, B, buf, 8);
  else if (t1 == G_CAPSULE && t2 == G_CAPSULE) n = capsule_capsule(A, B, buf, 8);
  else if (t1 == G_BOX && t2 == G_BOX) n = box_box(A, B, buf, 8);
  return n;
}

// ---- one narrow-phase pair, for all three schedules: the shapes come from the geom poses `gpos` / `gmat` (the fused kernel's workspace,
// or the environment's workspace row), the contacts are counted and returned as records in `buf`

// the pair's geoms in type order (the narrow-phase routines take the lower type first; contacts carry the geoms in this order)
template <typename R> DEV void pair_geoms(const DModel<R>& m, int pidx, int& g1, int& g2) {
  g1 = m.pair_geom[2 * pidx]; g2 = m.pair_geom[2 * pidx + 1];
  if (m.geom_type[g1] > m.geom_type[g2]) { int t = g1; g1 = g2; g2 = t; }
}

// one analytic pair, one lane: up to 8 records
template <typename R>
DEV int narrow_pair_analytic(const DModel<R>& m, const DState<R>& s, int env, int pidx, const R* gpos, const R* gmat, R* buf) {
  int g1, g2;
  pair_geoms(m, pidx, g1, g2);
  Shape<R> A, B;
  shape_from(m, s, env, g1, gpos, gmat, A);
  shape_from(m, s, env, g2, gpos, gmat, B);
  return narrow_analytic(A, B, buf);
}

// one convex pair, the whole warp: at most one record.  `scratch` holds the EPA polytope; `cache` is the pair's GJK warm-start
// direction and `stage` (stage_cap words) the hull staging area, or nullptr - the fused kernel passes nullptr for both, so that its
// results never depend on earlier substeps.  item_stats: -DB2S_INSTR per-item cost histogram and slow-item log (the phase-1 convex role)
template <typename R>
DEV int narrow_pair_convex(const DModel<R>& m, const DState<R>& s, int env, int pidx, const R* gpos, const R* gmat, R* buf, R* scratch,
                           R* cache, R* stage, int stage_cap, int lane, bool item_stats) {
  int g1, g2;
  pair_geoms(m, pidx, g1, g2);
  Shape<R> A, B;
  shape_from(m, s, env, g1, gpos, gmat, A);
  shape_from(m, s, env, g2, gpos, gmat, B);
#ifdef B2S_INSTR
  long long it0 = clock64();
#endif
  int n = convex_convex(A, B, buf, 1, scratch, lane, cache, EPA_MAXV, EPA_MAXF, stage, stage_cap);
#ifdef B2S_INSTR
  if (item_stats && lane == 0 && s.stats) {  // bucket k = cycles in [2^(k+8), 2^(k+9)), by shape types (mesh-mesh / other)
    long long dt = clock64() - it0;
    int k = 0;
    while (k < 11 && (dt >> (k + 9)) > 0) k++;
    atomicAdd(s.stats + 500 - 12 * ((A.type == G_MESH && B.type == G_MESH) ? 2 : 1) + k, 1);
    if (n > 0) atomicAdd(s.stats + 18, 1);
    if (dt > (1 << 19) && s.slowlog) {  // items above 524 k cycles (~270 us): what are they?
      int j = atomicAdd(s.stats + 20, 1);
      if (j < 64) {
        const int* sp = reinterpret_cast<const int*>(scratch + 9 * EPA_MAXV + 4 * EPA_MAXF) + EPA_MAXF + 64;
        int* o = s.slowlog + 12 * j;
        o[0] = (int)dt; o[1] = A.type; o[2] = B.type; o[3] = A.nvert; o[4] = B.nvert; o[5] = sp[0]; o[6] = sp[1]; o[7] = sp[2]; o[8] = sp[3];
        o[9] = sp[4]; o[10] = g1; o[11] = g2;
      }
    }
  }
#endif
  return n;
}

// Cull the static pair list (bounding spheres, then oriented boxes); candidate pair indices in pair order.
template <typename R> DEV void cull_pairs(Eng<R> e, int* cand, int* cand_g, int maxa, int maxg, int& na_out, int& ng_out) {
  const DModel<R>& m = e.model();
  const DState<R>& st = e.state();
  const WSLayout& L = e.lay();
  int lane = e.lane, na = 0, ng = 0;
  const R* gpos = e.p(L.gpos); const R* gmat = e.p(L.gmat);
  for (int base = 0; base < m.npair; base += 32) {
    int pidx = base + lane;
    int pass = 0, isg = 0;
    if (pidx < m.npair) {
      int g1 = m.pair_geom[2 * pidx], g2 = m.pair_geom[2 * pidx + 1];
      int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
      int k1 = m.geom_cgid[g1], k2 = m.geom_cgid[g2];
      if (t1 != G_PLANE && t2 != G_PLANE) {
        R df[3];
        v3sub(df, gpos + 3 * k1, gpos + 3 * k2);
        R bound = geom_rbound_of(m, st, g1, e.env) + geom_rbound_of(m, st, g2, e.env);
        pass = v3dot(df, df) <= bound * bound;
      } else {
        int kp = t1 == G_PLANE ? k1 : k2, ko = t1 == G_PLANE ? k2 : k1, go = t1 == G_PLANE ? g2 : g1;
        R nrm[3] = COLV(gmat + 9 * kp, 2), df[3];
        v3sub(df, gpos + 3 * ko, gpos + 3 * kp);
        pass = v3dot(df, nrm) <= geom_rbound_of(m, st, go, e.env);
      }
      if (pass) pass = obb_overlap(e, g1, g2);
      isg = is_gjk_pair<R>(t1, t2);
    }
    unsigned ma = __ballot_sync(B2S_FULL, pass && !isg), mg = __ballot_sync(B2S_FULL, pass && isg);
    unsigned lt = (1u << lane) - 1;
    if (pass && !isg) { int r = na + __popc(ma & lt); if (r < maxa) cand[r] = pidx; }
    if (pass && isg) { int r = ng + __popc(mg & lt); if (r < maxg) cand_g[r] = pidx; }
    na += __popc(ma);
    ng += __popc(mg);
  }
  na_out = na; ng_out = ng;
  __syncwarp();
}

// per contact: condim + friction mixing (shared by the fused and the pipelined collision paths)
template <typename R> DEV void finish_contacts(const Eng<R>& e, int ncon) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  R* cfric = e.p(L.c_fric);
  int* cint = e.pi(L.c_int);
  for (int c = e.lane; c < ncon; c += 32) {
    R f3[3];
    int dim;
    mix_contact(m, e.state(), e.env, cint[5 * c], cint[5 * c + 1], f3, dim);
    cfric[3 * c] = f3[0]; cfric[3 * c + 1] = f3[1]; cfric[3 * c + 2] = f3[2];
    cint[5 * c + 2] = dim;
    cint[5 * c + 3] = -1;
  }
  __syncwarp();
}

// The fused kernel's collision stage, composed of the shared pieces: broad phase (at most 96 analytic and 96 convex candidates),
// analytic candidates one lane each, convex candidates the whole warp each, contacts ordered by pair index, friction / condim mixing.
// Fills the contact arrays in the workspace; returns ncon (warp-uniform).  warn bit 4 on candidate or contact overflow (the contacts
// kept are the first maxcon found, analytic before convex).
template <typename R> DEVN int collide(Eng<R> e, int& warn) {
  const DModel<R>& m = e.model();
  const DState<R>& st = e.state();
  const WSLayout& L = e.lay();
  const int lane = e.lane, MAXC = 96;
  const R* gpos = e.p(L.gpos); const R* gmat = e.p(L.gmat);
  int* cand = e.pi(L.scratch);  // candidate pair indices: analytic, convex at +MAXC
  int* cand_g = cand + MAXC;
  int na, ng;
  cull_pairs(e, cand, cand_g, MAXC, MAXC, na, ng);
  if (na > MAXC) { na = MAXC; warn |= 4; }
  if (ng > MAXC) { ng = MAXC; warn |= 4; }
  R* cpos = e.p(L.c_pos); R* cfr = e.p(L.c_frame); R* cdist = e.p(L.c_dist);
  int* cint = e.pi(L.c_int);
  int ncon = 0;
  // --- analytic candidates: one lane per pair
  for (int base = 0; base < na; base += 32) {
    int ci = base + lane;
    R buf[8 * CREC];
    int n = 0, g1 = 0, g2 = 0, pidx = 0;
    if (ci < na) {
      pidx = cand[ci];
      pair_geoms(m, pidx, g1, g2);
      n = narrow_pair_analytic(m, st, e.env, pidx, gpos, gmat, buf);
    }
    // ordered compaction
    int off = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(B2S_FULL, off, o); if (lane >= o) off += t; }
    int total = __shfl_sync(B2S_FULL, off, 31);
    off = ncon + off - n;
    for (int k = 0; k < n; k++) {
      int c = off + k;
      if (c >= L.mc) break;
      const R* b = buf + CREC * k;
      cpos[3 * c] = b[0]; cpos[3 * c + 1] = b[1]; cpos[3 * c + 2] = b[2];
      cfr[3 * c] = b[3]; cfr[3 * c + 1] = b[4]; cfr[3 * c + 2] = b[5];
      cdist[c] = b[6];
      cint[5 * c] = g1; cint[5 * c + 1] = g2; cint[5 * c + 4] = pidx;
    }
    ncon += total;
  }
  if (ncon > L.mc) { ncon = L.mc; warn |= 4; }
  __syncwarp();
  // --- convex candidates: the whole warp per pair (the fused kernel appends the EPA polytope area to every warp's workspace)
  R* epa_scratch = e.ws + L.total;
  for (int ci = 0; ci < ng; ci++) {
    int pidx = cand_g[ci], g1, g2;
    pair_geoms(m, pidx, g1, g2);
    R buf[CREC];
    int n = narrow_pair_convex(m, st, e.env, pidx, gpos, gmat, buf, epa_scratch, (R*)nullptr, (R*)nullptr, 0, lane, false);
    if (n > 0) {
      if (ncon < L.mc) {
        int c = ncon;
        if (lane == 0) {
          cpos[3 * c] = buf[0]; cpos[3 * c + 1] = buf[1]; cpos[3 * c + 2] = buf[2];
          cfr[3 * c] = buf[3]; cfr[3 * c + 1] = buf[4]; cfr[3 * c + 2] = buf[5];
          cdist[c] = buf[6];
          cint[5 * c] = g1; cint[5 * c + 1] = g2; cint[5 * c + 4] = pidx;
        }
        ncon++;
      } else warn |= 4;
    }
    __syncwarp();
  }
  __syncwarp();
  // --- order contacts by pair index (stable): up to 32 by rank = #contacts with a smaller key, more by insertion on lane 0
  if (ng > 0 && ncon > 1) {
    if (ncon <= 32) {
      int c = lane;
      R rec[7];
      int gi1 = 0, gi2 = 0, key = 0x7fffffff, rank = 0;
      if (c < ncon) {
        key = cint[5 * c + 4] * 256 + c;
        gi1 = cint[5 * c]; gi2 = cint[5 * c + 1];
        rec[0] = cpos[3 * c]; rec[1] = cpos[3 * c + 1]; rec[2] = cpos[3 * c + 2];
        rec[3] = cfr[3 * c]; rec[4] = cfr[3 * c + 1]; rec[5] = cfr[3 * c + 2];
        rec[6] = cdist[c];
      }
      for (int o = 0; o < 32; o++) {
        int ok = __shfl_sync(B2S_FULL, key, o);
        if (ok < key) rank++;
      }
      __syncwarp();
      if (c < ncon) {
        cpos[3 * rank] = rec[0]; cpos[3 * rank + 1] = rec[1]; cpos[3 * rank + 2] = rec[2];
        cfr[3 * rank] = rec[3]; cfr[3 * rank + 1] = rec[4]; cfr[3 * rank + 2] = rec[5];
        cdist[rank] = rec[6];
        cint[5 * rank] = gi1; cint[5 * rank + 1] = gi2; cint[5 * rank + 4] = key / 256;
      }
    } else if (lane == 0) {
      for (int i = 1; i < ncon; i++)
        for (int j = i; j > 0 && cint[5 * j + 4] < cint[5 * (j - 1) + 4]; j--) {
          for (int q = 0; q < 3; q++) { R t = cpos[3 * j + q]; cpos[3 * j + q] = cpos[3 * (j - 1) + q]; cpos[3 * (j - 1) + q] = t; }
          for (int q = 0; q < 3; q++) { R t = cfr[3 * j + q]; cfr[3 * j + q] = cfr[3 * (j - 1) + q]; cfr[3 * (j - 1) + q] = t; }
          { R t = cdist[j]; cdist[j] = cdist[j - 1]; cdist[j - 1] = t; }
          for (int q = 0; q < 5; q++) { int t = cint[5 * j + q]; cint[5 * j + q] = cint[5 * (j - 1) + q]; cint[5 * (j - 1) + q] = t; }
        }
    }
    __syncwarp();
  }
  finish_contacts(e, ncon);
  return ncon;
}
