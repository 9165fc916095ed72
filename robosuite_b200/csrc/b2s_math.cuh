// Small vector / quaternion / warp helpers (device, templated on the arithmetic type).
#pragma once
#include "b2s_types.cuh"

#define DEV __device__ __forceinline__
#define DEVN __device__ __noinline__

template <typename R> DEV R r_sqrt(R x);
template <> DEV float r_sqrt<float>(float x) { return sqrtf(x); }
template <> DEV double r_sqrt<double>(double x) { return sqrt(x); }
template <typename R> DEV R r_abs(R x) { return x < R(0) ? -x : x; }
template <typename R> DEV R r_max(R a, R b) { return a > b ? a : b; }
template <typename R> DEV R r_min(R a, R b) { return a < b ? a : b; }
template <typename R> DEV R r_clamp(R x, R lo, R hi) { return x < lo ? lo : (x > hi ? hi : x); }
template <typename R> DEV void r_sincos(R x, R* s, R* c);
template <> DEV void r_sincos<float>(float x, float* s, float* c) { sincosf(x, s, c); }
template <> DEV void r_sincos<double>(double x, double* s, double* c) { sincos(x, s, c); }
template <typename R> DEV R r_pow(R x, R y);
template <> DEV float r_pow<float>(float x, float y) { return powf(x, y); }
template <> DEV double r_pow<double>(double x, double y) { return pow(x, y); }
template <typename R> DEV R r_atan2(R y, R x);
template <> DEV float r_atan2<float>(float y, float x) { return atan2f(y, x); }
template <> DEV double r_atan2<double>(double y, double x) { return atan2(y, x); }
template <typename R> struct Lim;
template <> struct Lim<float> { static DEV float big() { return 3.0e38f; } static DEV float minval() { return 1e-15f; } static DEV float eps() { return 1.1920929e-7f; } };
template <> struct Lim<double> { static DEV double big() { return 1.0e300; } static DEV double minval() { return 1e-15; } static DEV double eps() { return 2.220446049250313e-16; } };

template <typename R> DEV void v3set(R* r, R a, R b, R c) { r[0] = a; r[1] = b; r[2] = c; }
template <typename R> DEV void v3copy(R* r, const R* a) { r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; }
template <typename R> DEV void v3add(R* r, const R* a, const R* b) { r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; }
template <typename R> DEV void v3sub(R* r, const R* a, const R* b) { r[0] = a[0] - b[0]; r[1] = a[1] - b[1]; r[2] = a[2] - b[2]; }
template <typename R> DEV void v3scl(R* r, const R* a, R s) { r[0] = a[0] * s; r[1] = a[1] * s; r[2] = a[2] * s; }
template <typename R> DEV void v3addscl(R* r, const R* a, const R* b, R s) { r[0] = a[0] + b[0] * s; r[1] = a[1] + b[1] * s; r[2] = a[2] + b[2] * s; }
template <typename R> DEV R v3dot(const R* a, const R* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
template <typename R> DEV R v3norm(const R* a) { return r_sqrt(v3dot(a, a)); }
template <typename R> DEV void v3cross(R* r, const R* a, const R* b) {
  R x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
template <typename R> DEV R v3normalize(R* a) {
  R n = v3norm(a);
  if (n < Lim<R>::minval()) { a[0] = 1; a[1] = 0; a[2] = 0; return 0; }
  R inv = R(1) / n;
  a[0] *= inv; a[1] *= inv; a[2] *= inv;
  return n;
}
template <typename R> DEV void m3mulv(R* r, const R* M, const R* v) {
  R x = M[0] * v[0] + M[1] * v[1] + M[2] * v[2], y = M[3] * v[0] + M[4] * v[1] + M[5] * v[2], z = M[6] * v[0] + M[7] * v[1] + M[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
template <typename R> DEV void m3mulTv(R* r, const R* M, const R* v) {
  R x = M[0] * v[0] + M[3] * v[1] + M[6] * v[2], y = M[1] * v[0] + M[4] * v[1] + M[7] * v[2], z = M[2] * v[0] + M[5] * v[1] + M[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
template <typename R> DEV void qmul(R* r, const R* a, const R* b) {
  R w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  R x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  R y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  R z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
// v rotated by the unit quaternion q:  v + 2 w (u x v) + 2 u x (u x v)
template <typename R> DEV void qrot(R* r, const R* q, const R* v) {
  R t[3] = {R(2) * (q[2] * v[2] - q[3] * v[1]), R(2) * (q[3] * v[0] - q[1] * v[2]), R(2) * (q[1] * v[1] - q[2] * v[0])};
  R x = v[0] + q[0] * t[0] + (q[2] * t[2] - q[3] * t[1]);
  R y = v[1] + q[0] * t[1] + (q[3] * t[0] - q[1] * t[2]);
  R z = v[2] + q[0] * t[2] + (q[1] * t[1] - q[2] * t[0]);
  r[0] = x; r[1] = y; r[2] = z;
}
template <typename R> DEV void qnormalize(R* q) {
  R n = r_sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < Lim<R>::minval()) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  R inv = R(1) / n;
  q[0] *= inv; q[1] *= inv; q[2] *= inv; q[3] *= inv;
}
template <typename R> DEV void q2mat(R* M, const R* q) {
  R w = q[0], x = q[1], y = q[2], z = q[3];
  M[0] = w * w + x * x - y * y - z * z; M[1] = 2 * (x * y - w * z); M[2] = 2 * (x * z + w * y);
  M[3] = 2 * (x * y + w * z); M[4] = w * w - x * x + y * y - z * z; M[5] = 2 * (y * z - w * x);
  M[6] = 2 * (x * z - w * y); M[7] = 2 * (y * z + w * x); M[8] = w * w - x * x - y * y + z * z;
}
template <typename R> DEV void aa2quat(R* q, const R* axis, R angle) {
  R s, c;
  r_sincos(R(0.5) * angle, &s, &c);
  q[0] = c; q[1] = axis[0] * s; q[2] = axis[1] * s; q[3] = axis[2] * s;
}

// ---- spatial algebra about the world origin: motion [w; vO], force [tauO; f], inertia (xx,yy,zz,xy,xz,yz,h3,m)
template <typename R> DEV void inert_mulv(R* f, const R* I, const R* v) {
  const R *w = v, *l = v + 3, *h = I + 6;
  R t[3];
  f[0] = I[0] * w[0] + I[3] * w[1] + I[4] * w[2];
  f[1] = I[3] * w[0] + I[1] * w[1] + I[5] * w[2];
  f[2] = I[4] * w[0] + I[5] * w[1] + I[2] * w[2];
  v3cross(t, h, l);
  v3add(f, f, t);
  v3cross(t, w, h);
  f[3] = I[9] * l[0] + t[0]; f[4] = I[9] * l[1] + t[1]; f[5] = I[9] * l[2] + t[2];
}
template <typename R> DEV R dot6(const R* a, const R* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5]; }
template <typename R> DEV void cross_motion(R* r, const R* v, const R* s) {
  R a[3], b[3];
  v3cross(r, v, s);
  v3cross(a, v, s + 3);
  v3cross(b, v + 3, s);
  v3add(r + 3, a, b);
}
template <typename R> DEV void cross_force(R* r, const R* v, const R* f) {
  R a[3], b[3];
  v3cross(a, v, f);
  v3cross(b, v + 3, f + 3);
  v3add(r, a, b);
  v3cross(r + 3, v, f + 3);
}

// ---- warp collectives
template <typename R> DEV R warp_sum(R v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(B2S_FULL, v, o);
  return v;
}
template <typename R> DEV R warp_max(R v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = r_max(v, __shfl_xor_sync(B2S_FULL, v, o));
  return v;
}
DEV int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(B2S_FULL, v, o);
  return v;
}
DEV int warp_or_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v |= __shfl_xor_sync(B2S_FULL, v, o);
  return v;
}
// (value, index) arg-max; ties resolve to the smallest index so that every lane agrees
template <typename R> DEV void warp_argmax(R& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    R ov = __shfl_xor_sync(B2S_FULL, v, o);
    int oi = __shfl_xor_sync(B2S_FULL, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
}

// Philox4x32-10 (Salmon et al., SC'11): the counter-based generator of the device draws (perturb_kernel, the observation corruptors)
DEV uint4 philox4x32_10(uint4 c, unsigned k0, unsigned k1) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const unsigned lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const unsigned lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}
