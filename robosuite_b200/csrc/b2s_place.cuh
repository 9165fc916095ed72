// Object placement on the device (b2s_place_config / b2s_place_objects): the reference's UniformRandomSampler /
// SequentialCompositeSampler.sample (utils/placement_samplers.py), lowered on the host to a flat program of entries in placement order.
// One warp per masked environment runs the program in order.  Each object gets up to B2S_PLACE_TRIES tries; lane i evaluates try
// 32 k + i of round k and __ballot_sync picks the lowest valid try, which is exactly the first success of the reference's
// sequential loop.  Draws are Philox4x32-10 keyed by the seed with counter (env, call counter, entry, try) for x (words 0, 1) and y
// (words 2, 3), and (env, call counter, entry, 0xFFFFFFFF) for the rotation's choice (words 0, 1) and angle (words 2, 3); u is formed
// from 53 bits as in perturb_kernel.  All arithmetic is fp64 with explicit roundings (no contraction), and sin / cos come from
// place_sincos below rather than libdevice, so tests/placement_ref.py restates every bit.
#pragma once
#include "b2s_math.cuh"

#define B2S_PLACE_MAX 32      // program entries per handle (one warp's lanes hold the placed positions)
#define B2S_PLACE_TRIES 5000  // the reference's tries per object
#define B2S_PLACE_ROUNDS ((B2S_PLACE_TRIES + 31) / 32)
#define B2S_PLACE_WARN 1024   // warn bit: some object of the environment had no valid try (the reference raises RandomizationError)

struct PlaceDev {
  double x_min, x_max, y_min, y_max, base[3], ref_dz, z_offset, bottom_dz, radius, bottom, top;
  double rot_min[8], rot_max[8];
  int qpos_adr, ref, ensure_valid, axis, n_rot, nov;
  // pose-override targets: [0] the entry's body (pose as placed), [k >= 1] overridden bodies welded to it, pose = placed * (lp, lq)
  void* ov_pos[4];
  void* ov_quat[4];
  double ov_lp[4][3], ov_lq[4][4];
};

__device__ __forceinline__ double place_u53(unsigned a, unsigned b) {
  return (double)(((unsigned long long)(a >> 5) << 26) | (b >> 6)) * 0x1p-53;
}

// sin and cos of a in fp64: Cody-Waite reduction by pi/2 (fdlibm's 33-bit split, exact products for |k| < 2^20) and fdlibm's
// __kernel_sin / __kernel_cos polynomials in Horner form, every operation rounded once.  Within an ulp of libm's values, or 2^-60
// absolute next to the zeros (tests/test_cpu_placement.py checks it against numpy on |a| < 20); the point is that a host
// restatement reproduces it.
__device__ __forceinline__ void place_sincos(double a, double* sn, double* cs) {
  const double k = rint(__dmul_rn(a, 6.36619772367581382433e-01));
  const double r = __dsub_rn(__dsub_rn(a, __dmul_rn(k, 1.57079632673412561417e+00)), __dmul_rn(k, 6.07710050650619224932e-11));
  const double z = __dmul_rn(r, r);
  double ps = __dadd_rn(-2.50507602534068634195e-08, __dmul_rn(z, 1.58969099521155010221e-10));
  ps = __dadd_rn(2.75573137070700676789e-06, __dmul_rn(z, ps));
  ps = __dadd_rn(-1.98412698298579493134e-04, __dmul_rn(z, ps));
  ps = __dadd_rn(8.33333333332248946124e-03, __dmul_rn(z, ps));
  ps = __dadd_rn(-1.66666666666666324348e-01, __dmul_rn(z, ps));
  const double s = __dadd_rn(r, __dmul_rn(__dmul_rn(z, r), ps));
  double pc = __dadd_rn(2.08757232129817482790e-09, __dmul_rn(z, -1.13596475577881948265e-11));
  pc = __dadd_rn(-2.75573143513906633035e-07, __dmul_rn(z, pc));
  pc = __dadd_rn(2.48015872894767294178e-05, __dmul_rn(z, pc));
  pc = __dadd_rn(-1.38888888888741095749e-03, __dmul_rn(z, pc));
  pc = __dadd_rn(4.16666666666666019037e-02, __dmul_rn(z, pc));
  const double hz = __dmul_rn(0.5, z), w = __dsub_rn(1.0, hz);
  const double c = __dadd_rn(w, __dadd_rn(__dsub_rn(__dsub_rn(1.0, w), hz), __dmul_rn(z, __dmul_rn(z, pc))));
  switch ((int)((long long)k & 3)) {
    case 0: *sn = s; *cs = c; break;
    case 1: *sn = c; *cs = -s; break;
    case 2: *sn = -s; *cs = -c; break;
    default: *sn = -c; *cs = s; break;
  }
}

template <typename R>
__global__ void __launch_bounds__(128) place_kernel(const PlaceDev* prog, int n, double* qpos, int nq, const uint8_t* mask, int n_env,
                                                    unsigned long long seed, unsigned counter, int* pending) {
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (env >= n_env || (mask && !mask[env])) return;
  const unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
  double px = 0, py = 0, pz = 0;  // lane j: where entry j was placed
  int failed = 0;
  for (int o = 0; o < n; o++) {
    const PlaceDev& p = prog[o];
    double bx = p.base[0], by = p.base[1], bz = p.base[2];
    if (p.ref >= 0) {
      bx = __shfl_sync(B2S_FULL, px, p.ref);
      by = __shfl_sync(B2S_FULL, py, p.ref);
      bz = __dadd_rn(__shfl_sync(B2S_FULL, pz, p.ref), p.ref_dz);
    }
    const double z = __dsub_rn(__dadd_rn(p.z_offset, bz), p.bottom_dz);
    const double wx = __dsub_rn(p.x_max, p.x_min), wy = __dsub_rn(p.y_max, p.y_min);
    double x = 0, y = 0;
    int found = 0;
    for (int k = 0; k < B2S_PLACE_ROUNDS && !found; k++) {
      const int t = 32 * k + lane;
      const uint4 w = philox4x32_10(make_uint4((unsigned)env, counter, (unsigned)o, (unsigned)t), k0, k1);
      const double cx = __dadd_rn(__dadd_rn(p.x_min, __dmul_rn(wx, place_u53(w.x, w.y))), bx);
      const double cy = __dadd_rn(__dadd_rn(p.y_min, __dmul_rn(wy, place_u53(w.z, w.w))), by);
      bool ok = t < B2S_PLACE_TRIES;
      if (p.ensure_valid) {
        for (int j = 0; j < o; j++) {
          const double ox = __shfl_sync(B2S_FULL, px, j), oy = __shfl_sync(B2S_FULL, py, j), oz = __shfl_sync(B2S_FULL, pz, j);
          const PlaceDev& q = prog[j];
          const double dx = __dsub_rn(cx, ox), dy = __dsub_rn(cy, oy);
          const double d = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
          if (d <= __dadd_rn(q.radius, p.radius) && __dsub_rn(z, oz) <= __dsub_rn(q.top, p.bottom)) ok = false;
        }
      }
      const unsigned hit = __ballot_sync(B2S_FULL, ok);
      // no valid try at all: the environment keeps the last one (try B2S_PLACE_TRIES - 1)
      const int src = hit ? __ffs(hit) - 1 : (B2S_PLACE_TRIES - 1) - 32 * (B2S_PLACE_ROUNDS - 1);
      if (hit || k == B2S_PLACE_ROUNDS - 1) {
        x = __shfl_sync(B2S_FULL, cx, src);
        y = __shfl_sync(B2S_FULL, cy, src);
      }
      found = hit != 0;
    }
    failed |= !found;
    if (lane == o) { px = x; py = y; pz = z; }
    const uint4 w = philox4x32_10(make_uint4((unsigned)env, counter, (unsigned)o, 0xFFFFFFFFu), k0, k1);
    int c = 0;
    if (p.n_rot > 1) c = min((int)floor(__dmul_rn(place_u53(w.x, w.y), (double)p.n_rot)), p.n_rot - 1);
    const double ang = __dadd_rn(p.rot_min[c], __dmul_rn(__dsub_rn(p.rot_max[c], p.rot_min[c]), place_u53(w.z, w.w)));
    double sn, cs;
    place_sincos(__dmul_rn(ang, 0.5), &sn, &cs);
    const double q[4] = {cs, p.axis == 0 ? sn : 0.0, p.axis == 1 ? sn : 0.0, p.axis == 2 ? sn : 0.0};
    if (p.qpos_adr >= 0) {
      const double v[7] = {x, y, z, q[0], q[1], q[2], q[3]};
      if (lane < 7) qpos[(size_t)env * nq + p.qpos_adr + lane] = v[lane];
    } else if (lane < p.nov) {  // lane k writes override k
      const int k = lane;
      double P[3] = {x, y, z}, Q[4] = {q[0], q[1], q[2], q[3]};
      if (k > 0) {
        const double* lp = p.ov_lp[k];
        const double* lq = p.ov_lq[k];
        const double M[9] = {
          __dsub_rn(__dsub_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])), __dmul_rn(q[3], q[3])),
          __dmul_rn(2.0, __dsub_rn(__dmul_rn(q[1], q[2]), __dmul_rn(q[0], q[3]))),
          __dmul_rn(2.0, __dadd_rn(__dmul_rn(q[1], q[3]), __dmul_rn(q[0], q[2]))),
          __dmul_rn(2.0, __dadd_rn(__dmul_rn(q[1], q[2]), __dmul_rn(q[0], q[3]))),
          __dsub_rn(__dadd_rn(__dsub_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])), __dmul_rn(q[3], q[3])),
          __dmul_rn(2.0, __dsub_rn(__dmul_rn(q[2], q[3]), __dmul_rn(q[0], q[1]))),
          __dmul_rn(2.0, __dsub_rn(__dmul_rn(q[1], q[3]), __dmul_rn(q[0], q[2]))),
          __dmul_rn(2.0, __dadd_rn(__dmul_rn(q[2], q[3]), __dmul_rn(q[0], q[1]))),
          __dadd_rn(__dsub_rn(__dsub_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])), __dmul_rn(q[3], q[3]))};
        for (int r = 0; r < 3; r++)
          P[r] = __dadd_rn(P[r], __dadd_rn(__dadd_rn(__dmul_rn(M[3 * r], lp[0]), __dmul_rn(M[3 * r + 1], lp[1])), __dmul_rn(M[3 * r + 2], lp[2])));
        Q[0] = __dsub_rn(__dsub_rn(__dsub_rn(__dmul_rn(q[0], lq[0]), __dmul_rn(q[1], lq[1])), __dmul_rn(q[2], lq[2])), __dmul_rn(q[3], lq[3]));
        Q[1] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], lq[1]), __dmul_rn(q[1], lq[0])), __dmul_rn(q[2], lq[3])), __dmul_rn(q[3], lq[2]));
        Q[2] = __dadd_rn(__dadd_rn(__dsub_rn(__dmul_rn(q[0], lq[2]), __dmul_rn(q[1], lq[3])), __dmul_rn(q[2], lq[0])), __dmul_rn(q[3], lq[1]));
        Q[3] = __dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(q[0], lq[3]), __dmul_rn(q[1], lq[2])), __dmul_rn(q[2], lq[1])), __dmul_rn(q[3], lq[0]));
      }
      R* dp = reinterpret_cast<R*>(p.ov_pos[k]) + (size_t)env * 3;
      R* dq = reinterpret_cast<R*>(p.ov_quat[k]) + (size_t)env * 4;
      for (int r = 0; r < 3; r++) dp[r] = (R)P[r];
      for (int r = 0; r < 4; r++) dq[r] = (R)Q[r];
    }
  }
  if (lane == 0) pending[env] = failed ? B2S_PLACE_WARN : 0;
}
