// Unit-queue mode (b2s_set_mode(h, 2)): the whole control step of every environment as ONE persistent kernel.
//
// The phase pipeline (b2s_pipeline.cuh) runs a substep of an environment group as three kernels; every kernel lasts as long as its
// slowest environment (a deep EPA, a 9-iteration Newton solve), so a group's chain costs max(P0) + max(narrow) + max(tail) per substep
// although the mean environment needs a quarter of that, and the GPU idles in the bubbles.  Here the schedulable unit is ONE SUBSTEP OF
// ONE ENVIRONMENT: resident warps pull units from a ticket ring in global memory, run kinematics / dynamics / broad phase, the
// environment's own narrow phase, constraint rows, controller, Newton solve, integration (the very stage functions of the pipeline,
// with their per-phase shared-memory layouts placed in the warp's one workspace area), and push the environment back for its
// next substep.  Nothing waits for anybody else's slow item: an expensive environment delays only itself, and the ring hands the next
// ready environment to whichever warp is free (FIFO, so all environments advance at the same rate).
//
//   ring[t], t in [0, n_env * nsub): ticket t's environment, encoded env + n_env * substep; -1 = not produced yet.  Consumers take
//     tickets with atomicAdd(head) and wait for their slot; a finished unit with substeps left publishes the environment at
//     atomicAdd(tail).  One slot per ticket of the control step: no reuse, no ABA.
//   Environments whose contacts / constraint rows do not fit the small-tier layout go to a second ring served by the large-role
//     warps of blocks [0, n_large) (fewer warps per block, the full-capacity layout), exactly the two-tier scheme of the pipeline.
//   Memory ordering: a unit's state round-trips through global memory; the hand-over is st.release.gpu / ld.acquire.gpu on the ring
//     slot (plus a proxy fence in front of TMA reads of rows another warp wrote through the async proxy).
#pragma once
#include "b2s_pipeline.cuh"

struct UnitQ {
  int* ring;      // [total]
  int* ovf_ring;  // [total]
  int* ctr;       // [8]: 0 head ticket, 1 tail ticket, 2 finished units, 3 overflow head, 4 overflow tail
  int total, n_large, wpb_large;
  int stride, stride_large;  // words of shared memory per warp: small role / large role
#ifdef B2S_INSTR
  unsigned long long* prof;  // array "unit_prof" [16]: clock64 cycles per stage of the small role summed over the blocks' rounds
                             // (thread 0 of every block), [15] = rounds
#endif
};

DEV int ld_acquire_gpu(const int* p) { int v; asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
DEV int ld_relaxed_gpu(const int* p) { int v; asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
DEV void st_release_gpu(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
DEV void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

template <typename R> __global__ void unit_init_kernel(UnitQ q, int n_env) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < q.total) { q.ring[i] = i < n_env ? i : -1; q.ovf_ring[i] = -1; }
  if (i < 8) q.ctr[i] = i == 1 ? n_env : 0;
}

// after the persistent kernel: a watchdog event (ctr[7] != 0: a ticket never arrived, the blocks drained) means the control step is
// INCOMPLETE - flag every environment (warn bit 64) so that the caller sees it in info["sim_warn"] without a host sync
template <typename R> __global__ void unit_check_kernel(UnitQ q, int slot) {
  const DState<R>& s = cstate<R>(slot);
  if (q.ctr[7] == 0) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.n_env; i += gridDim.x * blockDim.x) s.warn[i] |= 64;
}

// ---- the stages of a unit: the shared stage functions of b2s_pipeline.cuh as separately compiled (noinline) functions.  The lockstep
// rounds of the small role put block barriers between them, and a kernel body that inlines all of it is the kind of function nvcc 12.9
// has mis-allocated before (DESIGN.md section 3).

// phase 0; the environment owns fixed output slots: analytic candidate i -> env * cl_maxa + i, convex candidate i -> env * cl_maxg + i.
// On the call's last substep (`last`) with b2s_set_step1_export, then the step-1 arrays, as in phase0_kernel.
template <typename R> DEVN int unit_phase0(R* area, int lane, int slot, int env, bool last) {
  const DState<R>& s = cstate<R>(slot);
  Eng<R> e(area, lane, slot, LAY_P0);
  int na, ng;
  const int warn = phase0_env(e, env, na, ng);
  phase0_publish(e, env, na, ng, warn, env * s.cl_maxa, env * s.cl_maxg, false);
  if (last && s.export_kin) export_kinematics(e, env);
  return na | (ng << 16);
}

// narrow phase of ONE environment by its own warp: analytic pairs one per lane, convex pairs one after the other with the warp's whole
// workspace area as EPA polytope + vertex staging scratch (phase 0's regions are in the global row by now)
template <typename R> DEVN void unit_narrow(R* area, int area_words, int lane, int slot, int env, int na, int ng) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  const WSLayout& RL = c_lay[slot][LAY_ROW];
  size_t E = env;
  const R* row = s.wsg + E * RL.total;
  const int* tab = s.cl_env + E * CL_ENVW(s);
  for (int base = 0; base < na; base += 32) {
    int i = base + lane;
    if (i < na) {
      R buf[8 * CREC];
      const int n = narrow_pair_analytic(m, s, env, tab[2 + 2 * i], row + RL.gpos, row + RL.gmat, buf);
      R* out = s.cl_outA + (E * s.cl_maxa + i) * CL_RECA;
      out[0] = R(n);
      for (int k = 0; k < n * CREC; k++) out[1 + k] = buf[k];
    }
  }
  __syncwarp();
  const int epa_words = EPA_AREA_WORDS(EPA_MAXV, EPA_MAXF), stage_cap = area_words - epa_words;
  for (int i = 0; i < ng; i++) {
    const int pidx = tab[2 + 2 * (s.cl_maxa + i)];
    R buf[CREC];
    const int n = narrow_pair_convex(m, s, env, pidx, row + RL.gpos, row + RL.gmat, buf, area, gjk_cache_of(m, s, env, pidx),
                                     stage_cap >= 64 ? area + epa_words : (R*)nullptr, stage_cap >= 64 ? stage_cap : 0, lane, false);
    if (lane == 0) {
      R* out = s.cl_outG + (E * s.cl_maxg + i) * 8;
      out[0] = R(n);
      for (int k = 0; k < CREC; k++) out[1 + k] = n ? buf[k] : R(0);
    }
    __syncwarp();
  }
  __syncwarp();
}

// the tail of a small-tier unit (the packed word of tail_rows, the warn bits of the dynamics)
template <typename R> DEVN int unit_tail_a(R* area, int lane, int slot, int env, unsigned long long* bar, unsigned& parity) {
  Eng<R> e(area, lane, slot, LAY_TS);
  return tail_rows(e, env, bar, parity);
}
template <typename R> DEVN void unit_tail_ctrl(R* area, int lane, int slot, int env, int sub, const R* action) {
  Eng<R> e(area, lane, slot, LAY_TS);
  tail_ctrl(e, env, sub, action);
}
template <typename R> DEVN int unit_tail_acc(R* area, int lane, int slot) {
  Eng<R> e(area, lane, slot, LAY_TS);
  return tail_accel(e);
}
template <typename R> DEVN int unit_tail_solve(R* area, int lane, int slot, int env, int nefc, int ncon) {
  Eng<R> e(area, lane, slot, LAY_TS);
  e.env = env;
  return tail_newton(e, nefc, ncon);
}
// the same two stages with the step-2 export (unit_kernel<R, true>): on the call's last substep (`last`) actuator_force, then after
// the solve the other step-2 arrays
template <typename R> DEVN int unit_tail_acc_dyn(R* area, int lane, int slot, int env, bool last) {
  Eng<R> e(area, lane, slot, LAY_TS);
  return tail_accel(e, tail_act_force_out(e, env, last));
}
template <typename R> DEVN int unit_tail_solve_dyn(R* area, int lane, int slot, int env, int nefc, int ncon, bool last) {
  Eng<R> e(area, lane, slot, LAY_TS);
  e.env = env;
  int niter;
  const int warn = tail_newton(e, nefc, ncon, &niter);
  if (last) export_dynamics(e, env, ncon, nefc, niter);
  return warn;
}
template <typename R>
DEVN void unit_tail_end(R* area, int lane, int slot, int env, int sub, int nsub, int phases, int ncon, int warn, unsigned long long* bar, unsigned& parity) {
  Eng<R> e(area, lane, slot, LAY_TS);
  tail_finish(e, env, sub, nsub, phases, ncon, warn, bar, parity);
}

// the unit is finished: hand the environment to whoever takes the next ticket (or count it as done after its last substep)
DEV void unit_finish(const UnitQ& q, int n_env, int env, int sub, int nsub, int lane) {
  __syncwarp();
  if (lane == 0) {
    __threadfence();
    if (sub + 1 < nsub) {
      int p = atomicAdd(q.ctr + 1, 1);
      st_release_gpu(q.ring + p, env + n_env * (sub + 1));
    }
    atomicAdd(q.ctr + 2, 1);
  }
  __syncwarp();
}


// One block of 16 warps per SM: what counts is that an SM executes ONE code region at a time (the hot code is ~10x the instruction
// cache).  Measured on 4096 Lift environments: 16 warps x 1 block 306 k env-steps/s, 8 warps x 2 blocks 248 k, 8 warps x 1 block 210 k,
// 4 warps x 4 blocks 158 k, free-running warps (no block barriers) 80 k.
constexpr int UNIT_THREADS = 512, UNIT_BLOCKS = 1;

// DYN: the step-2 export's instantiation (launched with PH_EXPORT_DYN; the other one has no writer code, see tail_act_force_out)
template <typename R, bool DYN>
__global__ void __launch_bounds__(UNIT_THREADS, UNIT_BLOCKS) unit_kernel(int phases, int nsub, const R* action, int slot, UnitQ q) {
  const DState<R>& s = cstate<R>(slot);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  R* smem = reinterpret_cast<R*>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_env = s.n_env;
  __shared__ unsigned long long mbar[32];
  if (lane == 0) mbar_init(&mbar[warp]);
  __syncwarp();
  unsigned parity = 0;
  if ((int)blockIdx.x < q.n_large) {
    // ---- large role: environments the small tier could not hold (phase 0 and the narrow phase are done; their results are in the row)
    if (warp >= q.wpb_large) return;
    R* area = smem + (size_t)warp * q.stride_large;
    for (;;) {
      int item = -1;
      if (lane == 0) {
        for (;;) {
          int h = ld_relaxed_gpu(q.ctr + 3), t = ld_acquire_gpu(q.ctr + 4);
          if (h < t) { if (atomicCAS(q.ctr + 3, h, h + 1) == h) { item = h; break; } continue; }
          if (ld_acquire_gpu(q.ctr + 2) >= q.total || ld_relaxed_gpu(q.ctr + 7) != 0) break;
          __nanosleep(400);
        }
      }
      item = __shfl_sync(B2S_FULL, item, 0);
      if (item < 0) break;
      int code = 0;
      if (lane == 0) { while ((code = ld_acquire_gpu(q.ovf_ring + item)) < 0) __nanosleep(100); }
      code = __shfl_sync(B2S_FULL, code, 0);
      __syncwarp();
      fence_proxy_async_all();  // the row was written through the async proxy of another SM
      const int env = code % n_env, sub = code / n_env;
      Eng<R> e(area, lane, slot, LAY_TL);
      const int pk = tail_rows(e, env, &mbar[warp], parity);  // the full-capacity layout holds every environment: no overflow
      const int ncon = TAIL_NCON(pk);
      int warn = TAIL_WARN(pk);
      if (phases & PH_CTRL) tail_ctrl(e, env, sub, action);
      if constexpr (DYN) {
        warn |= tail_accel(e, tail_act_force_out(e, env, sub == nsub - 1));
        int niter;
        warn |= tail_newton(e, TAIL_NEFC(pk), ncon, &niter);
        if (sub == nsub - 1) export_dynamics(e, env, ncon, TAIL_NEFC(pk), niter);
      } else {
        warn |= tail_accel(e);
        warn |= tail_newton(e, TAIL_NEFC(pk), ncon);
      }
      tail_finish(e, env, sub, nsub, phases, ncon, warn, &mbar[warp], parity);
      unit_finish(q, n_env, env, sub, nsub, lane);
    }
    return;
  }
  // ---- small role: the block takes `wpb` consecutive tickets per round and walks them through the stages in LOCKSTEP (block barriers
  // between the stages).  Free-running warps - every warp of an SM somewhere else in 300 KB of SASS - missed the instruction cache
  // on nearly every fetch (measured: 1.1 ms per unit against ~0.2 ms of work); in lockstep an SM executes one or two code regions at
  // a time, like the phase kernels, and a stage costs the slowest of the block's 8 units (1.0-1.3x the mean) instead of the slowest
  // of a 512-environment launch (2.5x).
  const int wpb = blockDim.x >> 5;
  __shared__ int sh_t0, sh_k;
  R* area = smem + (size_t)warp * q.stride;
#ifdef B2S_INSTR
#define UTICK(k) if (threadIdx.x == 0) { long long tn_ = clock64(); atomicAdd(q.prof + (k), (unsigned long long)(tn_ - tprev)); tprev = tn_; }
  long long tprev = clock64();
#else
#define UTICK(k)
#endif
  for (;;) {
    // the block takes up to `wpb` tickets that are ALREADY PRODUCED (head < tail).  The first lockstep version took `wpb` tickets
    // whether they existed or not and waited for the missing ones in front of the first stage barrier: every control step stalled until
    // the watchdog on the GPU (the ticket arithmetic itself terminates: tests/test_unit_queue_protocol.py).  No wait inside a round now.
    __syncthreads();
    if (threadIdx.x == 0) {
      int t0v = 0x7fffffff, k = 0, spins = 0;
      for (;;) {
        if (ld_relaxed_gpu(q.ctr + 7) != 0) break;
        const int H = ld_relaxed_gpu(q.ctr);
        if (H >= q.total) break;
        const int P = ld_acquire_gpu(q.ctr + 1);
        if (H < P) {
          k = min(wpb, P - H);
          if (atomicCAS(q.ctr, H, H + k) == H) { t0v = H; break; }
          k = 0;
          continue;
        }
        __nanosleep(100);
        if (++spins > (1 << 22)) { atomicCAS(q.ctr + 7, 0, 2); break; }
      }
      sh_t0 = t0v; sh_k = k;
    }
    __syncthreads();
    const int t0 = sh_t0;
    if (t0 == 0x7fffffff) break;
    UTICK(0)
#ifdef B2S_INSTR
    if (threadIdx.x == 0) atomicAdd(q.prof + 15, 1ull);
#endif
    const int t = warp < sh_k ? t0 + warp : q.total;
    bool live = t < q.total;
    int code = 0;
    if (live) {
      if (lane == 0) {
        // watchdog: a ticket that is not produced within ~0.5 s means the ring protocol is broken - flag it (ctr[7], with the ticket
        // and the ring counters beside it) and let every block drain instead of hanging the device
        int spins = 0;
        while ((code = ld_acquire_gpu(q.ring + t)) < 0) {
          __nanosleep(64);
          if (++spins > (1 << 22) || ((spins & 1023) == 0 && ld_relaxed_gpu(q.ctr + 7) != 0)) {
            if (atomicCAS(q.ctr + 7, 0, 1) == 0) { q.ctr[5] = t; q.ctr[6] = ld_relaxed_gpu(q.ctr + 1); }
            break;
          }
        }
      }
      code = __shfl_sync(B2S_FULL, code, 0);
      __syncwarp();
      if (code < 0) { live = false; code = 0; }
    }
    const int env = code % n_env, sub = code / n_env;
    __syncthreads();
    UTICK(1)
    int nn = 0;
    if (live) nn = unit_phase0<R>(area, lane, slot, env, sub == nsub - 1);
    __syncthreads();
    UTICK(2)
    if (live) unit_narrow<R>(area, q.stride, lane, slot, env, nn & 0xffff, nn >> 16);
    __syncthreads();
    UTICK(3)
    int warn = 0, ncon = 0, nefc = 0;
    if (live) {
      const int pk = unit_tail_a<R>(area, lane, slot, env, &mbar[warp], parity);
      ncon = TAIL_NCON(pk); nefc = TAIL_NEFC(pk); warn = TAIL_WARN(pk);
      if (TAIL_OVF(pk)) {  // does not fit the small tier: to the large-role warps, nothing of the state has been touched
        if (lane == 0) {
          __threadfence();
          int p = atomicAdd(q.ctr + 4, 1);
          st_release_gpu(q.ovf_ring + p, code);
        }
        __syncwarp();
        live = false;
      }
    }
    __syncthreads();
    UTICK(4)
    if (live && (phases & PH_CTRL)) unit_tail_ctrl<R>(area, lane, slot, env, sub, action);
    __syncthreads();
    UTICK(5)
    if constexpr (DYN) { if (live) warn |= unit_tail_acc_dyn<R>(area, lane, slot, env, sub == nsub - 1); }
    else if (live) warn |= unit_tail_acc<R>(area, lane, slot);
    __syncthreads();
    UTICK(6)
    if constexpr (DYN) { if (live) warn |= unit_tail_solve_dyn<R>(area, lane, slot, env, nefc, ncon, sub == nsub - 1); }
    else if (live) warn |= unit_tail_solve<R>(area, lane, slot, env, nefc, ncon);
    __syncthreads();
    UTICK(7)
    if (live) {
      unit_tail_end<R>(area, lane, slot, env, sub, nsub, phases, ncon, warn, &mbar[warp], parity);
      unit_finish(q, n_env, env, sub, nsub, lane);
    }
    UTICK(8)
  }
#undef UTICK
}
