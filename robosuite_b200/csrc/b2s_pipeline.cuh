// Pipeline mode: one substep = phase 0 (kinematics + dynamics + broad phase) | work-list narrow phase (analytic, convex) beside the
// thread-per-environment controller kernel | tail (contact gather, constraint rows, solve, integrate, observations), exchanging a
// per-environment workspace row through L2.  Same device functions as the fused kernel (the narrow phase of one pair included,
// b2s_collide.cuh), and the stage sequences (phase 0, the tail stages) are defined here once for this pipeline and the unit queue; what
// changes is scheduling and MEMORY:
// every kernel has its own compact shared-memory layout (LAY_P0 / LAY_TS / LAY_TL), so 24-28 warps are resident per SM instead of
// the 14 the one-size-fits-all layout allowed, and the tail runs in two capacity tiers: the small tier holds the contact / row counts
// almost every environment has, the few that need more are re-run by the large tier in the same block (same results, no truncation).
#pragma once
#include "b2s_kernel.cuh"

// ---- TMA 1-D bulk copies (SASS: UBLKCP).  One elected lane per warp issues the copies; completion of loads is signalled on
// the warp's mbarrier (transaction bytes), stores are tracked with a bulk async-group.
DEV unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
DEV void mbar_init(unsigned long long* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
DEV void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
DEV void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
DEV void tma_load_1d(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
DEV void tma_store_1d(void* gdst, const void* smem_src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

// Every region of a phase's load / store list is 16-byte aligned in both its shared-memory and its global-row offset and in its
// length (build_layouts); regions adjacent on both sides are merged into spans on the host, so a phase moves its workspace with
// a handful of bulk copies: lane k issues span k.
template <typename R> DEV void ws_load(const Eng<R>& e, const R* row, const PhaseIO& io, unsigned long long* bar, unsigned& parity) {
  if (io.nload == 0) return;
  // the destination may have been read / written through the generic proxy before (the constraint Jacobian under the late poses, the
  // previous environment of a large-tier warp): order those accesses before the async-proxy writes of the bulk copies
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();
  if (e.lane == 0) mbar_expect_tx(bar, (unsigned)io.load_words * (unsigned)sizeof(R));
  __syncwarp();
  if (e.lane < io.nload) {
    Region r = io.load[e.lane];
    tma_load_1d(e.ws + r.off, row + r.goff, (unsigned)r.len * sizeof(R), bar);
  }
  mbar_wait(bar, parity);
  parity ^= 1u;
}
template <typename R> DEV void ws_store(const Eng<R>& e, R* row, const PhaseIO& io) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // this lane's generic-proxy writes -> visible to the async proxy
  __syncwarp();
  if (e.lane < io.nstore) {
    Region r = io.store[e.lane];
    tma_store_1d(row + r.goff, e.ws + r.off, (unsigned)r.len * sizeof(R));
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
  __syncwarp();
}

// A launch covers one group of environments [env0, env0 + nenv); groups run on separate streams so that the tail of one
// group's kernel (its slowest environment) overlaps with other groups' work.  slot = descriptor slot of the owning handle.
struct Grp { int env0, nenv, gid, sub, slot; };
// this group's counters: nA, nG, (spare), next convex item.  phase0_kernel(s) appends, phase1_kernel(s) consumes, tail_kernel(s) zeroes
// them at entry for phase0_kernel(s + 1); the memset at the head of the group's graph zeroes them for substep 0
#define CLC(s, g) ((s).cl_cnt + CL_CNT_STRIDE * (g).gid)
// then the environments per tail cost class, one set per substep parity: phase0_kernel(s) counts into set s & 1, every block of
// tail_kernel(s) reads it, tail_kernel(s) zeroes set (s + 1) & 1 for phase0_kernel(s + 1); the head memset zeroes both
#define CLK(s, g, sub) (CLC(s, g) + 8 + TAIL_NKEY * ((sub) & 1))

// Tail cost class of an environment-substep, 0 .. TAIL_NKEY - 1 (most expensive last), from its deterministic counts: Newton
// iterations, constraint rows, and whether it needed the full-capacity tier.  Fitted against the INSTR build's recorded tail cycles
// (tools/probe_tail_order.py, DESIGN.md section 6); the probe repeats this formula.
DEV int tail_cost_key(int niter, int nefc, bool large) {
  return large ? TAIL_NKEY - 1 : min(TAIL_NKEY - 2, (niter * (nefc + 24) + 2 * nefc) / 48);
}

// -DB2S_INSTR: every launch stamps its first / last %globaltimer into st_begin / st_end (device timeline of the CUDA-graph
// replay, which events cannot subdivide), warps record their clock64 cost per environment-substep.  Empty in product builds.
#ifdef B2S_INSTR
DEV unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define INSTR_SLOT(g, kind) ((((g).gid & 63) * 32 + ((g).sub & 31)) * 8 + (kind))
#define INSTR_BEGIN(st, g, kind) if (threadIdx.x == 0 && (st).st_begin) atomicMin((st).st_begin + INSTR_SLOT(g, kind), gtimer());
#define INSTR_END(st, g, kind) if ((threadIdx.x & 31) == 0 && (st).st_end) atomicMax((st).st_end + INSTR_SLOT(g, kind), gtimer());
#else
#define INSTR_BEGIN(st, g, kind)
#define INSTR_END(st, g, kind)
#endif
#include "b2s_ctrlkernel.cuh"

// ---- phase 1: the three consumers of phase 0's outputs in ONE launch (block roles) -----------------------------------------------
// Controller, convex and analytic narrow phase are independent of each other.  As separate graph nodes on forked streams they
// serialised the environment groups (measured: any fork inside the captured graph halves the throughput); as roles of one kernel
// node they overlap with no fork: blocks [0, nG) convex narrow phase, [nG, nG + nC) controller, the rest analytic narrow phase -
// the role with the longest single work item (a deep EPA) is scheduled first.  Every block is one warp.
struct P1Cfg { int nG, nC, sub; };

// the convex pair's GJK warm-start direction (the separating direction of its last test in this environment), nullptr without the cache
template <typename R> DEV R* gjk_cache_of(const DModel<R>& m, const DState<R>& s, int env, int pidx) {
  return s.gjk_cache ? s.gjk_cache + ((size_t)env * m.npair + pidx) * 3 : (R*)nullptr;
}

// analytic pairs: ONE THREAD per candidate pair of any environment (32 different pairs per warp)
template <typename R> DEV void narrow_analytic_block(const Grp& g, int rb) {
  const DState<R>& s = cstate<R>(g.slot);
  const WSLayout& RL = c_lay[g.slot][LAY_ROW];
  int tid = rb * 32 + threadIdx.x;
  if (tid >= CLC(s, g)[0]) return;
  tid += g.env0 * s.cl_maxa;  // this group's slice of the candidate list / output slots
  int code = s.cl_listA[tid];
  int env = code >> 12;
  const R* row = s.wsg + (size_t)env * RL.total;
  R buf[8 * CREC];
  const int n = narrow_pair_analytic(cmodel<R>(g.slot), s, env, code & 4095, row + RL.gpos, row + RL.gmat, buf);
  R* out = s.cl_outA + (size_t)tid * CL_RECA;
  out[0] = R(n);
  for (int k = 0; k < n * CREC; k++) out[1 + k] = buf[k];
}

// convex pairs: ONE WARP per candidate pair (mesh support scans split over the lanes).  The block owns one EPA polytope and the
// vertex staging area in shared memory; warps claim work items through an atomic counter, so the few expensive pairs (penetrating
// meshes: tens of EPA expansions) never hold idle neighbours resident.
template <typename R> DEV void narrow_convex_block(const Grp& g, unsigned char* smem_raw) {
  const DModel<R>& m = cmodel<R>(g.slot);
  const DState<R>& s = cstate<R>(g.slot);
  const WSLayout& RL = c_lay[g.slot][LAY_ROW];
  int lane = threadIdx.x & 31;
  R* scratch = reinterpret_cast<R*>(smem_raw);
  const int cnt = CLC(s, g)[1];
  while (true) {
    int item = 0;
    if (lane == 0) item = atomicAdd(CLC(s, g) + 3, 1);
    item = __shfl_sync(B2S_FULL, item, 0);
    if (item >= cnt) break;
    int wid = item + g.env0 * s.cl_maxg;
    int code = s.cl_listG[wid], env = code >> 12, pidx = code & 4095;
    const R* row = s.wsg + (size_t)env * RL.total;
    R buf[CREC];
    const int n = narrow_pair_convex(m, s, env, pidx, row + RL.gpos, row + RL.gmat, buf, scratch, gjk_cache_of(m, s, env, pidx),
                                     m.stage_cap > 0 ? scratch + EPA_AREA_WORDS(EPA_MAXV, EPA_MAXF) : (R*)nullptr, m.stage_cap, lane, true);
    if (lane == 0) {
      R* out = s.cl_outG + (size_t)wid * 8;
      out[0] = R(n);
      for (int k = 0; k < CREC; k++) out[1 + k] = n ? buf[k] : R(0);
    }
    __syncwarp();
  }
}

template <typename R>
__global__ void __launch_bounds__(32) phase1_kernel(const R* action, Grp g, P1Cfg c) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
#ifdef B2S_INSTR
  const DState<R>& s = cstate<R>(g.slot);
  const int kind = b < c.nG ? 2 : (b < c.nG + c.nC ? 4 : 1);
  INSTR_BEGIN(s, g, kind)
#endif
  if (b < c.nG) narrow_convex_block<R>(g, smem_raw);
  else if (b < c.nG + c.nC) ctrl_osc_block<R>(g.sub, action, g.env0, g.nenv, g.gid, g.slot, smem_raw, b - c.nG);
  else narrow_analytic_block<R>(g, b - c.nG - c.nC);
#ifdef B2S_INSTR
  INSTR_END(s, g, kind)
#endif
}

// collect this environment's contacts from the work-list outputs, in static-pair order (what the fused collide produces)
template <typename R> DEVN int gather_contacts(Eng<R> e, int env, int& warn) {
  const DModel<R>& m = e.model();
  const DState<R>& s = e.state();
  const WSLayout& L = e.lay();
  int lane = e.lane;
  const int* tab = s.cl_env + (size_t)env * CL_ENVW(s);
  int na = tab[0], ng = tab[1], nc = na + ng;  // nc <= CL_MAXA + CL_MAXG = 96: up to IT candidates per lane
  const int IT = 3;
  int nchunk = (nc + 31) >> 5;
  int pairv[IT], slotv[IT], isgv[IT], cntv[IT], offv[IT];
#pragma unroll
  for (int it = 0; it < IT; it++) {
    int j = lane + 32 * it;
    pairv[it] = 0x7fffffff; slotv[it] = 0; isgv[it] = 0; cntv[it] = 0; offv[it] = 0;
    if (j < na) { pairv[it] = tab[2 + 2 * j]; slotv[it] = tab[3 + 2 * j]; cntv[it] = (int)s.cl_outA[(size_t)slotv[it] * CL_RECA]; }
    else if (j < nc) {
      int k = j - na;
      isgv[it] = 1; pairv[it] = tab[2 + 2 * (s.cl_maxa + k)]; slotv[it] = tab[3 + 2 * (s.cl_maxa + k)];
      cntv[it] = (int)s.cl_outG[(size_t)slotv[it] * 8];
    }
  }
  // contact offset = contacts of candidates with a smaller pair index
  int total = 0;
#pragma unroll
  for (int it2 = 0; it2 < IT; it2++) {
    if (it2 >= nchunk) break;
    int lim = nc - 32 * it2 < 32 ? nc - 32 * it2 : 32;
    for (int o = 0; o < lim; o++) {
      int op = __shfl_sync(B2S_FULL, pairv[it2], o), on = __shfl_sync(B2S_FULL, cntv[it2], o);
      total += on;
#pragma unroll
      for (int it = 0; it < IT; it++)
        if (op < pairv[it]) offv[it] += on;
    }
  }
  if (total > L.mc) { warn |= 4; if (L.mc < m.maxcon) return L.mc; }  // small tier: the caller hands the environment to the large tier
  R* cpos = e.p(L.c_pos); R* cfr = e.p(L.c_frame); R* cdist = e.p(L.c_dist);
  int* cint = e.pi(L.c_int);
#pragma unroll
  for (int it = 0; it < IT; it++) {
    if (lane + 32 * it >= nc) continue;
    int pair = pairv[it], slot = slotv[it], n = cntv[it], off = offv[it];
    const R* rec = isgv[it] ? s.cl_outG + (size_t)slot * 8 + 1 : s.cl_outA + (size_t)slot * CL_RECA + 1;
    int g1, g2;
    pair_geoms(m, pair, g1, g2);
    for (int k = 0; k < n; k++) {
      int c = off + k;
      if (c >= L.mc) break;
      const R* b = rec + CREC * k;
      cpos[3 * c] = b[0]; cpos[3 * c + 1] = b[1]; cpos[3 * c + 2] = b[2];
      cfr[3 * c] = b[3]; cfr[3 * c + 1] = b[4]; cfr[3 * c + 2] = b[5];
      cdist[c] = b[6];
      cint[5 * c] = g1; cint[5 * c + 1] = g2; cint[5 * c + 4] = pair;
    }
  }
  if (total > L.mc) total = L.mc;
  __syncwarp();
  finish_contacts(e, total);
  return total;
}

// ---- the stages of one environment-substep.  The phase kernels and the unit queue both run these; they differ only in how they hand
// environments to warps.  Each stage is inlined into its caller (the inline boundaries decide register allocation and FMA contraction).

// phase 0 up to the broad phase: state rows in, kinematics, velocity stage + RNE bias, CRB -> M, collision candidates (in the
// layout's scratch: analytic, then convex at +96) clamped to the candidate-list capacities.  Returns the warn bits.
template <typename R> DEV int phase0_env(Eng<R>& e, int env, int& na, int& ng) {
  const DModel<R>& m = e.model();
  const DState<R>& s = e.state();
  const WSLayout& L = e.lay();
  const int lane = e.lane;
  const size_t E = env;
  e.env = env;
  load_row(e.p(L.qpos), s.qpos + E * m.nq, m.nq, lane);
  load_row(e.p(L.qvel), s.qvel + E * m.nv, m.nv, lane);
  __syncwarp();
  const int was_reset = e.kinematics();
  if (was_reset) {  // diverged state reset to the model defaults (mj_checkPos / mj_checkVel): the tail reads the state from global memory
    for (int i = lane; i < m.nq; i += 32) s.qpos[E * m.nq + i] = e.p(L.qpos)[i];
    for (int i = lane; i < m.nv; i += 32) { s.qvel[E * m.nv + i] = 0; s.qacc[E * m.nv + i] = 0; s.qacc_ws[E * m.nv + i] = 0; }
    if (lane == 0) s.time[env] = 0;
    __syncwarp();
  }
  e.velocity();
  e.crb();
  int* cand = e.pi(L.scratch);
  int warn = was_reset;
  cull_pairs(e, cand, cand + 96, s.cl_maxa, s.cl_maxg, na, ng);
  if (na > s.cl_maxa) { na = s.cl_maxa; warn |= 4; }
  if (ng > s.cl_maxg) { ng = s.cl_maxg; warn |= 4; }
  return warn;
}

// end of phase 0: the environment's candidate table (pair index and output slot: analytic candidate i -> baseA + i, convex i -> baseG + i),
// the warn word of the row header, phase 0's workspace regions -> the row.  worklist: the candidates also go to the group's work lists.
template <typename R> DEV void phase0_publish(const Eng<R>& e, int env, int na, int ng, int warn, int baseA, int baseG, bool worklist) {
  const DState<R>& s = e.state();
  const WSLayout& L = e.lay();
  const WSLayout& RL = c_lay[e.slot][LAY_ROW];
  const int lane = e.lane;
  const size_t E = env;
  const int* cand = e.pi(L.scratch);
  const int* cand_g = cand + 96;
  int* tab = s.cl_env + E * CL_ENVW(s);
  if (lane == 0) { tab[0] = na; tab[1] = ng; }
  for (int i = lane; i < na; i += 32) {
    if (worklist) s.cl_listA[baseA + i] = (env << 12) | cand[i];
    tab[2 + 2 * i] = cand[i]; tab[3 + 2 * i] = baseA + i;
  }
  for (int i = lane; i < ng; i += 32) {
    if (worklist) s.cl_listG[baseG + i] = (env << 12) | cand_g[i];
    tab[2 + 2 * (s.cl_maxa + i)] = cand_g[i]; tab[3 + 2 * (s.cl_maxa + i)] = baseG + i;
  }
  R* row = s.wsg + E * RL.total;
  if (lane == 0) reinterpret_cast<int*>(row + RL.hdr)[2] = warn;
  __syncwarp();
  ws_store(e, row, c_pio[e.slot][PIO_P0]);
}

// The tail stages take the engine of the tier's layout (LAY_TS / LAY_TL).
// Rows: workspace regions and state rows in, contacts gathered from the narrow-phase outputs, constraint rows, and whether the
// environment fits this tier (if not, nothing of its state has been touched).  Returns the packed word below; nefc <= the layout's row
// capacity, far below 2^14 in any layout that fits shared memory.
#define TAIL_NCON(pk) ((pk) & 255)
#define TAIL_WARN(pk) (((pk) >> 8) & 255)
#define TAIL_NEFC(pk) (((pk) >> 16) & 0x3fff)
#define TAIL_OVF(pk) ((pk) >> 30)
template <typename R> DEV int tail_rows(Eng<R>& e, int env, unsigned long long* bar, unsigned& parity) {
  const DModel<R>& m = e.model();
  const DState<R>& s = e.state();
  const WSLayout& L = e.lay();
  const WSLayout& RL = c_lay[e.slot][LAY_ROW];
  const int lane = e.lane;
  const bool tiered = L.mc < m.maxcon || L.me < m.maxefc;
  const size_t E = env;
  e.env = env;
  const R* row = s.wsg + E * RL.total;
  const int warn = reinterpret_cast<const int*>(row + RL.hdr)[2];  // phase 0: divergence reset, candidate-list overflow
  ws_load(e, row, c_pio[e.slot][e.lid == LAY_TL ? PIO_TL : PIO_TS], bar, parity);
  load_row(e.p(L.qpos), s.qpos + E * m.nq, m.nq, lane);
  load_row(e.p(L.qvel), s.qvel + E * m.nv, m.nv, lane);
  load_row(e.p(L.ctrl), s.ctrl + E * m.nu, m.nu, lane);
  load_row(e.p(L.qacc_ws), s.qacc_ws + E * m.nv, m.nv, lane);
  __syncwarp();
  int wl = 0;
  const int ncon = gather_contacts(e, env, wl);
  const int nefc = (tiered && (wl & 4)) ? 0 : make_constraint(e, ncon, wl);
  wl = warp_or_i(wl);  // make_constraint flags a dropped contact on the lane that owns it: the verdict must be warp-uniform
  const int ovf = (tiered && (wl & 12)) ? 1 : 0;
  return (ncon & 255) | (((warn | wl) & 255) << 8) | ((nefc & 0x3fff) << 16) | (ovf << 30);
}

// Controller run inside the tail (JV / joint controllers; OSC when it is not a phase-1 role): ctrl -> global memory
template <typename R> DEV void tail_ctrl(Eng<R>& e, int env, int sub, const R* action) {
  const DModel<R>& m = e.model();
  const DState<R>& s = e.state();
  const WSLayout& L = e.lay();
  const size_t E = env;
  CtrlState<R> cs;
  ctrl_load(e, cs, env);
  ctrl_run(e, cs, env, sub == 0 ? action : (const R*)nullptr);
  for (int i = e.lane; i < m.nu; i += 32) s.ctrl[E * m.nu + i] = e.p(L.ctrl)[i];
  if (sub == 0) ctrl_store(e, cs, env);
  __syncwarp();
}

// Dynamics, in two parts (the unit queue puts a block barrier between them): actuation + smooth acceleration, then the Newton solve.
// Both return warn bits; the solve also reports its Newton iterations.  act_force_out: where actuation writes actuator_force (the
// step-2 export's last substep), nullptr otherwise.
template <typename R> DEV int tail_accel(Eng<R>& e, R* act_force_out = nullptr) {
  e.actuation(act_force_out);
  return e.acceleration() ? 1 : 0;
}
template <typename R> DEV int tail_newton(Eng<R>& e, int nefc, int ncon, int* niter = nullptr) {
  int warn = 0;
  const int it = solve(e, nefc, ncon, warn);
  if (niter) *niter = it;
  return warn;
}

// The step-2 export (b2s_set_step2_export) in the tail: on the call's last substep, actuation writes actuator_force and, right after
// the solve (before Euler and before tail_finish's late pose load overlays J), export_dynamics writes the rest; only the tier that
// finishes the environment gets there.  The tail kernels and the unit queue have an instantiation with it (DYN, launched with
// PH_EXPORT_DYN) and one without, whose code is the tail's as it was before the export existed: with the writer compiled in but not
// called, NutAssemblyRound's pipeline ran 1.2 % slower (DESIGN.md section 6).
template <typename R> DEV R* tail_act_force_out(const Eng<R>& e, int env, bool last) {
  return last ? e.state().actuator_force + (size_t)env * e.model().nu : (R*)nullptr;
}

// Finish: on the last substep of the call the contact records (b2s_set_contact_export), Euler, the rows of the observables that
// sample on this substep (obs_due: all of them on the last substep without modifiers), on the last substep of a control step the
// task rows, state write-back.  Only the tier that finishes the environment gets here: a small-tier overflow returned before touching
// anything.
template <typename R>
DEV void tail_finish(Eng<R>& e, int env, int sub, int nsub, int phases, int ncon, int warn, unsigned long long* bar, unsigned& parity) {
  const DState<R>& s = e.state();
  // first in the stage (after the call the caller keeps fewer values live than at the end: measured with -Xptxas -v)
  if (s.export_con && sub == nsub - 1) export_contacts(e, env, ncon);
  e.env = env;  // Euler reads the environment's damping
  R time = s.time[env];
  if (!(phases & PH_NOINTEGRATE)) {
    { int eb = e.euler(&time); if (eb & 32) warn |= 32; else if (eb) warn |= 2; }
  }
  if ((phases & PH_OBS) && e.ccfg().obs_dim > 0) {
    // The reference's observables sample on the LAST substep of a control step at the default rate: reset()'s forced update
    // already advances their period timer by one model timestep (utils/observables.py:214-259, environments/base.py:418-427),
    // so the period closes after substep 24 and the next update - substep 25 - takes the sample.  Other rates: obs_due.
    const bool last = sub == nsub - 1, only_fresh = (phases & PH_NOINTEGRATE) != 0;
    const unsigned due = obs_due(e, env, last, only_fresh);
    // Body / site poses of this substep's step1 arrive now, over the (dead) constraint Jacobian (`due` is warp-uniform).
    if (due || last)
      ws_load(e, s.wsg + (size_t)env * c_lay[e.slot][LAY_ROW].total, c_pio[e.slot][e.lid == LAY_TL ? PIO_TL_LATE : PIO_TS_LATE], bar, parity);
    if (due) write_obs(e, env, only_fresh, due);
    if (last) write_task(e, env, ncon);
  }
  store_state(e, env, time, warn);
}

// Launch bounds (threads per block, resident blocks per SM the register allocation is sized for).  (256, 2) = 128 registers per
// thread: with (256, 3) = 80 registers the heavily spilling build mis-executed solve() on 21-dof models (a corrupted workspace
// pointer, found with compute-sanitizer) - the same family of nvcc 12.9 stack-slot problems as DESIGN.md section 3 records.
// The kernels are latency bound at 4096 environments (every environment's warp is resident either way), so the lost occupancy
// costs nothing measurable (256 x 2 was the fastest of the launch-bound variants measured for phase 0).
// The tail has a second block shape, ONE block of 16 warps per SM, (512, 1), also 128 registers: such a block takes the whole register
// file, so an SM executes one tail block and nothing else until the block is done, instead of two 8-warp blocks (often of different
// substeps or groups) beside 1-warp phase-1 blocks.  choose_blocks (b2s_capi.cu) says which shape a model gets.
constexpr int P0_THREADS = 256, P0_BLOCKS = 2;      // phase 0
constexpr int TAIL_THREADS = 256, TAIL_BLOCKS = 2;  // tail kernel, two blocks per SM
constexpr int TAIL_WIDE_THREADS = 512;              // tail kernel, one block per SM

// ---- phase 0: kinematics, velocity stage + RNE bias, CRB -> M, broad phase -> global candidate work lists; with PH_LAST_SUB in
// `phases` and b2s_set_step1_export, the step-1 arrays
template <typename R>
__global__ void __launch_bounds__(P0_THREADS, P0_BLOCKS) phase0_kernel(int phases, Grp g) {
  const DState<R>& s = cstate<R>(g.slot);
  const WSLayout& L = c_lay[g.slot][LAY_P0];
  extern __shared__ __align__(16) unsigned char smem_raw[];
  R* smem = reinterpret_cast<R*>(smem_raw);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  int env = blockIdx.x * wpb + warp;
  INSTR_BEGIN(s, g, 0)
#ifdef B2S_INSTR
  long long instr_t0 = clock64();
#endif
  if (env >= g.nenv) return;
  env += g.env0;
  Eng<R> e(smem + (size_t)warp * L.total, lane, g.slot, LAY_P0);
  int na, ng;
  const int warn = phase0_env(e, env, na, ng);
  // output slots of the candidates: appended to the group's work lists (slots by warp-aggregated atomics)
  int baseA = 0, baseG = 0;
  if (lane == 0) {
    if (na) baseA = g.env0 * s.cl_maxa + atomicAdd(CLC(s, g), na);
    if (ng) baseG = g.env0 * s.cl_maxg + atomicAdd(CLC(s, g) + 1, ng);
    if (s.tail_sorted) {  // the environment's cost class of its last tail files it for this substep's tail (tail_env_at)
      const int k = s.tail_key[env];
      s.tail_list[(size_t)g.env0 * TAIL_NKEY + k * g.nenv + atomicAdd(CLK(s, g, g.sub) + k, 1)] = env;
    }
  }
  baseA = __shfl_sync(B2S_FULL, baseA, 0);
  baseG = __shfl_sync(B2S_FULL, baseG, 0);
  phase0_publish(e, env, na, ng, warn, baseA, baseG, true);
  // the call's last substep (its graph node carries PH_LAST_SUB): the step-1 arrays, last in the kernel, where the fewest values are live
  if ((phases & PH_LAST_SUB) && s.export_kin) export_kinematics(e, env);
#ifdef B2S_INSTR
  if (lane == 0 && s.cyc) s.cyc[((size_t)env * 32 + (g.sub & 31)) * 8] = (float)(clock64() - instr_t0);
#endif
  INSTR_END(s, g, 0)
}

// The environment at warp position p of the group's tail launch.  The group's environments are ranked by the cost classes phase 0
// filed them under, most expensive first, in filing order within a class.  Low positions are the blocks the scheduler starts first,
// so the expensive environments share blocks (a block holds its SM until its slowest warp is done) and start early.  The first
// TAIL_SOLO blocks are the exception: warp 0 of block b takes rank b and the block's other warps the cheapest ranks, so the launch's
// most expensive environments run beside warps that are soon done instead of beside other expensive ones (the launch, and with it
// the group's chain, ends with its slowest environment).
template <typename R> DEV int tail_env_at(const Grp& g, int p, int lane) {
  const DState<R>& s = cstate<R>(g.slot);
  const int wpb = blockDim.x >> 5;
  if (TAIL_SOLO * wpb <= g.nenv) {  // p -> rank
    const int b = p / wpb, w = p - b * wpb;
    if (b >= TAIL_SOLO) p -= TAIL_SOLO * (wpb - 1);
    else p = w == 0 ? b : g.nenv - 1 - (b * (wpb - 1) + w - 1);
  }
  const int cnt = lane < TAIL_NKEY ? CLK(s, g, g.sub)[TAIL_NKEY - 1 - lane] : 0;
  int incl = cnt;
#pragma unroll
  for (int d = 1; d < TAIL_NKEY; d <<= 1) {
    const int v = __shfl_up_sync(B2S_FULL, incl, d);
    if (lane >= d) incl += v;
  }
  const int c = __ffs(__ballot_sync(B2S_FULL, incl > p)) - 1;  // a lane below TAIL_NKEY: the counts of the group sum to nenv > rank p
  const int rank = p - __shfl_sync(B2S_FULL, incl - cnt, c);
  return s.tail_list[(size_t)g.env0 * TAIL_NKEY + (TAIL_NKEY - 1 - c) * g.nenv + rank];
}

// ---- tail: gather contacts, constraint rows + Jacobian, (in-kernel controller), actuation, Newton solve, Euler, observations.  One
// environment with the layout `lid` in the warp's `area`; returns 1 (nothing of the environment's state touched) if it does not fit
// the layout.  Compiled separately: the kernel calls it for both tiers.  SORTED (the cost order): `env` is the environment for the
// large tier; for the small tier it is the warp's position in the launch, resolved here (tail_env_at, recorded in tail_order) so that
// the kernel body keeps no loaded value live across the call; the cost class of the environment is written for the next substep.
template <typename R, bool SORTED, bool DYN>
DEVN int tail_env(R* area, int lane, int lid, Grp g, int env, int nsub, int phases, const R* action, unsigned long long* bar, unsigned& parity) {
  const int sub = g.sub;
  if (SORTED && lid == LAY_TS) {
    const int p = env;
    env = tail_env_at<R>(g, p, lane);
    if (lane == 0) cstate<R>(g.slot).tail_order[g.env0 + p] = env;
  }
  Eng<R> e(area, lane, g.slot, lid);
#ifdef B2S_INSTR
  const DState<R>& s = cstate<R>(g.slot);
  long long instr_t0 = clock64();
#endif
  const int pk = tail_rows(e, env, bar, parity);
  if (TAIL_OVF(pk)) return 1;
  const int ncon = TAIL_NCON(pk), nefc = TAIL_NEFC(pk);
  int warn = TAIL_WARN(pk);
  if ((phases & PH_CTRL) && !(phases & PH_CTRL_EXT)) tail_ctrl(e, env, sub, action);
  if constexpr (DYN) warn |= tail_accel(e, tail_act_force_out(e, env, sub == nsub - 1));
  else warn |= tail_accel(e);
  int niter;
  warn |= tail_newton(e, nefc, ncon, &niter);
  if (SORTED && lane == 0) e.state().tail_key[env] = tail_cost_key(niter, nefc, lid == LAY_TL);
  if constexpr (DYN) if (sub == nsub - 1) export_dynamics(e, env, ncon, nefc, niter);
  tail_finish(e, env, sub, nsub, phases, ncon, warn, bar, parity);
#ifdef B2S_INSTR
  if (lane == 0 && s.cyc) {
    float* c = s.cyc + ((size_t)env * 32 + (sub & 31)) * 8;
    c[1] = (float)(clock64() - instr_t0);
    c[2] = (float)niter; c[3] = (float)s.solve_ls[env]; c[4] = (float)nefc; c[5] = (float)ncon;
    c[6] = lid == LAY_TL ? 1.f : 0.f; c[7] = (float)blockIdx.x;
  }
  if (lane == 0 && s.stats) { atomicAdd(s.stats + 32 + min(ncon, 128), 1); atomicAdd(s.stats + 176 + min(nefc, 320), 1); if (lid == LAY_TL) atomicAdd(s.stats + 19, 1); }
#endif
  return 0;
}

// Warp per environment of the group with the small-capacity layout (`stride` words per warp), in the order of tail_env_at (SORTED)
// or by id; an environment that does not fit is left in the block's overflow list.  After a block barrier the first `nlw` warps re-run
// the block's overflowed environments with the full-capacity layout (`stride_l` words per warp, over the small tier's dead areas).
// An overflowed environment waits for its own block only, not for the whole group.
template <typename R, int THREADS, bool SORTED, bool DYN>
__global__ void __launch_bounds__(THREADS, THREADS == TAIL_WIDE_THREADS ? 1 : TAIL_BLOCKS) tail_kernel(int phases, int nsub, const R* action, Grp g, int stride, int stride_l, int nlw) {
  const DState<R>& s = cstate<R>(g.slot);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  R* smem = reinterpret_cast<R*>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  INSTR_BEGIN(s, g, 3)
  __shared__ unsigned long long mbar[32];  // one transaction barrier per warp (TMA loads of its workspace regions)
  __shared__ int ovf[32];                  // per warp: its position if its environment did not fit the small tier, else -1
  if (blockIdx.x == 0 && warp == 0) {  // phase1_kernel is done with the work-list counters; phase0_kernel(s + 1) files into the other set
    int* c = CLC(s, g);
    if (lane == 0) { c[0] = 0; c[1] = 0; c[3] = 0; }
    if (lane < TAIL_NKEY) CLK(s, g, g.sub + 1)[lane] = 0;
  }
  if (lane == 0) mbar_init(&mbar[warp]);
  __syncwarp();
  unsigned parity = 0;
  const int p = blockIdx.x * wpb + warp;
  int o = -1;
  if (p < g.nenv && tail_env<R, SORTED, DYN>(smem + (size_t)warp * stride, lane, LAY_TS, g, SORTED ? p : g.env0 + p, nsub, phases, action, &mbar[warp], parity)) o = p;
  if (lane == 0) ovf[warp] = o;
  // the small tier's areas are dead from here on (every fitting environment has stored its state, ws_store waited for its bulk
  // stores); order this thread's generic accesses to them before the large tier's bulk loads into the same shared memory
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (warp < nlw)
    for (int k = warp; k < wpb; k += nlw)
      if (ovf[k] >= 0)
        tail_env<R, SORTED, DYN>(smem + (size_t)warp * stride_l, lane, LAY_TL, g, SORTED ? s.tail_order[g.env0 + ovf[k]] : g.env0 + ovf[k], nsub, phases, action, &mbar[warp], parity);
  INSTR_END(s, g, 3)
}
