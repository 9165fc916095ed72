// libb2s: C ABI + host side of the batched engine (model upload, workspace layout, kernel launches).
// Entry points are declared in include/b2s.h; each cites the reference call it replaces.
#include "../../include/b2s.h"
#include "b2s_unit.cuh"
#include "b2s_snapshot.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CUDA_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(B2S_ERR_CUDA, std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

// ------------------------------------------------------------------------------------------------ blob reader
struct BlobRec { char name[48]; int32_t dtype, ndim, shape[4]; int64_t off, nbytes; };
struct Blob {
  const char* p; size_t n;
  const BlobRec* find(const char* name) const {
    int64_t cnt; memcpy(&cnt, p + 8, 8);
    const BlobRec* r = (const BlobRec*)(p + 16);
    for (int64_t i = 0; i < cnt; i++) if (!strcmp(r[i].name, name)) return r + i;
    return nullptr;
  }
  bool has(const char* name) const { return find(name) != nullptr; }
  // FNV-1a of every record (name, dtype, shape, data) except the capacity records: tier choices are bit-exact, so two handles that
  // differ only in capacities accept each other's snapshots
  uint64_t hash() const;
  const double* f64(const char* name, int64_t* count = nullptr) const {
    const BlobRec* r = find(name);
    if (!r || r->dtype != 0) throw std::string("model blob: missing f64 field ") + name;
    if (count) *count = r->nbytes / 8;
    return (const double*)(p + r->off);
  }
  const int* i32(const char* name, int64_t* count = nullptr) const {
    const BlobRec* r = find(name);
    if (!r || r->dtype != 1) throw std::string("model blob: missing i32 field ") + name;
    if (count) *count = r->nbytes / 4;
    return (const int*)(p + r->off);
  }
  int scalar_i(const char* name) const { return i32(name)[0]; }
  double scalar_f(const char* name) const { return f64(name)[0]; }
};
static const uint64_t FNV_BASIS = 1469598103934665603ull;
static uint64_t fnv1a(uint64_t h, const void* p, size_t n) {
  const unsigned char* c = (const unsigned char*)p;
  for (size_t i = 0; i < n; i++) { h ^= c[i]; h *= 1099511628211ull; }
  return h;
}
uint64_t Blob::hash() const {
  int64_t cnt; memcpy(&cnt, p + 8, 8);
  const BlobRec* r = (const BlobRec*)(p + 16);
  uint64_t h = FNV_BASIS;
  for (int64_t i = 0; i < cnt; i++) {
    const char* nm = r[i].name;
    if (!strcmp(nm, "opt_maxcon") || !strcmp(nm, "opt_maxefc") || !strcmp(nm, "opt_maxcon_small") || !strcmp(nm, "opt_maxefc_small")) continue;
    h = fnv1a(h, nm, strnlen(nm, sizeof(r[i].name)) + 1);
    h = fnv1a(h, &r[i].dtype, sizeof(int32_t) * 6);  // dtype, ndim, shape
    h = fnv1a(h, p + r[i].off, (size_t)r[i].nbytes);
  }
  return h;
}

// ------------------------------------------------------------------------------------------------ sim object
struct ArrayInfo { void* ptr; int dtype; int ndim; int64_t shape[4]; };
struct SnapSecHost { std::string name; int64_t off, count; int dtype; void* ptr; };  // off: bytes into the row; count: elements per env
#define SNAP_MAXSEC 128

struct b2s_sim {
  int n_env = 0, device = 0, precision = B2S_F32;
  int num_sms = 1;  // streaming multiprocessors of `device` (grid sizes of the claim-based launches)
  cudaStream_t stream = 0;
  std::vector<void*> allocs;
  std::map<std::string, ArrayInfo> arrays;
  WSLayout lay[B2S_NLAY]{};  // LAY_FULL (fused kernel), LAY_P0, LAY_TS / LAY_TL (tail tiers), LAY_ROW (global workspace row)
  int slot = -1;             // constant-memory descriptor slot (per device)
  int mc_small = 0, me_small = 0;  // capacities of the small tail tier (== maxcon / maxefc: no tiering)
  int osc_in_tail = 0;       // layouts built for the in-kernel OSC controller (B2S_CTRL_SPLIT=0)
  // phase 0: warps per block; tail: warps per block, words per warp of the small and of the large tier, warps per block that run
  // the large tier
  int wpb0 = 8, wpb5 = 8, stride5 = 0, stride5l = 0, nlw5 = 1, tail_wide = 0;
  size_t smem0 = 0, smem5 = 0;
  DModel<float> mf{};
  DModel<double> md{};
  DState<float> sf{};
  DState<double> sd{};
  CtrlCfgDev ctrl{};
  int has_ctrl = 0;
  int wpb_fused = 4;    // fused kernel: workspace + EPA polytope area per warp
  size_t smem_fused = 0;
  int64_t launches = 0;
  int nq = 0, nv = 0, nu = 0, nbody = 0, ngeom = 0, nsite = 0, maxcon = 0, maxefc = 0, ncg = 0, hc_stride = 0;
  std::vector<double> qpos0;
  std::vector<int> site_bodyid, cgid;
  std::map<std::string, std::vector<std::string>> names;  // object type -> names by id (MjModel name tables)
  int has_obs = 0, export_env_step = 1, dirty = 1, mode = 0, ngroups = 8;
  int ctrl_split = 1;  // pipeline: OSC controller as its own thread-per-environment kernel (B2S_CTRL_SPLIT=0: inside the tail kernel)
  // pipeline: one CUDA graph per environment group, replayed on the group's stream and joined to `stream` through gevents
  std::vector<cudaStream_t> gstreams;
  std::vector<cudaEvent_t> gevents;
  cudaEvent_t in_event = nullptr;
  void* action_buf = nullptr;
  std::map<long long, cudaGraphExec_t> graphs;
  PhaseIO pio[B2S_NPIO];
  std::map<std::string, Region> reg;
  // unit-queue mode (mode 2, b2s_unit.cuh)
  int* uq_ring = nullptr; int* uq_ovf = nullptr; int* uq_ctr = nullptr; int uq_cap = 0;
  int uq_wpb = 0, uq_stride = 0, uq_stride_large = 0, uq_wpb_large = 0, uq_nlarge = 0, uq_grid = 0;
  size_t uq_smem = 0;
#ifdef B2S_INSTR
  unsigned long long* uq_prof = nullptr;  // the unit queue's stage counters (UnitQ::prof)
#endif
  std::vector<double> xpos0_h, xquat0_h;  // world poses of the bodies welded to the world (model constants)
  std::vector<int> body_weldid_h;
  // model values that b2s_model_override copies per environment, and the host-computed constants derived from them
  std::vector<int> geom_type_h;
  std::vector<double> geom_size_h, geom_friction_h, geom_rbound_h, geom_aabb_h, body_mass_h, body_inertia_h, dof_iw_h, body_iw_h;
  std::vector<double> geom_solref_h, geom_solimp_h, dof_damping_h, dof_armature_h, dof_frictionloss_h;
  double meaninertia_h = 1;
  int sc_words = 0;  // set-constants pass: words of shared memory per warp (0 until its first launch)
  // b2s_perturb_config: entry and item tables on the device (perturb_kernel), items per environment (0 = not configured)
  PerturbEntry* pert_ent = nullptr;
  PerturbItem* pert_item = nullptr;
  int pert_nitems = 0;
  // snapshots (b2s_snapshot / b2s_restore): every entry point that allocates a per-environment array or changes what the signature
  // covers bumps layout_version; the section table is rebuilt when it differs from snap_version
  int layout_version = 0, snap_version = -1;
  std::vector<SnapSecHost> snap;
  size_t snap_row_bytes = 0;
  uint64_t snap_sig = 0, blob_hash = 0;  // blob_hash: the model blob without its capacity records
  SnapSec* snap_dev = nullptr;           // device copy of the section table (capacity SNAP_MAXSEC)
  std::vector<int> obs_tab_h, task_tab_h;  // host copies of the observation / task op tables (signature)
  // b2s_obs_modifiers: the device table (allocated at the first call), observables of the per-environment arrays (0: none yet),
  // whether a configuration is active, the model's timestep in fp64
  ObsModDev* obs_mod_dev = nullptr;
  int obs_arr_n = 0, obs_mod_on = 0;
  double timestep_h = 0;
};

// Every entry point picks the handle's precision once: f(DModel<R>&, DState<R>&) runs with R = float or double, and
// real_of<decltype(m)> names R inside a generic lambda.
template <typename F> static auto with_real(b2s_sim* s, F&& f) { return s->precision == B2S_F32 ? f(s->mf, s->sf) : f(s->md, s->sd); }
template <typename M> struct RealOf;
template <typename R> struct RealOf<DModel<R>> { using type = R; };
template <typename M> using real_of = typename RealOf<std::remove_cv_t<std::remove_reference_t<M>>>::type;
static size_t real_size(const b2s_sim* s) { return s->precision == B2S_F32 ? sizeof(float) : sizeof(double); }

static int launch_set_const(b2s_sim* s, const uint8_t* mask);  // the set-constants pass (no-op without model overrides)

template <typename T> static T* dev_upload(b2s_sim* s, const std::vector<T>& h) {
  T* d = nullptr;
  size_t n = h.size() ? h.size() : 1;
  if (cudaMalloc(&d, n * sizeof(T)) != cudaSuccess) throw std::string("cudaMalloc failed");
  s->allocs.push_back(d);
  if (h.size()) cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  // cudaMemcpy from pageable memory returns once the data is STAGED; the DMA runs on the legacy stream, which non-blocking streams
  // (the handle's group streams, every torch stream) do not wait for: finish it here
  cudaStreamSynchronize(cudaStreamLegacy);
  return d;
}
template <typename R> static const R* up_f(b2s_sim* s, const Blob& b, const char* name) {
  int64_t n; const double* p = b.f64(name, &n);
  std::vector<R> h(n);
  for (int64_t i = 0; i < n; i++) h[i] = (R)p[i];
  return dev_upload(s, h);
}
static const int* up_i(b2s_sim* s, const Blob& b, const char* name) {
  int64_t n; const int* p = b.i32(name, &n);
  std::vector<int> h(p, p + n);
  return dev_upload(s, h);
}
template <typename R> static const R* up_vec(b2s_sim* s, const std::vector<double>& v) {
  std::vector<R> h(v.size());
  for (size_t i = 0; i < v.size(); i++) h[i] = (R)v[i];
  return dev_upload(s, h);
}

static void h_quat2mat(double* M, const double* q) {
  double w = q[0], x = q[1], y = q[2], z = q[3];
  M[0] = w * w + x * x - y * y - z * z; M[1] = 2 * (x * y - w * z); M[2] = 2 * (x * z + w * y);
  M[3] = 2 * (x * y + w * z); M[4] = w * w - x * x + y * y - z * z; M[5] = 2 * (y * z - w * x);
  M[6] = 2 * (x * z - w * y); M[7] = 2 * (y * z + w * x); M[8] = w * w - x * x - y * y + z * z;
}
static void h_qmul(double* r, const double* a, const double* b) {
  double w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  double x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  double y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  double z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}

template <typename R> static void build_model(b2s_sim* s, const Blob& b, DModel<R>& m) {
  m.nq = b.scalar_i("nq"); m.nv = b.scalar_i("nv"); m.nu = b.scalar_i("nu"); m.nbody = b.scalar_i("nbody");
  m.njnt = b.scalar_i("njnt"); m.ngeom = b.scalar_i("ngeom"); m.nsite = b.scalar_i("nsite"); m.npair = b.scalar_i("npair");
  m.nmocap = b.scalar_i("nmocap");
  s->timestep_h = b.scalar_f("opt_timestep");
  m.timestep = (R)s->timestep_h; m.impratio = (R)b.scalar_f("opt_impratio");
  m.density = (R)b.scalar_f("opt_density"); m.viscosity = (R)b.scalar_f("opt_viscosity");
  m.tolerance = (R)b.scalar_f("opt_tolerance"); m.meaninertia = (R)b.scalar_f("stat_meaninertia");
  m.iterations = b.scalar_i("opt_iterations"); m.ls_iterations = b.scalar_i("opt_ls_iterations");
  const double* grav = b.f64("opt_gravity");
  for (int k = 0; k < 3; k++) m.gravity[k] = (R)grav[k];
  const double* wind = b.f64("opt_wind");
  for (int k = 0; k < 3; k++) m.wind[k] = (R)wind[k];
  if (b.scalar_i("opt_cone") != 1) throw std::string("only elliptic friction cones are implemented (reference models set cone=elliptic)");
  if (m.nv > 64) throw std::string("nv > 64 not supported");
  int nb = m.nbody, nv = m.nv, nj = m.njnt, ng = m.ngeom;
  const int* parent = b.i32("body_parentid");
  const int* jntnum = b.i32("body_jntnum");
  const int* jntadr = b.i32("body_jntadr");
  const int* dofnum = b.i32("body_dofnum");
  const int* dofadr = b.i32("body_dofadr");
  const int* weld = b.i32("body_weldid");
  const int* jtype = b.i32("jnt_type");
  const int* jdofadr = b.i32("jnt_dofadr");
  const int* dofjnt = b.i32("dof_jntid");
  const int* dofpar = b.i32("dof_parentid");
  const int* dofbody = b.i32("dof_bodyid");
  // one joint per body (free joints included); ball joints unsupported
  std::vector<int> body_jntid(nb, -1), depth(nb, 0), sub_end(nb, 0);
  for (int i = 0; i < nb; i++) {
    if (jntnum[i] > 1) throw std::string("bodies with more than one joint are not supported");
    if (jntnum[i] == 1) { body_jntid[i] = jntadr[i]; if (jtype[jntadr[i]] == JNT_BALL) throw std::string("ball joints are not supported"); }
  }
  int maxdepth = 0;
  for (int i = 1; i < nb; i++) {
    depth[i] = weld[i] == 0 ? 0 : depth[parent[i]] + 1;
    if (depth[i] > maxdepth) maxdepth = depth[i];
  }
  for (int i = nb - 1; i >= 0; i--) {
    if (sub_end[i] < i + 1) sub_end[i] = i + 1;
    if (i > 0 && sub_end[parent[i]] < sub_end[i]) sub_end[parent[i]] = sub_end[i];
  }
  m.maxdepth = maxdepth;
  // static world poses
  std::vector<double> xpos0(3 * nb, 0.0), xquat0(4 * nb, 0.0);
  const double* bpos = b.f64("body_pos");
  const double* bquat = b.f64("body_quat");
  xquat0[0] = 1;
  for (int i = 1; i < nb; i++) {
    if (weld[i] != 0) { xquat0[4 * i] = 1; continue; }
    double Mp[9];
    h_quat2mat(Mp, &xquat0[4 * parent[i]]);
    for (int r = 0; r < 3; r++)
      xpos0[3 * i + r] = xpos0[3 * parent[i] + r] + Mp[3 * r] * bpos[3 * i] + Mp[3 * r + 1] * bpos[3 * i + 1] + Mp[3 * r + 2] * bpos[3 * i + 2];
    h_qmul(&xquat0[4 * i], &xquat0[4 * parent[i]], bquat + 4 * i);
  }
  // dof tables
  std::vector<int> dkind(nv), cddstart(nv), fl_dof, lim_jnt;
  const double* floss = b.f64("dof_frictionloss");
  for (int i = 0; i < nv; i++) {
    int j = dofjnt[i], k = i - jdofadr[j];
    if (jtype[j] == JNT_FREE) {
      dkind[i] = k < 3 ? DK_FREE_T : DK_FREE_R;
      cddstart[i] = k < 3 ? -1 : jdofadr[j] + 2;  // rotational axes: velocity of the three translations only
    } else {
      dkind[i] = jtype[j] == JNT_SLIDE ? DK_SLIDE : DK_HINGE;
      cddstart[i] = dofpar[i];
    }
    if (floss[i] > 0) fl_dof.push_back(i);
  }
  const int* jlim = b.i32("jnt_limited");
  for (int j = 0; j < nj; j++)
    if (jlim[j] && (jtype[j] == JNT_SLIDE || jtype[j] == JNT_HINGE)) lim_jnt.push_back(j);
  std::vector<int> spr_jnt;
  const double* stiff = b.f64("jnt_stiffness");
  for (int j = 0; j < nj; j++) {
    if (stiff[j] == 0) continue;
    if (jtype[j] == JNT_FREE) throw std::string("stiffness on a free joint is not supported");
    spr_jnt.push_back(j);
  }
  m.nfl = (int)fl_dof.size(); m.nlim = (int)lim_jnt.size(); m.nspr = (int)spr_jnt.size();
  std::vector<unsigned long long> dofmask(nb, 0ull);
  for (int i = 1; i < nb; i++) {
    dofmask[i] = dofmask[parent[i]];
    for (int d = 0; d < dofnum[i]; d++) dofmask[i] |= 1ull << (dofadr[i] + d);
  }
  // kinematic trees: dofs of one tree are contiguous (DFS numbering); world-welded bodies have tree id -1
  const int* rootid = b.i32("body_rootid");
  std::vector<int> treebase(nv, 0), treesize(nv, 0), body_tree(nb, -1);
  {
    std::vector<int> root_first(nb, -1), root_last(nb, -1);
    for (int i = 0; i < nv; i++) {
      int r = rootid[dofbody[i]];
      if (root_first[r] < 0) root_first[r] = i;
      root_last[r] = i;
    }
    int mx = 0;
    for (int i = 0; i < nv; i++) {
      int r = rootid[dofbody[i]];
      treebase[i] = root_first[r];
      treesize[i] = root_last[r] - root_first[r] + 1;
      if (treesize[i] > mx) mx = treesize[i];
    }
    m.max_treesize = mx;
    for (int i = 1; i < nb; i++) body_tree[i] = weld[i] == 0 ? -1 : rootid[i];
  }
  m.dof_treebase = dev_upload(s, treebase); m.dof_treesize = dev_upload(s, treesize); m.body_treeid = dev_upload(s, body_tree);
  std::vector<int> ment_i, ment_j;
  for (int i = 0; i < nv; i++)
    for (int j = i; j >= 0; j = dofpar[j]) { ment_i.push_back(i); ment_j.push_back(j); }
  m.nment = (int)ment_i.size();
  // colliding geoms
  const int* pair = b.i32("pair_geom");
  std::vector<int> cgid(ng, -1), cg;
  for (int p = 0; p < m.npair; p++)
    for (int k = 0; k < 2; k++) { int g = pair[2 * p + k]; if (cgid[g] < 0) cgid[g] = 1; }
  for (int g = 0; g < ng; g++) if (cgid[g] > 0) { cgid[g] = (int)cg.size(); cg.push_back(g); }
  m.ncg = (int)cg.size();
  s->cgid = cgid;
  if (m.ncg > 64) throw std::string("more than 64 colliding geoms not supported");
  const int* condim = b.i32("geom_condim");
  int maxdim = 1;
  for (int g : cg) if (condim[g] > maxdim) maxdim = condim[g];
  m.hc_stride = maxdim * maxdim;
  m.maxcon = s->maxcon; m.maxefc = s->maxefc;

  m.body_parentid = up_i(s, b, "body_parentid"); m.body_jntid = dev_upload(s, body_jntid);
  m.body_dofnum = up_i(s, b, "body_dofnum"); m.body_dofadr = up_i(s, b, "body_dofadr"); m.body_weldid = up_i(s, b, "body_weldid");
  m.body_subtree_end = dev_upload(s, sub_end); m.body_depth = dev_upload(s, depth);
  m.body_pos = up_f<R>(s, b, "body_pos"); m.body_quat = up_f<R>(s, b, "body_quat"); m.body_ipos = up_f<R>(s, b, "body_ipos");
  m.body_iquat = up_f<R>(s, b, "body_iquat"); m.body_mass = up_f<R>(s, b, "body_mass"); m.body_inertia = up_f<R>(s, b, "body_inertia");
  m.body_invweight0 = up_f<R>(s, b, "body_invweight0");
  m.body_xpos0 = up_vec<R>(s, xpos0); m.body_xquat0 = up_vec<R>(s, xquat0);
  s->xpos0_h = xpos0; s->xquat0_h = xquat0;
  { const int* wd = b.i32("body_weldid"); s->body_weldid_h.assign(wd, wd + nb); }
  {
    auto host = [&](const char* name, std::vector<double>& v) { int64_t n = 0; const double* p = b.f64(name, &n); v.assign(p, p + n); };
    host("geom_size", s->geom_size_h); host("geom_friction", s->geom_friction_h); host("geom_rbound", s->geom_rbound_h);
    host("geom_aabb", s->geom_aabb_h); host("body_mass", s->body_mass_h); host("body_inertia", s->body_inertia_h);
    host("dof_invweight0", s->dof_iw_h); host("body_invweight0", s->body_iw_h);
    host("geom_solref", s->geom_solref_h); host("geom_solimp", s->geom_solimp_h); host("dof_damping", s->dof_damping_h);
    host("dof_armature", s->dof_armature_h); host("dof_frictionloss", s->dof_frictionloss_h);
    s->meaninertia_h = b.scalar_f("stat_meaninertia");
    const int* gt = b.i32("geom_type"); s->geom_type_h.assign(gt, gt + ng);
  }
  m.jnt_type = up_i(s, b, "jnt_type"); m.jnt_qposadr = up_i(s, b, "jnt_qposadr"); m.jnt_dofadr = up_i(s, b, "jnt_dofadr");
  m.jnt_bodyid = up_i(s, b, "jnt_bodyid"); m.jnt_limited = up_i(s, b, "jnt_limited");
  m.jnt_pos = up_f<R>(s, b, "jnt_pos"); m.jnt_axis = up_f<R>(s, b, "jnt_axis"); m.jnt_range = up_f<R>(s, b, "jnt_range");
  m.jnt_margin = up_f<R>(s, b, "jnt_margin");
  m.jnt_solref = up_f<R>(s, b, "jnt_solref"); m.jnt_solimp = up_f<R>(s, b, "jnt_solimp"); m.qpos0 = up_f<R>(s, b, "qpos0");
  m.dof_bodyid = up_i(s, b, "dof_bodyid"); m.dof_jntid = up_i(s, b, "dof_jntid"); m.dof_parentid = up_i(s, b, "dof_parentid");
  m.dof_kind = dev_upload(s, dkind); m.dof_cddstart = dev_upload(s, cddstart); m.fl_dof = dev_upload(s, fl_dof);
  m.lim_jnt = dev_upload(s, lim_jnt); m.body_dofmask = dev_upload(s, dofmask);
  m.spr_jnt = dev_upload(s, spr_jnt); m.jnt_stiffness = up_f<R>(s, b, "jnt_stiffness"); m.qpos_spring = up_f<R>(s, b, "qpos_spring");
  m.dof_armature = up_f<R>(s, b, "dof_armature"); m.dof_damping = up_f<R>(s, b, "dof_damping");
  m.dof_frictionloss = up_f<R>(s, b, "dof_frictionloss"); m.dof_solref = up_f<R>(s, b, "dof_solref");
  m.dof_solimp = up_f<R>(s, b, "dof_solimp"); m.dof_invweight0 = up_f<R>(s, b, "dof_invweight0");
  m.ment_i = dev_upload(s, ment_i); m.ment_j = dev_upload(s, ment_j);
  m.geom_type = up_i(s, b, "geom_type"); m.geom_bodyid = up_i(s, b, "geom_bodyid"); m.geom_condim = up_i(s, b, "geom_condim");
  m.geom_dataid = up_i(s, b, "geom_dataid"); m.geom_priority = up_i(s, b, "geom_priority");
  m.geom_cgid = dev_upload(s, cgid); m.cg_geom = dev_upload(s, cg);
  m.geom_size = up_f<R>(s, b, "geom_size"); m.geom_pos = up_f<R>(s, b, "geom_pos"); m.geom_quat = up_f<R>(s, b, "geom_quat");
  m.geom_friction = up_f<R>(s, b, "geom_friction"); m.geom_solmix = up_f<R>(s, b, "geom_solmix");
  m.geom_solref = up_f<R>(s, b, "geom_solref"); m.geom_solimp = up_f<R>(s, b, "geom_solimp");
  m.geom_rbound = up_f<R>(s, b, "geom_rbound"); m.geom_aabb = up_f<R>(s, b, "geom_aabb");
  m.pair_geom = up_i(s, b, "pair_geom");
  m.mesh_vertadr = up_i(s, b, "mesh_vertadr"); m.mesh_vertnum = up_i(s, b, "mesh_vertnum"); m.mesh_vert = up_f<R>(s, b, "mesh_vert");
  {  // staging area of the convex narrow-phase kernel: room for the two largest hulls (at most 56 KB), see convex_convex
    int64_t nm = 0; const int* vn = b.i32("mesh_vertnum", &nm);
    int n1 = 0, n2 = 0;
    for (int64_t i = 0; i < nm; i++) { int v = vn[i]; if (v > n1) { n2 = n1; n1 = v; } else if (v > n2) n2 = v; }
    int need = 24 + ((3 * n1 + 3) & ~3) + ((3 * n2 + 3) & ~3);  // two poses, two hulls
    int cap = (int)(56 * 1024 / sizeof(R));
    m.stage_cap = std::min(need, cap);
  }
  m.site_bodyid = up_i(s, b, "site_bodyid"); m.site_pos = up_f<R>(s, b, "site_pos"); m.site_quat = up_f<R>(s, b, "site_quat");
  m.act_trnid = up_i(s, b, "actuator_trnid"); m.act_ctrllimited = up_i(s, b, "actuator_ctrllimited");
  m.act_forcelimited = up_i(s, b, "actuator_forcelimited"); m.act_biastype = up_i(s, b, "actuator_biastype");
  m.act_ctrlrange = up_f<R>(s, b, "actuator_ctrlrange"); m.act_forcerange = up_f<R>(s, b, "actuator_forcerange");
  {
    int64_t n; const double* g6 = b.f64("actuator_gear", &n);
    std::vector<double> g1(m.nu);
    for (int i = 0; i < m.nu; i++) g1[i] = g6[6 * i];
    m.act_gear = up_vec<R>(s, g1);
  }
  m.act_gainprm = up_f<R>(s, b, "actuator_gainprm"); m.act_biasprm = up_f<R>(s, b, "actuator_biasprm");
}

template <typename T> static T* dev_zeros(b2s_sim* s, size_t n) {
  T* d = nullptr;
  if (n == 0) n = 1;
  if (cudaMalloc(&d, n * sizeof(T)) != cudaSuccess) throw std::string("cudaMalloc failed");
  // cudaMemset is asynchronous and runs on the legacy stream; the handle's kernels run on non-blocking streams that do not wait for
  // it (a zero-fill of the action buffer that landed in the middle of the first control step made two concurrent handles diverge)
  cudaMemset(d, 0, n * sizeof(T));
  cudaStreamSynchronize(cudaStreamLegacy);
  s->allocs.push_back(d);
  return d;
}
// per precision: the dtype code of its arrays and its constant-memory descriptor banks
template <typename R> struct DT;
template <> struct DT<float> {
  static const int code = B2S_F32;
  static const void* model_bank() { return &c_model_f; }
  static const void* state_bank() { return &c_state_f; }
};
template <> struct DT<double> {
  static const int code = B2S_F64;
  static const void* model_bank() { return &c_model_d; }
  static const void* state_bank() { return &c_state_d; }
};

template <typename R>
static R* state_arr(b2s_sim* s, const char* name, int64_t d1, int64_t d2 = 0, int64_t d3 = 0) {
  size_t per = (size_t)(d1 ? d1 : 1) * (d2 ? d2 : 1) * (d3 ? d3 : 1);
  R* p = dev_zeros<R>(s, (size_t)s->n_env * per);
  ArrayInfo a{p, DT<R>::code, 1 + (d1 > 0) + (d2 > 0) + (d3 > 0), {s->n_env, d1, d2, d3}};
  if (d1 == 0) a.ndim = 1;
  s->arrays[name] = a;
  return p;
}
static int* state_arr_i(b2s_sim* s, const char* name, int64_t d1, int64_t d2 = 0) {
  size_t per = (size_t)(d1 ? d1 : 1) * (d2 ? d2 : 1);
  int* p = dev_zeros<int>(s, (size_t)s->n_env * per);
  ArrayInfo a{p, B2S_I32, 1 + (d1 > 0) + (d2 > 0), {s->n_env, d1, d2, 0}};
  s->arrays[name] = a;
  return p;
}

template <typename R> static void build_state(b2s_sim* s, const DModel<R>& m, DState<R>& st) {
  st.n_env = s->n_env;
  int nq = m.nq, nv = m.nv, nu = m.nu, nb = m.nbody, ng = m.ngeom, ns = m.nsite, mc = m.maxcon, me = m.maxefc;
  st.qpos = state_arr<R>(s, "qpos", nq); st.qvel = state_arr<R>(s, "qvel", nv); st.qacc = state_arr<R>(s, "qacc", nv);
  st.qacc_ws = state_arr<R>(s, "qacc_warmstart", nv); st.ctrl = state_arr<R>(s, "ctrl", nu); st.time = state_arr<R>(s, "time", 0);
  st.xpos = state_arr<R>(s, "xpos", nb, 3); st.xquat = state_arr<R>(s, "xquat", nb, 4); st.xmat = state_arr<R>(s, "xmat", nb, 9);
  st.site_xpos = state_arr<R>(s, "site_xpos", ns, 3); st.site_xmat = state_arr<R>(s, "site_xmat", ns, 9);
  st.geom_xpos = state_arr<R>(s, "geom_xpos", ng, 3); st.geom_xmat = state_arr<R>(s, "geom_xmat", ng, 9);
  st.qM = state_arr<R>(s, "qM", nv, nv); st.qfrc_bias = state_arr<R>(s, "qfrc_bias", nv);
  st.qfrc_passive = state_arr<R>(s, "qfrc_passive", nv); st.qfrc_actuator = state_arr<R>(s, "qfrc_actuator", nv);
  st.qfrc_constraint = state_arr<R>(s, "qfrc_constraint", nv); st.qfrc_smooth = state_arr<R>(s, "qfrc_smooth", nv);
  st.qacc_smooth = state_arr<R>(s, "qacc_smooth", nv); st.actuator_force = state_arr<R>(s, "actuator_force", nu);
  st.cdof = state_arr<R>(s, "cdof", nv, 6);
  st.ncon = state_arr_i(s, "ncon", 0); st.contact_geom = state_arr_i(s, "contact_geom", mc, 2);
  st.contact_dim = state_arr_i(s, "contact_dim", mc); st.nefc = state_arr_i(s, "nefc", 0);
  st.efc_type = state_arr_i(s, "efc_type", me); st.warn = state_arr_i(s, "warn", 0); st.solver_niter = state_arr_i(s, "solver_niter", 0);
  st.contact_dist = state_arr<R>(s, "contact_dist", mc); st.contact_pos = state_arr<R>(s, "contact_pos", mc, 3);
  st.contact_frame = state_arr<R>(s, "contact_frame", mc, 9); st.contact_friction = state_arr<R>(s, "contact_friction", mc, 3);
  st.contact_solref = nullptr; st.contact_solimp = nullptr;
  st.efc_J = state_arr<R>(s, "efc_J", me, nv); st.efc_force = state_arr<R>(s, "efc_force", me);
  st.efc_aref = state_arr<R>(s, "efc_aref", me); st.efc_D = state_arr<R>(s, "efc_D", me); st.efc_R = state_arr<R>(s, "efc_R", me);
  st.goal_pos = state_arr<R>(s, "ctrl_goal_pos", 3); st.goal_ori = state_arr<R>(s, "ctrl_goal_ori", 9);
  st.init_qpos_arm = state_arr<R>(s, "ctrl_initial_joint", 8); st.grip_state = state_arr<R>(s, "ctrl_grip_state", 4);
  st.ctrl_torque = state_arr<R>(s, "ctrl_torque", 8);
  st.jv_state = state_arr<R>(s, "ctrl_jv_state", 72);
  st.wsg = nullptr;
}

// ---- workspace layouts.  Every region is 16-byte aligned in offset and length (TMA bulk copies).
struct LayB {
  int o = 0;
  int take(int n) { int r = o; o += (n + 3) & ~3; return r; }
};
struct Dims { int nq, nv, nu, nb, ncg, ns, hc; };

// the one-size-fits-all layout of the fused kernel (every phase's regions at once)
static void layout_full(const Dims& d, int mc, int me, WSLayout& L) {
  LayB B;
  int nq = d.nq, nv = d.nv, nu = d.nu, nb = d.nb, ncg = d.ncg, ns = d.ns;
  L = WSLayout{};
  L.mc = mc; L.me = me;
  L.qpos = B.take(nq); L.qvel = B.take(nv); L.qacc = B.take(nv); L.qacc_ws = B.take(nv); L.ctrl = B.take(nu);
  L.xpos = B.take(3 * nb); L.xquat = B.take(4 * nb); L.xmat = B.take(9 * nb);
  L.cdof = B.take(6 * nv); L.cvel = B.take(6 * nb);
  L.M = B.take(nv * nv); L.H = B.take(nv * nv);
  L.bias = B.take(nv); L.passive = B.take(nv); L.qact = B.take(nv); L.qsmooth = B.take(nv); L.qaccs = B.take(nv); L.qcon = B.take(nv);
  L.spos = B.take(3 * ns); L.smat = B.take(9 * ns);
  L.c_pos = B.take(3 * mc); L.c_frame = B.take(3 * mc); L.c_dist = B.take(mc); L.c_fric = B.take(3 * mc); L.c_int = B.take(5 * mc);
  L.e_D = B.take(me); L.e_R = B.take(me); L.e_aref = B.take(me); L.e_jar = B.take(me); L.e_jv = B.take(me);
  L.e_force = B.take(me); L.e_floss = B.take(me); L.e_int = B.take(me);
  L.Ma = B.take(nv); L.grad = B.take(nv); L.search = B.take(nv); L.Mv = B.take(nv);
  // union: kinematics intermediates that are dead once collision is done  |  the constraint Jacobian
  int ubase = B.o;
  L.xipos = B.take(3 * nb); L.cdofdot = B.take(6 * nv); L.cinert = B.take(10 * nb); L.frne = B.take(6 * nb); L.ffl = B.take(6 * nb);
  L.gpos = B.take(3 * ncg); L.gmat = B.take(9 * ncg);
  L.J = ubase;
  if (ubase + me * nv > B.o) B.o = ubase + ((me * nv + 3) & ~3);
  int sc = std::max(std::max(10 * nb, 200), std::max(me + d.hc * mc + 64, 9 * mc));
  if (sc < 672) sc = 672;  // controller work area (336 doubles)
  L.scratch_size = sc; L.scratch = B.take(sc);
  L.hdr = B.take(8);
  L.total = B.o;
  L.fused_stride = L.total + EPA_AREA_WORDS(EPA_MAXV, EPA_MAXF);
}

// phase 0: kinematics, velocity stage, CRB, broad phase.  The regions it hands to the other kernels come first, in row order.
static void layout_p0(const Dims& d, WSLayout& L) {
  LayB B;
  int nq = d.nq, nv = d.nv, nb = d.nb, ncg = d.ncg, ns = d.ns;
  L = WSLayout{};
  L.qpos = B.take(nq); L.qvel = B.take(nv);
  L.xpos = B.take(3 * nb); L.xquat = B.take(4 * nb); L.cdof = B.take(6 * nv); L.cvel = B.take(6 * nb);
  bool m_own = 12 * nb < nv * nv;  // otherwise M (written by crb) lives over frne + ffl (dead after velocity)
  if (m_own) L.M = B.take(nv * nv);
  L.bias = B.take(nv); L.passive = B.take(nv); L.spos = B.take(3 * ns); L.smat = B.take(9 * ns);
  L.gpos = B.take(3 * ncg); L.gmat = B.take(9 * ncg);
  L.xmat = B.take(9 * nb); L.xipos = B.take(3 * nb); L.cdofdot = B.take(6 * nv); L.cinert = B.take(10 * nb);
  L.frne = B.take(6 * nb); L.ffl = B.take(6 * nb);
  if (!m_own) L.M = L.frne;
  int sc = std::max(10 * nb, 200);  // kinematics locals (8 nb), composite inertias (10 nb), candidate lists (96 + 32 + ...)
  L.scratch_size = sc; L.scratch = B.take(sc);
  L.hdr = B.take(8);
  L.total = B.o;
}

// tail kernel with capacities (mc, me).  osc_in_tail: the OSC controller runs inside (needs body velocities and site poses from
// the start); otherwise the poses the observation / task tables read arrive late, over the dead constraint Jacobian.
static void layout_tail(const Dims& d, int mc, int me, bool osc_in_tail, WSLayout& L) {
  LayB B;
  int nq = d.nq, nv = d.nv, nu = d.nu, nb = d.nb, ns = d.ns;
  L = WSLayout{};
  L.mc = mc; L.me = me;
  L.qpos = B.take(nq); L.qvel = B.take(nv); L.qacc = B.take(nv); L.qacc_ws = B.take(nv); L.ctrl = B.take(nu);
  L.cdof = B.take(6 * nv);
  L.M = B.take(nv * nv); L.H = B.take(nv * nv);
  L.bias = B.take(nv); L.passive = B.take(nv); L.qact = B.take(nv); L.qsmooth = B.take(nv); L.qaccs = B.take(nv); L.qcon = B.take(nv);
  L.c_pos = B.take(3 * mc); L.c_frame = B.take(3 * mc); L.c_dist = B.take(mc); L.c_fric = B.take(3 * mc); L.c_int = B.take(5 * mc);
  L.e_D = B.take(me); L.e_R = B.take(me); L.e_aref = B.take(me); L.e_jar = B.take(me); L.e_jv = B.take(me);
  L.e_force = B.take(me); L.e_floss = B.take(me); L.e_int = B.take(me);
  L.Ma = B.take(nv); L.grad = B.take(nv); L.search = B.take(nv); L.Mv = B.take(nv);
  L.J = B.o;
  int jwords = (me * nv + 3) & ~3;
  if (osc_in_tail) {
    B.o += jwords;
    L.xpos = B.take(3 * nb); L.xquat = B.take(4 * nb); L.spos = B.take(3 * ns); L.smat = B.take(9 * ns); L.cvel = B.take(6 * nb);
  } else {
    LayB O; O.o = B.o;  // overlay on J: loaded after the solve, before the observation sample
    L.xpos = O.take(3 * nb); L.xquat = O.take(4 * nb); L.spos = O.take(3 * ns); L.smat = O.take(9 * ns);
    B.o = std::max(B.o + jwords, O.o);
  }
  int sc = std::max(me + d.hc * mc + 64, 9 * mc);
  if (osc_in_tail && sc < 672) sc = 672;  // in-kernel OSC work area (336 doubles)
  L.scratch_size = sc; L.scratch = B.take(sc);
  L.hdr = B.take(8);
  L.total = B.o;
}

// global workspace row: what phase 0 hands to the narrow phase, the controller kernel and the tail
static void layout_row(const Dims& d, WSLayout& L) {
  LayB B;
  int nv = d.nv, nb = d.nb, ncg = d.ncg, ns = d.ns;
  L = WSLayout{};
  L.xpos = B.take(3 * nb); L.xquat = B.take(4 * nb); L.cdof = B.take(6 * nv); L.cvel = B.take(6 * nb);
  L.M = B.take(nv * nv); L.bias = B.take(nv); L.passive = B.take(nv); L.spos = B.take(3 * ns); L.smat = B.take(9 * ns);
  L.gpos = B.take(3 * ncg); L.gmat = B.take(9 * ncg);
  L.hdr = B.take(8);
  L.total = B.o;
}

// load / store list of one phase: (shared-memory offset, row offset, words) per named region, adjacent regions merged into spans
static void make_io(const Dims& d, const WSLayout& S, const WSLayout& ROW, std::initializer_list<const char*> names, Region* out, int& n, int* words) {
  int nv = d.nv, nb = d.nb, ncg = d.ncg, ns = d.ns;
  auto a4 = [](int x) { return (x + 3) & ~3; };
  std::vector<Region> v;
  for (const char* nm : names) {
    std::string k = nm;
    Region r{0, 0, 0, 0};
#define REG(name, field, len_) if (k == name) { r.off = S.field; r.goff = ROW.field; r.len = a4(len_); }
    REG("xpos", xpos, 3 * nb) REG("xquat", xquat, 4 * nb) REG("cdof", cdof, 6 * nv) REG("cvel", cvel, 6 * nb) REG("M", M, nv * nv)
    REG("bias", bias, nv) REG("passive", passive, nv) REG("spos", spos, 3 * ns) REG("smat", smat, 9 * ns)
    REG("gpos", gpos, 3 * ncg) REG("gmat", gmat, 9 * ncg)
#undef REG
    if (r.len > 0) v.push_back(r);
  }
  std::sort(v.begin(), v.end(), [](const Region& a, const Region& b) { return a.goff < b.goff; });
  n = 0;
  if (words) *words = 0;
  for (const Region& r : v) {
    if (n > 0 && out[n - 1].off + out[n - 1].len == r.off && out[n - 1].goff + out[n - 1].len == r.goff) out[n - 1].len += r.len;
    else { if (n >= B2S_MAXREG) throw std::string("too many workspace spans"); out[n++] = r; }
  }
  if (words) for (int k = 0; k < n; k++) *words += out[k].len;
}

static void build_layouts(b2s_sim* s, int ncg, int hc_stride) {
  Dims d{s->nq, s->nv, s->nu, s->nbody, ncg, s->nsite, hc_stride};
  layout_full(d, s->maxcon, s->maxefc, s->lay[LAY_FULL]);
  layout_p0(d, s->lay[LAY_P0]);
  layout_tail(d, s->mc_small, s->me_small, s->osc_in_tail != 0, s->lay[LAY_TS]);
  layout_tail(d, s->maxcon, s->maxefc, s->osc_in_tail != 0, s->lay[LAY_TL]);
  layout_row(d, s->lay[LAY_ROW]);
  for (int k = 0; k < B2S_NPIO; k++) s->pio[k] = PhaseIO{};
  const WSLayout& ROW = s->lay[LAY_ROW];
  make_io(d, s->lay[LAY_P0], ROW, {"xpos", "xquat", "cdof", "cvel", "M", "bias", "passive", "spos", "smat", "gpos", "gmat"},
          s->pio[PIO_P0].store, s->pio[PIO_P0].nstore, nullptr);
  for (int t = 0; t < 2; t++) {
    const WSLayout& T = s->lay[t ? LAY_TL : LAY_TS];
    PhaseIO& early = s->pio[t ? PIO_TL : PIO_TS];
    PhaseIO& late = s->pio[t ? PIO_TL_LATE : PIO_TS_LATE];
    if (s->osc_in_tail) make_io(d, T, ROW, {"cdof", "cvel", "M", "bias", "passive", "xpos", "xquat", "spos", "smat"}, early.load, early.nload, &early.load_words);
    else {
      make_io(d, T, ROW, {"cdof", "M", "bias", "passive"}, early.load, early.nload, &early.load_words);
      make_io(d, T, ROW, {"xpos", "xquat", "spos", "smat"}, late.load, late.nload, &late.load_words);
    }
  }
}

// opt a kernel in to the device's maximum dynamic shared memory (the limit is the opt-in maximum MINUS the kernel's static shared
// memory: asking for the full 227 KB on a kernel with a static mbarrier array is an invalid argument)
template <typename F> static cudaError_t optin_max_smem(F fn, int device, int* limit_out = nullptr) {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, fn);
  if (e != cudaSuccess) return e;
  int optin = 0;
  e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  if (e != cudaSuccess) return e;
  int lim = optin - (int)a.sharedSizeBytes;
  if (limit_out) *limit_out = lim;
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, lim);
}

// block shapes: warps per block bounded by the kernels' launch bounds and by 227 KB of shared memory per block
static int fit_wpb(size_t per_warp, int cap) {
  int w = cap;
  while (w > 1 && per_warp * w > 226 * 1024) w--;
  return w;
}
static int choose_blocks(b2s_sim* s) {
  size_t rsz = real_size(s);
  // the tail's per-warp areas start on 16-byte boundaries
  auto a4 = [](int x) { return (x + 3) & ~3; };
  s->stride5 = a4(s->lay[LAY_TS].total);
  s->stride5l = a4(s->lay[LAY_TL].total);
  size_t pw0 = s->lay[LAY_P0].total * rsz, pws = s->stride5 * rsz, pwl = s->stride5l * rsz, pwf = s->lay[LAY_FULL].fused_stride * rsz;
  if (std::max(std::max(pw0, pws), std::max(pwl, pwf)) > 226 * 1024) return fail(B2S_ERR_UNSUPPORTED, "model workspace exceeds shared memory");
  // warps per block: as many as the launch bounds allow while the launch bounds' blocks per SM still fit one SM's shared memory
  auto pick = [&](size_t pw, int lb_threads, int lb_blocks) {
    int cap = lb_threads / 32, w = cap;
    while (w > 1 && (pw * w + 1024) * lb_blocks > 228 * 1024) w--;  // 1 KB per block is reserved by the system
    if ((pw * w + 1024) * lb_blocks > 228 * 1024) w = fit_wpb(pw, cap);  // cannot reach the block count: largest block that fits
    return w;
  };
  s->wpb0 = pick(pw0, P0_THREADS, P0_BLOCKS);
  // tail block shape: one 16-warp block per SM when 16 small-tier areas take at most 160 KB, else two blocks per SM.  Measured on an
  // H100 80GB HBM3 (700 W), env-steps/s two blocks -> one: Lift / Panda f32 (16 areas 146 KB) 310 k -> 325 k; Stack / Sawyer JV f32
  // (202 KB) 385 k -> 369 k; NutAssemblyRound (52 KB per area: 4 warps in one block) 55.2 k -> 49.9 k
  s->wpb5 = pick(pws, TAIL_THREADS, TAIL_BLOCKS);
  const int wide_w = TAIL_WIDE_THREADS / 32;
  s->tail_wide = pws * wide_w <= 160 * 1024;
  if (s->tail_wide) s->wpb5 = wide_w;
  // the tail's cost order (tail_kernel<.., SORTED = true>) for blocks of 8 warps or more: the slack it recovers (a block waits for the
  // slowest of its warps) grows with the warps per block.  Measured on an H100 80GB HBM3 (700 W), env-steps/s by id -> sorted: Lift /
  // Panda f32 (16 warps) 323 k -> 335 k, Stack / Sawyer JV f32 (8 warps, two blocks per SM) 383 k -> 397 k; NutAssemblyRound (52 KB
  // areas, 2 warps per block) 55.2 k -> 54.0 k.  Smaller blocks run the id-order instantiation, which has none of the order's code.
  const int sorted = s->wpb5 >= 8 ? 1 : 0;
  with_real(s, [&](auto&, auto& st) { st.tail_sorted = sorted; return 0; });
  // the large tier reuses the block's small-tier areas: as many full-capacity areas as they hold, at least one
  s->smem5 = std::max(pws * s->wpb5, pwl);
  s->nlw5 = std::max(1, std::min(s->wpb5, (int)(s->smem5 / pwl)));
  s->smem0 = pw0 * s->wpb0;
  int wf = fit_wpb(pwf, 16);
  s->wpb_fused = wf; s->smem_fused = pwf * wf;
  if (getenv("B2S_VERBOSE"))
    fprintf(stderr, "[b2s] slot %d words/warp: fused %d, P0 %d (%d warps/block), tail small %d [mc %d me %d] (%d warps/block, wide %d), tail large %d [mc %d me %d] (%d), row %d\n",
            s->slot, s->lay[LAY_FULL].fused_stride, s->lay[LAY_P0].total, s->wpb0, s->lay[LAY_TS].total, s->mc_small, s->me_small, s->wpb5, s->tail_wide,
            s->lay[LAY_TL].total, s->maxcon, s->maxefc, s->nlw5, s->lay[LAY_ROW].total);
  return B2S_OK;
}

static b2s_sim* g_slots[64][B2S_NSLOT] = {{nullptr}};  // live handles per device: descriptor slot owners

// The phase / narrow-phase kernels need different amounts of per-thread local memory (stack).  By default the driver shrinks the
// local-memory pool after a launch and grows it again for the next kernel that needs more - a device-wide reallocation worth
// ~200 us in front of every narrow_convex launch.  Ask the context to keep the pool at its high-water mark
// (cudaDeviceLmemResizeToMax / CU_CTX_LMEM_RESIZE_TO_MAX); works on the already-initialised primary context torch created.
static void keep_local_memory_pool() {
  unsigned flags = 0;
  if (cudaGetDeviceFlags(&flags) == cudaSuccess && (flags & cudaDeviceLmemResizeToMax)) return;
  const char* how = "unchanged";
  if (cudaSetDeviceFlags((flags & cudaDeviceMask) | cudaDeviceLmemResizeToMax) == cudaSuccess) how = "cudaSetDeviceFlags";
  else {
    cudaGetLastError();
    typedef int (*get_fn)(unsigned*);
    typedef int (*set_fn)(unsigned);
    void *fg = nullptr, *fs = nullptr;
    cudaDriverEntryPointQueryResult q1, q2;
    if (cudaGetDriverEntryPoint("cuCtxGetFlags", &fg, cudaEnableDefault, &q1) == cudaSuccess &&
        cudaGetDriverEntryPoint("cuCtxSetFlags", &fs, cudaEnableDefault, &q2) == cudaSuccess && fg && fs) {
      unsigned cf = 0;
      if (((get_fn)fg)(&cf) == 0 && ((set_fn)fs)(cf | 0x10u /* CU_CTX_LMEM_RESIZE_TO_MAX */) == 0) how = "cuCtxSetFlags";
    }
    cudaGetLastError();
  }
  if (getenv("B2S_VERBOSE")) fprintf(stderr, "[b2s] local-memory pool kept at high-water mark: %s\n", how);
}


// ------------------------------------------------------------------------------------------------ API
extern "C" {

const char* b2s_last_error(void) { return g_err.c_str(); }

int b2s_create(const void* blob_host, size_t nbytes, int n_env, int device, int precision, b2s_sim** out) {
  if (!blob_host || !out || n_env <= 0) return fail(B2S_ERR_ARG, "b2s_create: bad argument");
  if (nbytes < 16 || memcmp(blob_host, "B2SMODEL", 8) != 0) return fail(B2S_ERR_MODEL, "b2s_create: not a model blob");
  if (precision != B2S_F32 && precision != B2S_F64) return fail(B2S_ERR_ARG, "b2s_create: precision must be B2S_F32 or B2S_F64");
  // work-list entries pack (env << 12 | pair) into an int, unit-queue tickets env + n_env * substep
  if (n_env >= (1 << 19)) return fail(B2S_ERR_UNSUPPORTED, "b2s_create: n_env must be below 524288 per handle (create several handles)");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(B2S_ERR_CUDA, "b2s_create: no CUDA device available (this library has no CPU fallback)");
  CUDA_TRY(cudaSetDevice(device));
  keep_local_memory_pool();
  b2s_sim* s = new b2s_sim();
  s->n_env = n_env; s->device = device; s->precision = precision;
  if (cudaDeviceGetAttribute(&s->num_sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) {
    b2s_destroy(s);
    return fail(B2S_ERR_CUDA, "b2s_create: cannot query the multiprocessor count");
  }
  Blob b{(const char*)blob_host, nbytes};
  try {
    s->nq = b.scalar_i("nq"); s->nv = b.scalar_i("nv"); s->nu = b.scalar_i("nu"); s->nbody = b.scalar_i("nbody");
    s->ngeom = b.scalar_i("ngeom"); s->nsite = b.scalar_i("nsite");
    s->blob_hash = b.hash();
    s->maxcon = b.has("opt_maxcon") ? b.scalar_i("opt_maxcon") : 32;
    s->maxefc = b.has("opt_maxefc") ? b.scalar_i("opt_maxefc") : 64;
    if (s->maxcon > 128) throw std::string("opt_maxcon > 128 not supported");
    const double* q0 = b.f64("qpos0");
    s->qpos0.assign(q0, q0 + s->nq);
    const int* sb = b.i32("site_bodyid");
    s->site_bodyid.assign(sb, sb + s->nsite);
    for (const char* ty : {"body", "joint", "geom", "site", "actuator", "mesh", "camera", "light"}) {
      std::string key = std::string("names_") + ty;
      if (!b.has(key.c_str())) continue;
      int64_t nc = 0; const int* cp = b.i32(key.c_str(), &nc);
      std::vector<std::string>& v = s->names[ty];
      std::string cur;
      for (int64_t i = 0; i < nc; i++) { if (cp[i] == '\n') { v.push_back(cur); cur.clear(); } else cur.push_back((char)cp[i]); }
      if (nc > 0) v.push_back(cur);
    }
    int nfl = 0;
    with_real(s, [&](auto& m, auto& st) {
      build_model(s, b, m);
      build_state(s, m, st);
      s->ncg = m.ncg; s->hc_stride = m.hc_stride; nfl = m.nfl;
    });
    // small tail tier: capacities almost every environment of this task stays within (compiled into the model blob by the task
    // class); environments that need more are re-run by the large tier
    s->mc_small = b.has("opt_maxcon_small") ? b.scalar_i("opt_maxcon_small") : s->maxcon;
    s->me_small = b.has("opt_maxefc_small") ? b.scalar_i("opt_maxefc_small") : s->maxefc;
    s->mc_small = std::min(std::max(s->mc_small, 4), s->maxcon);
    s->me_small = std::min(std::max(s->me_small, nfl + 8), s->maxefc);  // friction-loss rows are always present
    if (s->maxefc < nfl + 8) throw std::string("opt_maxefc too small for the model's friction-loss rows");
    // descriptor slot
    for (int k = 0; k < B2S_NSLOT && s->slot < 0; k++)
      if (!g_slots[device & 63][k]) { g_slots[device & 63][k] = s; s->slot = k; }
    if (s->slot < 0) throw std::string("more than 8 live handles on one device");
    build_layouts(s, s->ncg, s->hc_stride);
  } catch (const std::string& e) {
    b2s_destroy(s);
    return fail(B2S_ERR_MODEL, "b2s_create: " + e);
  }
  if (choose_blocks(s) != B2S_OK) { b2s_destroy(s); return B2S_ERR_UNSUPPORTED; }
  {
    // the attribute belongs to the FUNCTION, not to the handle: always opt in to the device maximum (a later handle with a
    // smaller workspace must not lower the limit of an earlier one - that broke mixed-task batches in round 1)
    cudaError_t e1 = with_real(s, [&](auto& m, auto&) {
      using R = real_of<decltype(m)>;
      cudaError_t e = optin_max_smem(step_kernel<R>, device);
      if (e == cudaSuccess) e = optin_max_smem(phase0_kernel<R>, device);
      if (e == cudaSuccess) e = optin_max_smem(tail_kernel<R, TAIL_THREADS, false>, device);
      if (e == cudaSuccess) e = optin_max_smem(tail_kernel<R, TAIL_THREADS, true>, device);
      if (e == cudaSuccess) e = optin_max_smem(tail_kernel<R, TAIL_WIDE_THREADS, true>, device);
      if (e == cudaSuccess) e = optin_max_smem(phase1_kernel<R>, device);
      return e;
    });
    if (e1 != cudaSuccess) { std::string msg = cudaGetErrorString(e1); b2s_destroy(s); return fail(B2S_ERR_CUDA, "cudaFuncSetAttribute: " + msg); }
  }
  *out = s;
  int rc = b2s_reset(s, nullptr);
  if (rc != 0) { b2s_destroy(s); *out = nullptr; return rc; }
  return B2S_OK;
}

void b2s_destroy(b2s_sim* s) {
  if (!s) return;
  if (s->slot >= 0 && g_slots[s->device & 63][s->slot] == s) g_slots[s->device & 63][s->slot] = nullptr;
  cudaSetDevice(s->device);
  cudaDeviceSynchronize();  // kernels of this handle may still be reading its buffers
  for (void* p : s->allocs) cudaFree(p);
  for (auto q : s->gstreams) cudaStreamDestroy(q);
  for (auto ev : s->gevents) cudaEventDestroy(ev);
  if (s->in_event) cudaEventDestroy(s->in_event);
  for (auto& kv : s->graphs) cudaGraphExecDestroy(kv.second);
  delete s;
}

int b2s_set_stream(b2s_sim* s, void* stream) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  s->stream = (cudaStream_t)stream;
  return B2S_OK;
}

int b2s_set_export(b2s_sim* s, int flag) { if (!s) return fail(B2S_ERR_ARG, "null handle"); s->export_env_step = flag != 0; return B2S_OK; }

int64_t b2s_launch_count(const b2s_sim* s) { return s ? s->launches : 0; }

int b2s_array(b2s_sim* s, const char* name, void** dev_ptr, int* dtype, int* ndim, int64_t shape[4]) {
  if (!s || !name) return fail(B2S_ERR_ARG, "b2s_array: bad argument");
  auto it = s->arrays.find(name);
  if (it == s->arrays.end()) return fail(B2S_ERR_ARG, std::string("b2s_array: unknown array '") + name + "'");
  if (dev_ptr) *dev_ptr = it->second.ptr;
  if (dtype) *dtype = it->second.dtype;
  if (ndim) *ndim = it->second.ndim;
  if (shape) for (int k = 0; k < 4; k++) shape[k] = it->second.shape[k];
  return B2S_OK;
}

// upload this handle's descriptors into its constant-memory slot (only after a configuration change)
static int bind_constants(b2s_sim* s) {
  CUDA_TRY(cudaSetDevice(s->device));
  if (!s->dirty) return B2S_OK;
  const size_t k = (size_t)s->slot;
  int rc = with_real(s, [&](auto& m, auto& st) -> int {
    using D = DT<real_of<decltype(m)>>;
    CUDA_TRY(cudaMemcpyToSymbolAsync(D::model_bank(), &m, sizeof(m), k * sizeof(m), cudaMemcpyHostToDevice, s->stream));
    CUDA_TRY(cudaMemcpyToSymbolAsync(D::state_bank(), &st, sizeof(st), k * sizeof(st), cudaMemcpyHostToDevice, s->stream));
    return B2S_OK;
  });
  if (rc != B2S_OK) return rc;
  CUDA_TRY(cudaMemcpyToSymbolAsync(c_lay, s->lay, sizeof(s->lay), k * sizeof(s->lay), cudaMemcpyHostToDevice, s->stream));
  CUDA_TRY(cudaMemcpyToSymbolAsync(c_cc, &s->ctrl, sizeof(s->ctrl), k * sizeof(s->ctrl), cudaMemcpyHostToDevice, s->stream));
  CUDA_TRY(cudaMemcpyToSymbolAsync(c_pio, s->pio, sizeof(s->pio), k * sizeof(s->pio), cudaMemcpyHostToDevice, s->stream));
  // the host structs must outlive the asynchronous copies only until they are enqueued: pageable-memory sources are staged
  s->dirty = 0;
  return B2S_OK;
}

// layouts depend on where the OSC controller runs; a change invalidates the captured graphs (they carry block shapes)
static int rebuild_layouts(b2s_sim* s) {
  const bool osc = s->ctrl.kind == B2S_CTRL_OSC_POSE || s->ctrl.kind == B2S_CTRL_OSC_POSITION;
  int want = (osc && (!s->ctrl_split || s->mode == 2)) ? 1 : 0;  // unit-queue mode runs the controller inside the unit
  if (want == s->osc_in_tail && s->smem0 != 0) return B2S_OK;
  s->uq_wpb = 0;
  s->osc_in_tail = want;
  try { build_layouts(s, s->ncg, s->hc_stride); } catch (const std::string& e) { return fail(B2S_ERR_MODEL, e); }
  int rc = choose_blocks(s);
  if (rc != B2S_OK) return rc;
  if (with_real(s, [](auto&, auto& st) { return st.wsg != nullptr; })) { cudaSetDevice(s->device); cudaDeviceSynchronize(); }
  for (auto& kv : s->graphs) cudaGraphExecDestroy(kv.second);
  s->graphs.clear();
  s->dirty = 1;
  return B2S_OK;
}

static int launch(b2s_sim* s, int phases, int nsub, const void* action = nullptr, const uint8_t* mask = nullptr) {
  int rc = bind_constants(s);
  if (rc != B2S_OK) return rc;
  int blocks = (s->n_env + s->wpb_fused - 1) / s->wpb_fused;
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    step_kernel<R><<<blocks, s->wpb_fused * 32, s->smem_fused, s->stream>>>(phases, nsub, (const R*)action, s->slot, mask);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

}  // extern "C"

// the launches of `nsub` substeps of ONE environment group on stream q
template <typename R>
static int enqueue_group(b2s_sim* s, const DModel<R>& m, const DState<R>& st, int phases, int nsub, const R* action, int gi, int G, cudaStream_t q) {
  const int epaw = (EPA_AREA_WORDS(EPA_MAXV, EPA_MAXF) + m.stage_cap) * (int)sizeof(R);
  const int p1smem = std::max(epaw, (int)osc_smem_bytes<R>());  // one block shape for the three roles of phase 1
  int e0 = (int)((long long)s->n_env * gi / G), e1 = (int)((long long)s->n_env * (gi + 1) / G);
  Grp g{e0, e1 - e0, gi, 0, s->slot};
  int blocks0 = (g.nenv + s->wpb0 - 1) / s->wpb0, blocks5 = (g.nenv + s->wpb5 - 1) / s->wpb5;
  int nA = g.nenv * st.cl_maxa, nG = g.nenv * st.cl_maxg;
  // convex role: one warp per block, items claimed through a counter.  ~1.6 items per environment are queued per substep (Lift), most of
  // them dismissed in a few microseconds: half a block per environment keeps every slow item on its own warp without flooding the
  // block scheduler with thousands of empty blocks per launch
  const int cvx_blocks = std::max(s->num_sms, g.nenv / 2);
  const bool ctrl_ext = (phases & PH_CTRL_EXT) != 0;
  // the group's work-list counters and both tail class sets for substep 0 (each tail launch zeroes them for the next substep)
  CUDA_TRY(cudaMemsetAsync(st.cl_cnt + CL_CNT_STRIDE * gi, 0, CL_CNT_STRIDE * sizeof(int), q));
  for (int sub = 0; sub < nsub; sub++) {
    g.sub = sub;
    phase0_kernel<R><<<blocks0, s->wpb0 * 32, s->smem0, q>>>(phases, g);
    // phase 1: convex narrow phase | controller | analytic narrow phase as block roles of ONE launch (no forks in the graph).
    // Upper bounds of the candidate counts size the grid; warps / threads beyond the device-side counts exit at once.
    P1Cfg c{std::min(nG, cvx_blocks), ctrl_ext ? (g.nenv + OSC_TPB - 1) / OSC_TPB : 0, sub};
    int nAb = (nA + 31) / 32;
    if (c.nG + c.nC + nAb > 0) phase1_kernel<R><<<c.nG + c.nC + nAb, 32, p1smem, q>>>(action, g, c);
    if (s->tail_wide) tail_kernel<R, TAIL_WIDE_THREADS, true><<<blocks5, s->wpb5 * 32, s->smem5, q>>>(phases, nsub, action, g, s->stride5, s->stride5l, s->nlw5);
    else if (st.tail_sorted) tail_kernel<R, TAIL_THREADS, true><<<blocks5, s->wpb5 * 32, s->smem5, q>>>(phases, nsub, action, g, s->stride5, s->stride5l, s->nlw5);
    else tail_kernel<R, TAIL_THREADS, false><<<blocks5, s->wpb5 * 32, s->smem5, q>>>(phases, nsub, action, g, s->stride5, s->stride5l, s->nlw5);
  }
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

// global workspace rows + per-environment candidate tables / narrow-phase output slots (pipeline and unit-queue modes)
template <typename R> static int ensure_ws(b2s_sim* s, const DModel<R>& m, DState<R>& st) {
  if (!st.wsg) {
    R* p = nullptr;
    if (cudaMalloc(&p, (size_t)s->n_env * s->lay[LAY_ROW].total * sizeof(R)) != cudaSuccess) return fail(B2S_ERR_CUDA, "cudaMalloc(pipeline workspace) failed");
    cudaMemsetAsync(p, 0, (size_t)s->n_env * s->lay[LAY_ROW].total * sizeof(R), s->stream);
    s->allocs.push_back(p);
    st.wsg = p;
    size_t ne = (size_t)s->n_env;
    st.cl_cnt = dev_zeros<int>(s, CL_CNT_STRIDE * 64);
    st.tail_key = dev_zeros<int>(s, ne); st.tail_list = dev_zeros<int>(s, ne * TAIL_NKEY); st.tail_order = dev_zeros<int>(s, ne);
    s->arrays["tail_key"] = ArrayInfo{st.tail_key, B2S_I32, 1, {(int64_t)ne, 0, 0, 0}};
    s->arrays["tail_order"] = ArrayInfo{st.tail_order, B2S_I32, 1, {(int64_t)ne, 0, 0, 0}};
    // candidate capacity per environment: small models keep small grids (the narrow-phase grids are sized by these bounds)
    st.cl_maxa = s->maxcon <= 32 ? 8 : (s->maxcon <= 48 ? 16 : CL_MAXA);
    st.cl_maxg = s->maxcon <= 32 ? 16 : CL_MAXG;
    st.cl_listA = dev_zeros<int>(s, ne * st.cl_maxa); st.cl_listG = dev_zeros<int>(s, ne * st.cl_maxg);
    st.cl_outA = dev_zeros<R>(s, ne * st.cl_maxa * CL_RECA); st.cl_outG = dev_zeros<R>(s, ne * st.cl_maxg * 8);
    st.cl_env = dev_zeros<int>(s, ne * CL_ENVW(st));
    st.gjk_cache = getenv("B2S_NO_GJK_CACHE") ? nullptr : dev_zeros<R>(s, ne * (size_t)m.npair * 3);
    s->action_buf = dev_zeros<R>(s, ne * 16);
#ifdef B2S_INSTR
    st.st_begin = dev_zeros<unsigned long long>(s, 64 * 32 * 8); st.st_end = dev_zeros<unsigned long long>(s, 64 * 32 * 8);
    st.stats = dev_zeros<int>(s, 512); st.cyc = dev_zeros<float>(s, ne * 32 * 8); st.solve_ls = dev_zeros<int>(s, ne);
    s->arrays["st_begin"] = ArrayInfo{st.st_begin, B2S_I64, 1, {64 * 32 * 8, 0, 0, 0}};
    s->arrays["st_end"] = ArrayInfo{st.st_end, B2S_I64, 1, {64 * 32 * 8, 0, 0, 0}};
    s->arrays["stats"] = ArrayInfo{st.stats, B2S_I32, 1, {512, 0, 0, 0}};
    s->arrays["cyc"] = ArrayInfo{st.cyc, B2S_F32, 3, {(int64_t)ne, 32, 8, 0}};
    st.slowlog = dev_zeros<int>(s, 64 * 12);
    s->arrays["slowlog"] = ArrayInfo{st.slowlog, B2S_I32, 2, {64, 12, 0, 0}};
    s->uq_prof = dev_zeros<unsigned long long>(s, 16);
    s->arrays["unit_prof"] = ArrayInfo{s->uq_prof, B2S_I64, 1, {16, 0, 0, 0}};
#endif
    s->dirty = 1;
    s->layout_version++;  // the GJK cache now exists
  }
  return B2S_OK;
}

// ---- pipeline mode: CUDA-graph replay.  The launch sequence of one environment group (nsub substeps x 3 kernels) is captured
// once per (phases, nsub, action given) and replayed on the group's own stream, forked from and joined to the handle's stream: the
// groups' chains then overlap freely (inside ONE graph, parallel branches were observed to share a limited number of execution
// lanes).  The action rows are staged into a fixed buffer so kernel arguments never change.
static int launch_pipeline(b2s_sim* s, int phases, int nsub, const void* action) {
  return with_real(s, [&](auto& m, auto& st) -> int {
    using R = real_of<decltype(m)>;
    { int rc0 = ensure_ws(s, m, st); if (rc0 != B2S_OK) return rc0; }
#ifdef B2S_INSTR
    cudaMemsetAsync(st.st_begin, 0xff, sizeof(unsigned long long) * 64 * 32 * 8, s->stream);
    cudaMemsetAsync(st.st_end, 0, sizeof(unsigned long long) * 64 * 32 * 8, s->stream);
#endif
    const bool osc = s->ctrl.kind == B2S_CTRL_OSC_POSE || s->ctrl.kind == B2S_CTRL_OSC_POSITION;
    if ((phases & PH_CTRL) && osc && s->ctrl_split) phases |= PH_CTRL_EXT;
    { int rc2 = rebuild_layouts(s); if (rc2 != B2S_OK) return rc2; }  // before the descriptors are (re)uploaded
    int rc = bind_constants(s);
    if (rc != B2S_OK) return rc;
    const int G = std::min(s->ngroups, s->n_env);
    while ((int)s->gstreams.size() < G) {
      cudaStream_t st2; cudaEvent_t ev;
      CUDA_TRY(cudaStreamCreateWithFlags(&st2, cudaStreamNonBlocking));
      CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
      s->gstreams.push_back(st2); s->gevents.push_back(ev);
    }
    if (!s->in_event) CUDA_TRY(cudaEventCreateWithFlags(&s->in_event, cudaEventDisableTiming));
    const int launches_per_call = G * nsub * 3;  // phase 0, phase 1 (narrow phase + controller), tail (both capacity tiers)
    const R* act_in = (const R*)action;
    if (action) {
      int ad = s->ctrl.action_dim > 0 ? s->ctrl.action_dim : 1;
      if (ad > 16) return fail(B2S_ERR_UNSUPPORTED, "action_dim > 16");
      CUDA_TRY(cudaMemcpyAsync(s->action_buf, action, (size_t)s->n_env * ad * sizeof(R), cudaMemcpyDeviceToDevice, s->stream));
      act_in = (const R*)s->action_buf;
    }
    CUDA_TRY(cudaEventRecord(s->in_event, s->stream));
    for (int gi = 0; gi < G; gi++) {
      long long key = ((long long)phases << 28) | ((long long)(gi + 1) << 20) | (long long)nsub << 4 | (action ? 1 : 0);
      cudaStream_t q = s->gstreams[gi];
      auto it = s->graphs.find(key);
      if (it == s->graphs.end()) {
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        CUDA_TRY(cudaStreamBeginCapture(q, cudaStreamCaptureModeRelaxed));
        rc = enqueue_group(s, m, st, phases, nsub, act_in, gi, G, q);
        cudaError_t ce = cudaStreamEndCapture(q, &graph);
        if (rc != B2S_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (ce != cudaSuccess) return fail(B2S_ERR_CUDA, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
        CUDA_TRY(cudaGraphInstantiate(&exec, graph, 0));
        cudaGraphDestroy(graph);
        it = s->graphs.emplace(key, exec).first;
      }
      CUDA_TRY(cudaStreamWaitEvent(q, s->in_event, 0));
      CUDA_TRY(cudaGraphLaunch(it->second, q));
      CUDA_TRY(cudaEventRecord(s->gevents[gi], q));
      CUDA_TRY(cudaStreamWaitEvent(s->stream, s->gevents[gi], 0));
    }
    s->launches += launches_per_call;
    return B2S_OK;
  });
}

// ---- unit-queue mode: one persistent kernel per control step (b2s_unit.cuh)
static int launch_unit(b2s_sim* s, int phases, int nsub, const void* action) {
  return with_real(s, [&](auto& m, auto& st) -> int {
    using R = real_of<decltype(m)>;
    { int rc0 = ensure_ws(s, m, st); if (rc0 != B2S_OK) return rc0; }
    { int rc2 = rebuild_layouts(s); if (rc2 != B2S_OK) return rc2; }
    const int total = s->n_env * nsub;
    if ((long long)s->n_env * nsub > (1ll << 30)) return fail(B2S_ERR_UNSUPPORTED, "unit-queue mode: n_env * nsub too large");
    if (total > s->uq_cap) {
      cudaStreamSynchronize(s->stream);
      int* p = nullptr;
      if (cudaMalloc(&p, sizeof(int) * (2 * (size_t)total + 8)) != cudaSuccess) return fail(B2S_ERR_CUDA, "cudaMalloc(unit ring) failed");
      s->allocs.push_back(p);
      s->uq_ring = p; s->uq_ovf = p + total; s->uq_ctr = p + 2 * (size_t)total; s->uq_cap = total;
#ifdef B2S_INSTR
      s->arrays["unit_ctr"] = ArrayInfo{s->uq_ctr, B2S_I32, 1, {8, 0, 0, 0}};
#endif
    }
    if (s->uq_wpb == 0) {
      // block shape: the warp's one workspace area holds phase 0's layout, then the EPA polytope + vertex staging, then the small tail tier
      const size_t rsz = sizeof(R);
      const bool tiered = s->mc_small < s->maxcon || s->me_small < s->maxefc;
      int stride = std::max(std::max(s->lay[LAY_P0].total, s->lay[LAY_TS].total), EPA_AREA_WORDS(EPA_MAXV, EPA_MAXF) + 24 + 384);
      stride = (stride + 3) & ~3;
      int stride_l = (s->lay[LAY_TL].total + 3) & ~3;
      CUDA_TRY(optin_max_smem(unit_kernel<R>, s->device));
      int best_w = 0, best_b = 0, best = 0;
      for (int w = UNIT_THREADS / 32; w >= 1; w--) {
        size_t sm = std::max((size_t)w * stride, tiered ? (size_t)stride_l : 0) * rsz;
        if (sm > 226 * 1024) continue;
        int b = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, unit_kernel<R>, w * 32, sm) != cudaSuccess) { cudaGetLastError(); continue; }
        if (w * b > best) { best = w * b; best_w = w; best_b = b; }
      }
      if (best == 0) return fail(B2S_ERR_UNSUPPORTED, "unit-queue mode: workspace does not fit shared memory");
      s->uq_stride = stride; s->uq_stride_large = stride_l;
      s->uq_smem = std::max((size_t)best_w * stride, tiered ? (size_t)stride_l : 0) * rsz;
      s->uq_wpb_large = tiered ? std::min(best_w, (int)(s->uq_smem / rsz / stride_l)) : 0;
      int slots = best_b * s->num_sms;
      // a large-role block occupies a block slot (a whole SM at one block per SM)
      int nl = tiered ? std::max(1, std::min(slots / 64, 12)) : 0;
      s->uq_nlarge = nl;
      if (best_w > s->n_env) best_w = s->n_env;  // the lockstep rounds need n_env >= warps per block (b2s_unit.cuh)
      s->uq_wpb = best_w;
      int small_blocks = std::min(std::max(slots - nl, 1), (s->n_env + best_w - 1) / best_w);
      s->uq_grid = nl + small_blocks;
      if (getenv("B2S_VERBOSE"))
        fprintf(stderr, "[b2s] unit-queue: %d warps/block x %d blocks/SM, %d words/warp (large role: %d words, %d warps/block, %d blocks), grid %d, smem %zu B\n",
                best_w, best_b, stride, stride_l, s->uq_wpb_large, nl, s->uq_grid, s->uq_smem);
    }
    int rc = bind_constants(s);
    if (rc != B2S_OK) return rc;
    UnitQ q{s->uq_ring, s->uq_ovf, s->uq_ctr, total, s->uq_nlarge, s->uq_wpb_large, s->uq_stride, s->uq_stride_large};
#ifdef B2S_INSTR
    q.prof = s->uq_prof;
#endif
    unit_init_kernel<R><<<(total + 255) / 256, 256, 0, s->stream>>>(q, s->n_env);
    unit_kernel<R><<<s->uq_grid, s->uq_wpb * 32, s->uq_smem, s->stream>>>(phases, nsub, (const R*)action, s->slot, q);
    unit_check_kernel<R><<<8, 256, 0, s->stream>>>(q, s->slot);
    s->launches += 3;
    CUDA_TRY(cudaGetLastError());
    return B2S_OK;
  });
}

extern "C" {

/* Host-only: the workspace layouts libb2s would build for a model of the given dimensions (no device needed).  out_words[5] receives
 * words per warp / row of LAY_FULL (incl. the EPA area), LAY_P0, LAY_TS, LAY_TL, LAY_ROW; out_layouts (may be NULL) receives the five
 * WSLayout structs as ints, out_pio (may be NULL) B2S_NPIO x (nload, nstore, load_words, then 12 + 12 regions x 4 ints). */
int b2s_debug_layouts(int nq, int nv, int nu, int nbody, int ncg, int nsite, int hc_stride, int maxcon, int maxefc, int mc_small,
                      int me_small, int osc_in_tail, int* out_words, int* out_layouts, int* out_pio) {
  b2s_sim tmp;
  tmp.nq = nq; tmp.nv = nv; tmp.nu = nu; tmp.nbody = nbody; tmp.nsite = nsite; tmp.maxcon = maxcon; tmp.maxefc = maxefc;
  tmp.mc_small = mc_small; tmp.me_small = me_small; tmp.osc_in_tail = osc_in_tail;
  try { build_layouts(&tmp, ncg, hc_stride); } catch (const std::string& e) { return fail(B2S_ERR_MODEL, e); }
  if (out_words) {
    out_words[0] = tmp.lay[LAY_FULL].fused_stride;
    for (int k = 1; k < B2S_NLAY; k++) out_words[k] = tmp.lay[k].total;
  }
  if (out_layouts) memcpy(out_layouts, tmp.lay, sizeof(tmp.lay));
  if (out_pio) {
    for (int k = 0; k < B2S_NPIO; k++) {
      int* o = out_pio + k * (3 + 2 * B2S_MAXREG * 4);
      o[0] = tmp.pio[k].nload; o[1] = tmp.pio[k].nstore; o[2] = tmp.pio[k].load_words;
      memcpy(o + 3, tmp.pio[k].load, sizeof(Region) * B2S_MAXREG);
      memcpy(o + 3 + 4 * B2S_MAXREG, tmp.pio[k].store, sizeof(Region) * B2S_MAXREG);
    }
  }
  return B2S_OK;
}

int b2s_set_mode(b2s_sim* s, int mode) {
  if (!s || mode < 0 || mode > 2) return fail(B2S_ERR_ARG, "b2s_set_mode: mode must be 0 (fused), 1 (pipeline) or 2 (unit queue)");
  s->mode = mode;
  const char* eg = getenv("B2S_GROUPS");
  if (eg) { int v = atoi(eg); if (v >= 1 && v <= 64) s->ngroups = v; }
  if (const char* v = getenv("B2S_CTRL_SPLIT")) s->ctrl_split = atoi(v) != 0;
  return B2S_OK;
}

static void clear_warm_start(b2s_sim* s, const uint8_t* mask) {
  with_real(s, [&](auto& m, auto& st) {
    using R = real_of<decltype(m)>;
    if (!st.gjk_cache || m.npair == 0) return;
    size_t total = (size_t)s->n_env * m.npair * 3;
    int blocks = (int)((total + 255) / 256);
    cache_reset_kernel<R><<<blocks, 256, 0, s->stream>>>(mask, s->slot);
    s->launches++;
  });
}

int b2s_reset(b2s_sim* s, const uint8_t* mask) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    reset_kernel<R><<<(s->n_env + 127) / 128, 128, 0, s->stream>>>(mask, s->slot);
  });
  clear_warm_start(s, mask);
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return launch_set_const(s, mask);
}

int b2s_forward(b2s_sim* s) { return s ? launch(s, PH_STEP1 | PH_STEP2 | PH_NOINTEGRATE | PH_EXPORT | (s->has_obs ? PH_OBS : 0), 1) : fail(B2S_ERR_ARG, "null handle"); }
int b2s_step1(b2s_sim* s) { return s ? launch(s, PH_STEP1 | PH_EXPORT, 1) : fail(B2S_ERR_ARG, "null handle"); }
int b2s_step2(b2s_sim* s) { return s ? launch(s, PH_STEP1 | PH_STEP2 | PH_EXPORT, 1) : fail(B2S_ERR_ARG, "null handle"); }
int b2s_step(b2s_sim* s, int n) {
  if (!s || n < 1) return fail(B2S_ERR_ARG, "b2s_step: bad argument");
  if (s->mode == 2) return launch_unit(s, PH_STEP1 | PH_STEP2, n, nullptr);
  if (s->mode == 1) return launch_pipeline(s, PH_STEP1 | PH_STEP2, n, nullptr);
  return launch(s, PH_STEP1 | PH_STEP2, n);
}

int b2s_jac_site(b2s_sim* s, int site_id, void* jacp, void* jacr) {
  if (!s || site_id < 0 || site_id >= s->nsite) return fail(B2S_ERR_ARG, "b2s_jac_site: bad argument");
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  int threads = 128, blocks = (s->n_env * s->nv + threads - 1) / threads;
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    jac_site_kernel<R><<<blocks, threads, 0, s->stream>>>(site_id, (R*)jacp, (R*)jacr, s->slot);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

int b2s_get_state(b2s_sim* s, void* out) {
  if (!s || !out) return fail(B2S_ERR_ARG, "b2s_get_state: bad argument");
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  size_t total = (size_t)s->n_env * (1 + s->nq + s->nv);
  int blocks = (int)((total + 255) / 256);
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    state_io_kernel<R><<<blocks, 256, 0, s->stream>>>((R*)out, 0, s->slot);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}
int b2s_set_state(b2s_sim* s, const void* in) {
  if (!s || !in) return fail(B2S_ERR_ARG, "b2s_set_state: bad argument");
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  size_t total = (size_t)s->n_env * (1 + s->nq + s->nv);
  int blocks = (int)((total + 255) / 256);
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    state_io_kernel<R><<<blocks, 256, 0, s->stream>>>((R*)in, 1, s->slot);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}
int b2s_name2id(const b2s_sim* s, const char* type, const char* name) {
  if (!s || !type || !name) return -1;
  auto it = s->names.find(type);
  if (it == s->names.end()) return -1;
  for (size_t i = 0; i < it->second.size(); i++) if (it->second[i] == name) return (int)i;
  return -1;
}
const char* b2s_id2name(const b2s_sim* s, const char* type, int id) {
  if (!s || !type) return nullptr;
  auto it = s->names.find(type);
  if (it == s->names.end() || id < 0 || id >= (int)it->second.size()) return nullptr;
  return it->second[id].c_str();
}
int b2s_full_m(b2s_sim* s, void* out) {
  if (!s || !out) return fail(B2S_ERR_ARG, "b2s_full_m: bad argument");
  const void* src = with_real(s, [](auto&, auto& st) -> const void* { return st.qM; });
  CUDA_TRY(cudaMemcpyAsync(out, src, (size_t)s->n_env * s->nv * s->nv * real_size(s), cudaMemcpyDeviceToDevice, s->stream));
  return B2S_OK;
}
static int jac_point(b2s_sim* s, int kind, int id, void* jacp, void* jacr) {
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  int threads = 128, blocks = (s->n_env * s->nv + threads - 1) / threads;
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    jac_point_kernel<R><<<blocks, threads, 0, s->stream>>>(kind, id, (R*)jacp, (R*)jacr, s->slot);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}
int b2s_jac_body(b2s_sim* s, int body_id, void* jacp, void* jacr) {
  if (!s || body_id < 0 || body_id >= s->nbody) return fail(B2S_ERR_ARG, "b2s_jac_body: bad argument");
  return jac_point(s, 0, body_id, jacp, jacr);
}
int b2s_jac_geom(b2s_sim* s, int geom_id, void* jacp, void* jacr) {
  if (!s || geom_id < 0 || geom_id >= s->ngeom) return fail(B2S_ERR_ARG, "b2s_jac_geom: bad argument");
  return jac_point(s, 1, geom_id, jacp, jacr);
}

int b2s_ctrl_config(b2s_sim* s, const b2s_ctrl_cfg* c) {
  if (!s || !c) return fail(B2S_ERR_ARG, "b2s_ctrl_config: bad argument");
  if (c->kind != B2S_CTRL_OSC_POSE && c->kind != B2S_CTRL_JOINT_VELOCITY && c->kind != B2S_CTRL_JOINT_POSITION &&
      c->kind != B2S_CTRL_JOINT_TORQUE && c->kind != B2S_CTRL_OSC_POSITION && c->kind != B2S_CTRL_NONE)
    return fail(B2S_ERR_UNSUPPORTED, "controller kind not implemented");
  if (c->n_arm > 8 || c->n_grip > 4) return fail(B2S_ERR_ARG, "b2s_ctrl_config: too many joints");
  CtrlCfgDev& d = s->ctrl;
  d.kind = c->kind; d.action_dim = c->action_dim; d.n_arm = c->n_arm; d.eef_site = c->eef_site; d.base_site = c->base_site;
  d.n_grip = c->n_grip; d.uncouple = c->uncouple_pos_ori;
  for (int i = 0; i < 8; i++) { d.arm_dof[i] = c->arm_dof[i]; d.arm_qpos[i] = c->arm_qpos[i]; d.arm_act[i] = c->arm_act[i]; }
  for (int i = 0; i < 4; i++) { d.grip_act[i] = c->grip_act[i]; d.grip_sign[i] = c->grip_sign[i]; }
  d.grip_speed = c->grip_speed; d.null_kp = c->null_kp;
  for (int i = 0; i < 6; i++) {
    d.kp[i] = c->kp[i]; d.kd[i] = 2.0 * sqrt(c->kp[i]) * c->damping_ratio[i];
    d.input_max[i] = c->input_max[i]; d.input_min[i] = c->input_min[i];
    d.output_max[i] = c->output_max[i]; d.output_min[i] = c->output_min[i];
  }
  for (int i = 0; i < 8; i++) {
    d.jv_kp[i] = c->jv_kp[i]; d.jv_ki[i] = c->jv_ki[i]; d.jv_kd[i] = c->jv_kd[i];
    d.jv_in_max[i] = c->jv_in_max[i]; d.jv_in_min[i] = c->jv_in_min[i]; d.jv_out_max[i] = c->jv_out_max[i]; d.jv_out_min[i] = c->jv_out_min[i];
  }
  d.jv_vel_lo = c->jv_vel_lo; d.jv_vel_hi = c->jv_vel_hi; d.jv_use_vel_limits = c->jv_use_vel_limits; d.jv_torque_comp = c->jv_torque_comp;
  s->has_ctrl = c->kind != B2S_CTRL_NONE;
  s->dirty = 1;
  s->layout_version++;  // the controller kind is part of the snapshot signature
  return B2S_OK;
}

int b2s_ctrl_reset(b2s_sim* s, const uint8_t* mask) {
  if (!s || !s->has_ctrl) return fail(B2S_ERR_ARG, "b2s_ctrl_reset: controller not configured");
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  int threads = 128, blocks = (s->n_env + threads - 1) / threads;
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    ctrl_reset_kernel<R><<<blocks, threads, 0, s->stream>>>(mask, s->slot);
  });
  clear_warm_start(s, mask);  // an environment whose controller is rebuilt starts a new episode
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

int b2s_reset_envs(b2s_sim* s, const uint8_t* mask, const void* qpos_new) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  int threads = 128, blocks = (s->n_env + threads - 1) / threads;
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    reset_envs_kernel<R><<<blocks, threads, 0, s->stream>>>(mask, (const R*)qpos_new, s->slot);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  { int rc = launch_set_const(s, mask); if (rc != B2S_OK) return rc; }  // after the warn bits were cleared: bit 128 survives
  int rc = launch(s, PH_STEP1 | PH_STEP2 | PH_NOINTEGRATE | PH_EXPORT | (s->has_obs ? PH_OBS : 0), 1, nullptr, mask);
  if (rc != B2S_OK) return rc;
  if (s->has_ctrl) return b2s_ctrl_reset(s, mask);
  clear_warm_start(s, mask);
  return B2S_OK;
}

}  // extern "C"
template <typename R> static int body_pose_override_t(b2s_sim* s, DState<R>& st, int body) {
  for (int k = 0; k < st.n_ov; k++) if (st.ov_body[k] == body) return B2S_OK;
  if (st.n_ov >= 4) return fail(B2S_ERR_UNSUPPORTED, "b2s_body_pose_override: at most 4 bodies per handle");
  std::vector<R> hp((size_t)s->n_env * 3), hq((size_t)s->n_env * 4);
  for (int e = 0; e < s->n_env; e++) {
    for (int k = 0; k < 3; k++) hp[(size_t)e * 3 + k] = (R)s->xpos0_h[3 * body + k];
    for (int k = 0; k < 4; k++) hq[(size_t)e * 4 + k] = (R)s->xquat0_h[4 * body + k];
  }
  const int k = st.n_ov;
  try { st.ov_pos[k] = dev_upload(s, hp); st.ov_quat[k] = dev_upload(s, hq); } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
  st.ov_body[k] = body;
  st.n_ov = k + 1;
  const int code = DT<R>::code;
  s->arrays["body_xpos_ov:" + std::to_string(body)] = ArrayInfo{st.ov_pos[k], code, 2, {s->n_env, 3, 0, 0}};
  s->arrays["body_xquat_ov:" + std::to_string(body)] = ArrayInfo{st.ov_quat[k], code, 2, {s->n_env, 4, 0, 0}};
  s->dirty = 1;
  s->layout_version++;
  return B2S_OK;
}
// ---- per-environment model values (b2s_model_override) and the set-constants pass
static bool has_model_overrides(b2s_sim* s) { return with_real(s, [](auto&, auto& st) { return st.dof_iw != nullptr; }); }

template <typename R> static void upload_rows(R* dst, const double* src, int k, size_t n_env) {  // n_env copies of src[0..k)
  std::vector<R> h(n_env * k);
  for (size_t e = 0; e < n_env; e++) for (int q = 0; q < k; q++) h[e * k + q] = (R)src[q];
  cudaMemcpy(dst, h.data(), h.size() * sizeof(R), cudaMemcpyHostToDevice);
  cudaStreamSynchronize(cudaStreamLegacy);  // see dev_upload
}

// geom fields a caller declares; declaring either one gives the geom a slot, and the slot also carries the geom's contact solref /
// solimp ("geom_solref:<id>", "geom_solimp:<id>"), as it carries its bounding radius and box
static bool is_geom_decl_field(const std::string& f) { return f == "geom_size" || f == "geom_friction"; }
// every per-environment geom array a perturbation may write
static bool is_geom_field(const std::string& f) { return is_geom_decl_field(f) || f == "geom_solref" || f == "geom_solimp"; }
static bool is_body_field(const std::string& f) { return f == "body_mass" || f == "body_inertia"; }
static bool is_dof_field(const std::string& f) { return f == "dof_damping" || f == "dof_armature" || f == "dof_frictionloss"; }
// name of the per-environment array of (field, id): "<field>" for the whole-vector dof fields, "<field>:<id>" otherwise
static std::string override_key(const std::string& f, int id) { return is_dof_field(f) ? f : f + ":" + std::to_string(id); }

template <typename R> static int model_override_t(b2s_sim* s, DState<R>& st, const std::string& field, int id) {
  const bool geom = is_geom_decl_field(field);
  const size_t N = s->n_env;
  const int code = DT<R>::code;
  try {
    if (!st.dof_iw) {  // first override of the handle: the banks of every slot, the derived constants from the model's values
      st.mg_size = dev_zeros<R>(s, B2S_MOV * N * 3); st.mg_fric = dev_zeros<R>(s, B2S_MOV * N * 3);
      st.mg_rbound = dev_zeros<R>(s, B2S_MOV * N); st.mg_aabb = dev_zeros<R>(s, B2S_MOV * N * 6);
      st.mg_solref = dev_zeros<R>(s, B2S_MOV * N * 2); st.mg_solimp = dev_zeros<R>(s, B2S_MOV * N * 5);
      st.mb_mass = dev_zeros<R>(s, B2S_MOV * N); st.mb_inertia = dev_zeros<R>(s, B2S_MOV * N * 3);
      R* diw = dev_zeros<R>(s, N * s->nv); R* biw = dev_zeros<R>(s, N * s->nbody * 2); R* mi = dev_zeros<R>(s, N);
      upload_rows(diw, s->dof_iw_h.data(), s->nv, N);
      upload_rows(biw, s->body_iw_h.data(), 2 * s->nbody, N);
      upload_rows(mi, &s->meaninertia_h, 1, N);
      s->arrays["dof_invweight0"] = ArrayInfo{diw, code, 2, {s->n_env, s->nv, 0, 0}};
      s->arrays["body_invweight0"] = ArrayInfo{biw, code, 3, {s->n_env, s->nbody, 2, 0}};
      s->arrays["meaninertia"] = ArrayInfo{mi, code, 1, {s->n_env, 0, 0, 0}};
      st.dof_iw = diw; st.body_iw = biw; st.mean_inertia = mi;
    }
    const std::string key = override_key(field, id);
    if (s->arrays.count(key)) return B2S_OK;
    if (is_dof_field(field)) {
      const std::vector<double>& h = field == "dof_damping" ? s->dof_damping_h : field == "dof_armature" ? s->dof_armature_h : s->dof_frictionloss_h;
      R* p = dev_zeros<R>(s, N * s->nv);
      upload_rows(p, h.data(), s->nv, N);
      (field == "dof_damping" ? st.dof_damp : field == "dof_armature" ? st.dof_arm : st.dof_floss) = p;
      s->arrays[key] = ArrayInfo{p, code, 2, {s->n_env, s->nv, 0, 0}};
    } else if (geom) {
      int k = 0;
      while (k < st.n_mg && st.mg_id[k] != id) k++;
      if (k == st.n_mg) {  // a new slot: size, friction, bounds, solref, solimp of this geom for every environment
        if (k >= B2S_MOV) return fail(B2S_ERR_UNSUPPORTED, "b2s_model_override: at most 8 geoms per handle");
        upload_rows(st.mg_size + k * N * 3, &s->geom_size_h[3 * id], 3, N);
        upload_rows(st.mg_fric + k * N * 3, &s->geom_friction_h[3 * id], 3, N);
        upload_rows(st.mg_rbound + k * N, &s->geom_rbound_h[id], 1, N);
        upload_rows(st.mg_aabb + k * N * 6, &s->geom_aabb_h[6 * id], 6, N);
        upload_rows(st.mg_solref + k * N * 2, &s->geom_solref_h[2 * id], 2, N);
        upload_rows(st.mg_solimp + k * N * 5, &s->geom_solimp_h[5 * id], 5, N);
        st.mg_id[k] = (short)id; st.n_mg = k + 1;
        s->arrays["geom_rbound:" + std::to_string(id)] = ArrayInfo{st.mg_rbound + k * N, code, 1, {s->n_env, 0, 0, 0}};
        s->arrays["geom_aabb:" + std::to_string(id)] = ArrayInfo{st.mg_aabb + k * N * 6, code, 2, {s->n_env, 6, 0, 0}};
        s->arrays["geom_solref:" + std::to_string(id)] = ArrayInfo{st.mg_solref + k * N * 2, code, 2, {s->n_env, 2, 0, 0}};
        s->arrays["geom_solimp:" + std::to_string(id)] = ArrayInfo{st.mg_solimp + k * N * 5, code, 2, {s->n_env, 5, 0, 0}};
      }
      R* p = field == "geom_size" ? st.mg_size + k * N * 3 : st.mg_fric + k * N * 3;
      s->arrays[key] = ArrayInfo{p, code, 2, {s->n_env, 3, 0, 0}};
    } else {
      int k = 0;
      while (k < st.n_mb && st.mb_id[k] != id) k++;
      if (k == st.n_mb) {
        if (k >= B2S_MOV) return fail(B2S_ERR_UNSUPPORTED, "b2s_model_override: at most 8 bodies per handle");
        upload_rows(st.mb_mass + k * N, &s->body_mass_h[id], 1, N);
        upload_rows(st.mb_inertia + k * N * 3, &s->body_inertia_h[3 * id], 3, N);
        st.mb_id[k] = (short)id; st.n_mb = k + 1;
      }
      if (field == "body_mass") s->arrays[key] = ArrayInfo{st.mb_mass + k * N, code, 1, {s->n_env, 0, 0, 0}};
      else s->arrays[key] = ArrayInfo{st.mb_inertia + k * N * 3, code, 2, {s->n_env, 3, 0, 0}};
    }
  } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
  s->dirty = 1;
  s->layout_version++;
  return B2S_OK;
}

static int launch_set_const(b2s_sim* s, const uint8_t* mask) {
  if (!has_model_overrides(s)) return B2S_OK;
  { int rc = bind_constants(s); if (rc != B2S_OK) return rc; }
  return with_real(s, [&](auto& m, auto&) -> int {
    using R = real_of<decltype(m)>;
    if (s->sc_words == 0) {
      CUDA_TRY(optin_max_smem(set_const_kernel<R>, s->device));
      s->sc_words = s->lay[LAY_FULL].total + ((s->nv * s->nv + 3) & ~3);
    }
    const int wpb = fit_wpb((size_t)s->sc_words * sizeof(R), 16), blocks = (s->n_env + wpb - 1) / wpb;
    const size_t smem = (size_t)s->sc_words * sizeof(R) * wpb;
    set_const_kernel<R><<<blocks, wpb * 32, smem, s->stream>>>(mask, s->slot, s->sc_words);
    s->launches++;
    CUDA_TRY(cudaGetLastError());
    return B2S_OK;
  });
}

extern "C" {
int b2s_model_override(b2s_sim* s, const char* field, int id) {
  if (!s || !field) return fail(B2S_ERR_ARG, "b2s_model_override: bad argument");
  const std::string f = field;
  if (is_geom_decl_field(f)) {
    if (id < 0 || id >= s->ngeom) return fail(B2S_ERR_ARG, "b2s_model_override: geom id out of range");
    const int t = s->geom_type_h[id];
    if (s->cgid[id] < 0 || !(t == G_SPHERE || t == G_CAPSULE || t == G_ELLIPSOID || t == G_CYLINDER || t == G_BOX))
      return fail(B2S_ERR_UNSUPPORTED, "b2s_model_override: only colliding sphere, capsule, ellipsoid, cylinder and box geoms have per-environment values");
  } else if (is_body_field(f)) {
    if (id < 0 || id >= s->nbody) return fail(B2S_ERR_ARG, "b2s_model_override: body id out of range");
    if (s->body_weldid_h[id] == 0) return fail(B2S_ERR_UNSUPPORTED, "b2s_model_override: the body does not move (world body or welded to it)");
  } else if (is_dof_field(f)) {
    if (id != -1) return fail(B2S_ERR_ARG, "b2s_model_override: the dof fields are whole vectors (id -1)");
    // any dof may get a friction-loss row: the large tier must hold nv of them besides the limit and contact rows
    if (f == "dof_frictionloss" && s->maxefc < s->nv + 8)
      return fail(B2S_ERR_UNSUPPORTED, "b2s_model_override: opt_maxefc cannot hold a friction-loss row for every dof (needs nv + 8)");
  } else {
    return fail(B2S_ERR_ARG, "b2s_model_override: unknown field '" + f + "' (geom_size, geom_friction, body_mass, body_inertia, "
                             "dof_damping, dof_armature, dof_frictionloss; a declared geom's solref / solimp come with its slot)");
  }
  CUDA_TRY(cudaSetDevice(s->device));
  return with_real(s, [&](auto&, auto& st) { return model_override_t(s, st, f, id); });
}

int b2s_set_const(b2s_sim* s, const uint8_t* env_mask) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  return launch_set_const(s, env_mask);
}

int b2s_perturb_config(b2s_sim* s, const b2s_perturb* spec, int n) {
  if (!s || n < 0 || (n > 0 && !spec)) return fail(B2S_ERR_ARG, "b2s_perturb_config: bad argument");
  std::vector<PerturbEntry> ent;
  std::vector<PerturbItem> item;
  for (int i = 0; i < n; i++) {
    const b2s_perturb& p = spec[i];
    const std::string f = p.field ? p.field : "";
    const std::string at = "b2s_perturb_config: entry " + std::to_string(i) + " ('" + f + "'): ";
    if (!(p.mode == B2S_PERTURB_SCALE || p.mode == B2S_PERTURB_SHIFT)) return fail(B2S_ERR_ARG, at + "mode must be scale or shift");
    if (!(p.amplitude >= 0) || !std::isfinite(p.amplitude)) return fail(B2S_ERR_ARG, at + "the amplitude must be finite and >= 0");
    if (p.mode == B2S_PERTURB_SCALE && p.amplitude >= 1) return fail(B2S_ERR_ARG, at + "a scale amplitude must be below 1");
    const bool dof = is_dof_field(f);
    if (!dof && !is_geom_field(f) && !is_body_field(f)) return fail(B2S_ERR_ARG, at + "unknown field");
    if (dof && (p.id < -1 || p.id >= s->nv)) return fail(B2S_ERR_ARG, at + "dof id out of range");
    auto it = s->arrays.find(override_key(f, p.id));
    if (it == s->arrays.end()) return fail(B2S_ERR_ARG, at + "the field is not declared (b2s_model_override)");
    const size_t rsz = real_size(s);
    PerturbEntry e{};
    e.mode = p.mode; e.one_draw = p.one_draw != 0; e.amp = p.amplitude;
    const double* model;
    int ncomp;
    if (dof) {  // id -1: every dof; a dof index: that component of the vector alone
      const std::vector<double>& h = f == "dof_damping" ? s->dof_damping_h : f == "dof_armature" ? s->dof_armature_h : s->dof_frictionloss_h;
      const int first = p.id < 0 ? 0 : p.id;
      e.stride = s->nv;
      e.dst = (char*)it->second.ptr + first * rsz;
      model = h.data() + first;
      ncomp = p.id < 0 ? s->nv : 1;
    } else {
      const int w = it->second.ndim == 1 ? 1 : (int)it->second.shape[1];
      const std::vector<double>& h = f == "geom_size" ? s->geom_size_h : f == "geom_friction" ? s->geom_friction_h : f == "geom_solref" ? s->geom_solref_h
                                   : f == "geom_solimp" ? s->geom_solimp_h : f == "body_mass" ? s->body_mass_h : s->body_inertia_h;
      e.stride = w;
      e.dst = it->second.ptr;
      model = h.data() + (size_t)w * p.id;
      ncomp = w;
    }
    for (int c = 0; c < ncomp; c++) item.push_back(PerturbItem{(int)ent.size(), c, model[c]});
    ent.push_back(e);
  }
  CUDA_TRY(cudaSetDevice(s->device));
  try {  // replaced tables stay allocated until the handle is destroyed (configuration is a set-up step)
    s->pert_ent = ent.empty() ? nullptr : dev_upload(s, ent);
    s->pert_item = item.empty() ? nullptr : dev_upload(s, item);
  } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
  s->pert_nitems = (int)item.size();
  return B2S_OK;
}

int b2s_perturb_model(b2s_sim* s, const uint8_t* env_mask, uint64_t seed, uint64_t counter) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  if (counter >> 32) return fail(B2S_ERR_ARG, "b2s_perturb_model: the counter must be below 2^32");
  if (s->pert_nitems == 0) return B2S_OK;
  CUDA_TRY(cudaSetDevice(s->device));
  const long long total = (long long)s->n_env * s->pert_nitems;
  const int threads = 256;
  const unsigned blocks = (unsigned)((total + threads - 1) / threads);
  with_real(s, [&](auto& m, auto&) {
    using R = real_of<decltype(m)>;
    perturb_kernel<R><<<blocks, threads, 0, s->stream>>>(s->pert_ent, s->pert_item, s->pert_nitems, s->n_env, env_mask, seed, (unsigned)counter);
  });
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

int b2s_body_pose_override(b2s_sim* s, int body_id) {
  if (!s || body_id <= 0 || body_id >= s->nbody) return fail(B2S_ERR_ARG, "b2s_body_pose_override: bad argument");
  if (s->body_weldid_h[body_id] != 0) return fail(B2S_ERR_UNSUPPORTED, "b2s_body_pose_override: the body is not welded to the world (move it through qpos)");
  CUDA_TRY(cudaSetDevice(s->device));
  return with_real(s, [&](auto&, auto& st) { return body_pose_override_t(s, st, body_id); });
}

int b2s_env_step(b2s_sim* s, const void* action, int nsub) {
  if (!s || !s->has_ctrl || !action || nsub < 1) return fail(B2S_ERR_ARG, "b2s_env_step: bad argument / controller not configured");
  if (s->mode == 2 && !s->export_env_step)
    return launch_unit(s, PH_STEP1 | PH_STEP2 | PH_CTRL | (s->has_obs ? PH_OBS : 0), nsub, action);
  if (s->mode == 1 && !s->export_env_step)
    return launch_pipeline(s, PH_STEP1 | PH_STEP2 | PH_CTRL | (s->has_obs ? PH_OBS : 0), nsub, action);
  return launch(s, PH_STEP1 | PH_STEP2 | PH_CTRL | (s->has_obs ? PH_OBS : 0) | (s->export_env_step ? PH_EXPORT : 0), nsub, action);
}

int b2s_obs_config(b2s_sim* s, int obs_dim, const int* op, const int* a, const int* b) {
  if (!s || obs_dim <= 0 || !op || !a || !b) return fail(B2S_ERR_ARG, "b2s_obs_config: bad argument");
  CUDA_TRY(cudaSetDevice(s->device));
  try {
    std::vector<int> vo(op, op + obs_dim), va(a, a + obs_dim), vb(b, b + obs_dim);
    s->ctrl.obs_dim = obs_dim;
    s->obs_tab_h = vo; s->obs_tab_h.insert(s->obs_tab_h.end(), va.begin(), va.end()); s->obs_tab_h.insert(s->obs_tab_h.end(), vb.begin(), vb.end());
    s->ctrl.obs_op = dev_upload(s, vo); s->ctrl.obs_a = dev_upload(s, va); s->ctrl.obs_b = dev_upload(s, vb);
    if (obs_dim > 128) throw std::string("obs_dim > 128 not supported");
    int* fresh = state_arr_i(s, "obs_fresh", 0);
    {
      std::vector<int> ones(s->n_env, 1);
      if (cudaMemcpy(fresh, ones.data(), sizeof(int) * s->n_env, cudaMemcpyHostToDevice) != cudaSuccess) throw std::string("obs_fresh upload failed");
      cudaStreamSynchronize(cudaStreamLegacy);
    }
    with_real(s, [&](auto& m, auto& st) {
      using R = real_of<decltype(m)>;
      st.obs = state_arr<R>(s, "obs", obs_dim); st.task_out = state_arr<R>(s, "task_out", 8); st.obs_fresh = fresh;
    });
  } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
  with_real(s, [](auto&, auto& st) { st.obs_mod = nullptr; });  // the rows of a previous table no longer exist
  if (s->obs_mod_on) s->obs_mod_on = 0;
  s->has_obs = 1;
  s->dirty = 1;
  s->layout_version++;
  return B2S_OK;
}

int b2s_obs_modifiers(b2s_sim* s, int nobs, const int* row_obs, const b2s_obs_mod* mods, uint64_t seed) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  if (!s->has_obs) return fail(B2S_ERR_ARG, "b2s_obs_modifiers: observations are not configured (b2s_obs_config)");
  if (nobs < 0 || nobs > B2S_MAXOBS) return fail(B2S_ERR_ARG, "b2s_obs_modifiers: nobs must be in [0, 32]");
  if (nobs > 0 && (!row_obs || !mods)) return fail(B2S_ERR_ARG, "b2s_obs_modifiers: bad argument");
  const int od = s->ctrl.obs_dim;
  ObsModDev h{};
  h.nobs = nobs; h.seed = seed; h.dt = s->timestep_h;
  for (int o = 0; o < nobs; o++) {
    const b2s_obs_mod& q = mods[o];
    const std::string at = "b2s_obs_modifiers: observable " + std::to_string(o) + ": ";
    if (!(q.period > 0) || !std::isfinite(q.period)) return fail(B2S_ERR_ARG, at + "the period must be finite and > 0");
    if (q.corruptor != B2S_CORRUPT_NONE && q.corruptor != B2S_CORRUPT_GAUSSIAN && q.corruptor != B2S_CORRUPT_UNIFORM)
      return fail(B2S_ERR_ARG, at + "unknown corruptor");
    if (q.corruptor != B2S_CORRUPT_NONE) {
      if (!std::isfinite(q.p0) || !std::isfinite(q.p1)) return fail(B2S_ERR_ARG, at + "noise parameters must be finite");
      if (q.corruptor == B2S_CORRUPT_GAUSSIAN && q.p1 < 0) return fail(B2S_ERR_ARG, at + "std < 0");
      if (q.corruptor == B2S_CORRUPT_UNIFORM && q.p1 < q.p0) return fail(B2S_ERR_ARG, at + "max_noise < min_noise");
      if (!(q.low <= q.high)) return fail(B2S_ERR_ARG, at + "low > high");
    }
    h.period[o] = q.period; h.kind[o] = q.corruptor; h.p0[o] = q.p0; h.p1[o] = q.p1; h.lo[o] = q.low; h.hi[o] = q.high;
  }
  for (int k = 0; k < od && nobs > 0; k++) {
    if (row_obs[k] < 0 || row_obs[k] >= nobs)
      return fail(B2S_ERR_ARG, "b2s_obs_modifiers: row " + std::to_string(k) + " is mapped to observable " + std::to_string(row_obs[k]) + ", out of range");
    h.row_obs[k] = row_obs[k];
  }
  CUDA_TRY(cudaSetDevice(s->device));
  const ObsModDev* dev = nullptr;
  if (nobs > 0) {
    try {
      if (!s->obs_mod_dev) s->obs_mod_dev = dev_zeros<ObsModDev>(s, 1);
      if (s->obs_arr_n != nobs) {  // replaced arrays stay allocated until the handle is destroyed
        s->arrays.erase("obs_timer"); s->arrays.erase("obs_sampled"); s->arrays.erase("obs_nsample");
        state_arr<double>(s, "obs_timer", nobs);
        state_arr_i(s, "obs_sampled", 0);
        state_arr_i(s, "obs_nsample", nobs);
        s->obs_arr_n = nobs;
        s->obs_mod_on = 0;
      }
    } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
    h.timer = (double*)s->arrays["obs_timer"].ptr; h.sampled = (int*)s->arrays["obs_sampled"].ptr; h.nsample = (int*)s->arrays["obs_nsample"].ptr;
    if (!s->obs_mod_on) {  // the state of the default rule at a control-step boundary; the sample counts are kept
      std::vector<double> t((size_t)s->n_env * nobs, s->timestep_h);
      std::vector<int> f(s->n_env, (int)(nobs == 32 ? 0xffffffffu : (1u << nobs) - 1u));
      CUDA_TRY(cudaMemcpyAsync(h.timer, t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice, s->stream));
      CUDA_TRY(cudaMemcpyAsync(h.sampled, f.data(), f.size() * sizeof(int), cudaMemcpyHostToDevice, s->stream));
      CUDA_TRY(cudaStreamSynchronize(s->stream));  // pageable sources
    }
    // stream-ordered behind the kernels that read the previous table
    CUDA_TRY(cudaMemcpyAsync(s->obs_mod_dev, &h, sizeof(h), cudaMemcpyHostToDevice, s->stream));
    CUDA_TRY(cudaStreamSynchronize(s->stream));
    dev = s->obs_mod_dev;
  }
  with_real(s, [&](auto&, auto& st) { st.obs_mod = dev; });
  if ((nobs > 0) != (s->obs_mod_on != 0)) s->layout_version++;  // the snapshot sections change
  s->obs_mod_on = nobs > 0;
  s->dirty = 1;
  return B2S_OK;
}

int b2s_task_config2(b2s_sim* s, int body2, const int* obj2, int no2) {
  if (!s || body2 >= s->nbody) return fail(B2S_ERR_ARG, "b2s_task_config2: bad argument");
  unsigned long long mk = 0;
  for (int i = 0; i < no2; i++) {
    if (obj2[i] < 0 || obj2[i] >= s->ngeom) return fail(B2S_ERR_ARG, "b2s_task_config2: geom id out of range");
    int k = s->cgid[obj2[i]];
    if (k >= 0) mk |= 1ull << k;
  }
  s->ctrl.task_body2 = body2; s->ctrl.mask_obj2 = mk; s->dirty = 1;
  return B2S_OK;
}

int b2s_task_table(b2s_sim* s, int n, const int* op, const int* a, const int* b) {
  if (!s || n <= 0 || n > 64 || !op || !a || !b) return fail(B2S_ERR_ARG, "b2s_task_table: bad argument");
  CUDA_TRY(cudaSetDevice(s->device));
  try {
    std::vector<int> vo(op, op + n), va(a, a + n), vb(b, b + n);
    s->ctrl.task_dim = n;
    s->task_tab_h = vo; s->task_tab_h.insert(s->task_tab_h.end(), va.begin(), va.end()); s->task_tab_h.insert(s->task_tab_h.end(), vb.begin(), vb.end());
    s->ctrl.task_op = dev_upload(s, vo); s->ctrl.task_a = dev_upload(s, va); s->ctrl.task_b = dev_upload(s, vb);
    with_real(s, [&](auto& m, auto& st) { st.task_vec = state_arr<real_of<decltype(m)>>(s, "task_vec", n); });
  } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
  s->dirty = 1;
  s->layout_version++;
  return B2S_OK;
}

int b2s_task_objects(b2s_sim* s, int nobjects, const int* geoms, const int* counts) {
  if (!s || nobjects < 0 || nobjects > 4 || (nobjects > 0 && (!geoms || !counts))) return fail(B2S_ERR_ARG, "b2s_task_objects: bad argument");
  int o = 0;
  for (int i = 0; i < 4; i++) s->ctrl.mask_objs[i] = 0;
  for (int i = 0; i < nobjects; i++)
    for (int k = 0; k < counts[i]; k++, o++) {
      if (geoms[o] < 0 || geoms[o] >= s->ngeom) return fail(B2S_ERR_ARG, "b2s_task_objects: geom id out of range");
      int cg = s->cgid[geoms[o]];
      if (cg >= 0) s->ctrl.mask_objs[i] |= 1ull << cg;
    }
  s->ctrl.n_objs = nobjects; s->dirty = 1;
  return B2S_OK;
}

int b2s_task_config(b2s_sim* s, int body, int site, const int* left, int nl, const int* right, int nr, const int* obj, int no) {
  if (!s || body < 0 || body >= s->nbody || site < 0 || site >= s->nsite) return fail(B2S_ERR_ARG, "b2s_task_config: bad argument");
  auto mk = [&](const int* g, int n, unsigned long long& out) {
    out = 0;
    for (int i = 0; i < n; i++) {
      if (g[i] < 0 || g[i] >= s->ngeom) return false;
      int k = s->cgid[g[i]];
      if (k >= 0) out |= 1ull << k;
    }
    return true;
  };
  if (!mk(left, nl, s->ctrl.mask_left) || !mk(right, nr, s->ctrl.mask_right) || !mk(obj, no, s->ctrl.mask_obj))
    return fail(B2S_ERR_ARG, "b2s_task_config: geom id out of range");
  s->ctrl.task_body = body; s->ctrl.task_site = site;
  if (s->ctrl.mask_obj2 == 0) s->ctrl.task_body2 = -1;
  s->dirty = 1;
  return B2S_OK;
}

}  // extern "C"

// ---- whole-environment snapshots.  The row is the handle's per-environment arrays in a fixed section order, each section 16-byte
// aligned; the table (and the signature) is rebuilt when an entry point changed what it covers (layout_version).
static int ensure_snap(b2s_sim* s) {
  if (s->snap_dev && s->snap_version == s->layout_version) return B2S_OK;
  std::vector<SnapSecHost> v;
  int64_t off = 0;
  auto add = [&](const std::string& name, const void* p, int64_t count, int dtype) {
    v.push_back(SnapSecHost{name, off, count, dtype, const_cast<void*>(p)});
    const int64_t es = (dtype == B2S_F64 || dtype == B2S_I64) ? 8 : 4;
    off += (count * es + 15) & ~(int64_t)15;
  };
  with_real(s, [&](auto& m, auto& st) {
    const int R = DT<real_of<decltype(m)>>::code;
    const size_t N = s->n_env;
    add("qpos", st.qpos, m.nq, R); add("qvel", st.qvel, m.nv, R); add("qacc", st.qacc, m.nv, R);
    add("qacc_warmstart", st.qacc_ws, m.nv, R); add("ctrl", st.ctrl, m.nu, R); add("time", st.time, 1, R);
    add("warn", st.warn, 1, B2S_I32);
    add("ctrl_goal_pos", st.goal_pos, 3, R); add("ctrl_goal_ori", st.goal_ori, 9, R); add("ctrl_initial_joint", st.init_qpos_arm, 8, R);
    add("ctrl_grip_state", st.grip_state, 4, R); add("ctrl_jv_state", st.jv_state, 72, R); add("ctrl_torque", st.ctrl_torque, 8, R);
    add("gjk_cache", st.gjk_cache, (int64_t)m.npair * 3, R);  // null until the pipeline's first use, or with B2S_NO_GJK_CACHE
    if (s->has_obs) { add("obs", st.obs, s->ctrl.obs_dim, R); add("obs_fresh", st.obs_fresh, 1, B2S_I32); add("task_out", st.task_out, 8, R); }
    if (s->obs_mod_on) {
      add("obs_timer", s->arrays["obs_timer"].ptr, s->obs_arr_n, B2S_F64); add("obs_sampled", s->arrays["obs_sampled"].ptr, 1, B2S_I32);
      add("obs_nsample", s->arrays["obs_nsample"].ptr, s->obs_arr_n, B2S_I32);
    }
    if (st.task_vec) add("task_vec", st.task_vec, s->ctrl.task_dim, R);
    for (int k = 0; k < st.n_ov; k++) {
      const std::string id = std::to_string(st.ov_body[k]);
      add("body_xpos_ov:" + id, st.ov_pos[k], 3, R); add("body_xquat_ov:" + id, st.ov_quat[k], 4, R);
    }
    for (int k = 0; k < st.n_mg; k++) {  // a geom slot carries all six values, whichever field declared it
      const std::string id = std::to_string(st.mg_id[k]);
      add("geom_size:" + id, st.mg_size + k * N * 3, 3, R); add("geom_friction:" + id, st.mg_fric + k * N * 3, 3, R);
      add("geom_rbound:" + id, st.mg_rbound + k * N, 1, R); add("geom_aabb:" + id, st.mg_aabb + k * N * 6, 6, R);
      add("geom_solref:" + id, st.mg_solref + k * N * 2, 2, R); add("geom_solimp:" + id, st.mg_solimp + k * N * 5, 5, R);
    }
    for (int k = 0; k < st.n_mb; k++) {
      const std::string id = std::to_string(st.mb_id[k]);
      add("body_mass:" + id, st.mb_mass + k * N, 1, R); add("body_inertia:" + id, st.mb_inertia + k * N * 3, 3, R);
    }
    if (st.dof_damp) add("dof_damping", st.dof_damp, m.nv, R);
    if (st.dof_arm) add("dof_armature", st.dof_arm, m.nv, R);
    if (st.dof_floss) add("dof_frictionloss", st.dof_floss, m.nv, R);
    if (st.dof_iw) {  // copied, not recomputed: a snapshot taken while they were stale restores them stale
      add("dof_invweight0", st.dof_iw, m.nv, R); add("body_invweight0", st.body_iw, 2 * (int64_t)m.nbody, R);
      add("meaninertia", st.mean_inertia, 1, R);
    }
  });
  if (v.size() > SNAP_MAXSEC) return fail(B2S_ERR_UNSUPPORTED, "snapshot: too many sections");
  std::vector<SnapSec> dev(v.size());
  uint64_t h = FNV_BASIS;
  for (size_t k = 0; k < v.size(); k++) {
    const SnapSecHost& x = v[k];
    const int64_t bytes = x.count * ((x.dtype == B2S_F64 || x.dtype == B2S_I64) ? 8 : 4);
    const int64_t next = k + 1 < v.size() ? v[k + 1].off : off;
    dev[k] = SnapSec{(char*)x.ptr, (long long)bytes, (int)(x.off / 4), (int)(bytes / 4), (int)((next - x.off) / 4),
                     ((uintptr_t)x.ptr % 16 == 0 && bytes % 16 == 0) ? 1 : 0};
    h = fnv1a(h, x.name.c_str(), x.name.size() + 1);
    h = fnv1a(h, &x.count, sizeof(x.count));
    h = fnv1a(h, &x.dtype, sizeof(x.dtype));
  }
  h = fnv1a(h, &s->precision, sizeof(int));
  h = fnv1a(h, &s->ctrl.kind, sizeof(int));
  const int no = (int)s->obs_tab_h.size(), nt = (int)s->task_tab_h.size();
  h = fnv1a(h, &no, sizeof(int)); h = fnv1a(h, s->obs_tab_h.data(), sizeof(int) * no);
  h = fnv1a(h, &nt, sizeof(int)); h = fnv1a(h, s->task_tab_h.data(), sizeof(int) * nt);
  h = fnv1a(h, &s->blob_hash, sizeof(uint64_t));
  CUDA_TRY(cudaSetDevice(s->device));
  if (!s->snap_dev) {
    try { s->snap_dev = dev_zeros<SnapSec>(s, SNAP_MAXSEC); } catch (const std::string& e) { return fail(B2S_ERR_CUDA, e); }
  }
  // stream-ordered behind every earlier snapshot / restore of this handle that read the old table
  if (!dev.empty()) CUDA_TRY(cudaMemcpyAsync(s->snap_dev, dev.data(), dev.size() * sizeof(SnapSec), cudaMemcpyHostToDevice, s->stream));
  s->snap = v;
  s->snap_row_bytes = (size_t)off;
  s->snap_sig = h;
  s->snap_version = s->layout_version;
  return B2S_OK;
}

extern "C" {

int b2s_snapshot_info(b2s_sim* s, size_t* row_bytes, uint64_t* signature, int* nsections) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  int rc = ensure_snap(s);
  if (rc != B2S_OK) return rc;
  if (row_bytes) *row_bytes = s->snap_row_bytes;
  if (signature) *signature = s->snap_sig;
  if (nsections) *nsections = (int)s->snap.size();
  return B2S_OK;
}

int b2s_snapshot_section(b2s_sim* s, int k, const char** name, int64_t* offset_bytes, int64_t* count, int* dtype) {
  if (!s) return fail(B2S_ERR_ARG, "null handle");
  int rc = ensure_snap(s);
  if (rc != B2S_OK) return rc;
  if (k < 0 || k >= (int)s->snap.size()) return fail(B2S_ERR_ARG, "b2s_snapshot_section: section index out of range");
  const SnapSecHost& x = s->snap[k];
  if (name) *name = x.name.c_str();
  if (offset_bytes) *offset_bytes = x.off;
  if (count) *count = x.count;
  if (dtype) *dtype = x.dtype;
  return B2S_OK;
}

int b2s_snapshot(b2s_sim* s, void* rows, const int* env_index, int n_rows) {
  if (!s || n_rows < 0 || (n_rows > 0 && !rows)) return fail(B2S_ERR_ARG, "b2s_snapshot: bad argument");
  if (!env_index && n_rows != s->n_env) return fail(B2S_ERR_ARG, "b2s_snapshot: without an index list n_rows must equal n_env");
  if (env_index)
    for (int r = 0; r < n_rows; r++)
      if (env_index[r] < 0 || env_index[r] >= s->n_env)
        return fail(B2S_ERR_ARG, "b2s_snapshot: environment index " + std::to_string(env_index[r]) + " out of range [0, " + std::to_string(s->n_env) + ")");
  CUDA_TRY(cudaSetDevice(s->device));
  int rc = ensure_snap(s);
  if (rc != B2S_OK) return rc;
  if (n_rows == 0) return B2S_OK;
  const int nsec = (int)s->snap.size(), row_words = (int)(s->snap_row_bytes / 4);
  if (!env_index) {
    snapshot_kernel<<<(n_rows + 7) / 8, 256, 0, s->stream>>>(s->snap_dev, nsec, row_words, (unsigned char*)rows, n_rows);
    s->launches++;
  } else {
    for (int first = 0; first < n_rows; first += SNAP_IDX) {
      const int n = std::min(SNAP_IDX, n_rows - first);
      SnapIdx ix;
      memcpy(ix.idx, env_index + first, sizeof(int) * n);
      snapshot_list_kernel<<<(n + 7) / 8, 256, 0, s->stream>>>(s->snap_dev, nsec, row_words, (unsigned char*)rows, first, n, ix);
      s->launches++;
    }
  }
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

int b2s_restore(b2s_sim* s, const void* rows, int n_rows, const int* src_row) {
  if (!s || n_rows < 0 || (n_rows > 0 && !rows)) return fail(B2S_ERR_ARG, "b2s_restore: bad argument");
  if (!src_row && n_rows != s->n_env) return fail(B2S_ERR_ARG, "b2s_restore: without a source-row map n_rows must equal n_env");
  CUDA_TRY(cudaSetDevice(s->device));
  if (s->mode != 0) {  // the pipeline / unit queue would create a zero GJK cache at their first step: create it now, so it is restored
    int rc0 = with_real(s, [&](auto& m, auto& st) { return ensure_ws(s, m, st); });
    if (rc0 != B2S_OK) return rc0;
  }
  int rc = ensure_snap(s);
  if (rc != B2S_OK) return rc;
  int* warn = with_real(s, [](auto&, auto& st) { return st.warn; });
  restore_kernel<<<(s->n_env + 7) / 8, 256, 0, s->stream>>>(s->snap_dev, (int)s->snap.size(), (int)(s->snap_row_bytes / 4),
                                                             (const unsigned char*)rows, n_rows, src_row, s->n_env, warn);
  s->launches++;
  CUDA_TRY(cudaGetLastError());
  return B2S_OK;
}

}  // extern "C"
