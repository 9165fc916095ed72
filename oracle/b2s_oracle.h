/* TEST INFRASTRUCTURE - CPU oracle (fp64, single environment, scalar C99).
 *
 * Restatement of the per-step path the reference reaches through `robosuite/utils/binding_utils.py:1101-1107`
 * (MjSim.step1 / step2 -> third-party engine `mujoco>=3.3,<3.10`, setup.py:21) plus the controller arithmetic of
 * `robosuite/controllers/parts/arm/osc.py:403-495`.  The engine's source is NOT under /root/reference and the
 * wheel is not installable here: the physics half of this oracle follows the engine's published computation
 * pipeline and is checked only against analytic known-answer tests  ==> "parity unpinned" for physics.
 * The controller half IS pinned against the reference's own Python (tests/golden/osc_*.npz).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this library.
 */
#ifndef B2S_ORACLE_H
#define B2S_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { O_JNT_FREE = 0, O_JNT_BALL = 1, O_JNT_SLIDE = 2, O_JNT_HINGE = 3 };
enum { O_GEOM_PLANE = 0, O_GEOM_HFIELD, O_GEOM_SPHERE, O_GEOM_CAPSULE, O_GEOM_ELLIPSOID, O_GEOM_CYLINDER,
       O_GEOM_BOX, O_GEOM_MESH };
enum { O_CNSTR_FRICTION_DOF = 1, O_CNSTR_LIMIT_JOINT = 3, O_CNSTR_CONTACT_FRICTIONLESS = 5,
       O_CNSTR_CONTACT_ELLIPTIC = 7 };
enum { O_STATE_SATISFIED = 0, O_STATE_QUADRATIC, O_STATE_LINEARNEG, O_STATE_LINEARPOS, O_STATE_CONE };

#define O_MAXCON 128
#define O_MAXEFC 512
#define O_MINVAL 1e-15

typedef struct {
  void* blob; /* owned copy of the packed model */
  /* sizes */
  int nq, nv, nu, nbody, njnt, ngeom, nsite, nmesh, nM, npair, nmocap, nsensordata, nmeshvert;
  /* options */
  double timestep, impratio, density, viscosity, tolerance, ls_tolerance, meaninertia;
  int iterations, ls_iterations, cone;
  const double* gravity; const double* wind;
  /* bodies */
  const int *body_parentid, *body_rootid, *body_weldid, *body_mocapid, *body_jntnum, *body_jntadr, *body_dofnum,
      *body_dofadr, *body_geomnum, *body_geomadr;
  const double *body_pos, *body_quat, *body_ipos, *body_iquat, *body_mass, *body_subtreemass, *body_inertia,
      *body_invweight0;
  /* joints / dofs */
  const int *jnt_type, *jnt_qposadr, *jnt_dofadr, *jnt_bodyid, *jnt_limited;
  const double *jnt_pos, *jnt_axis, *jnt_range, *jnt_margin, *jnt_solref, *jnt_solimp, *jnt_stiffness;
  const int *dof_bodyid, *dof_jntid, *dof_parentid, *dof_Madr;
  const double *dof_armature, *dof_damping, *dof_frictionloss, *dof_solref, *dof_solimp, *dof_invweight0, *dof_M0;
  const double *qpos0, *qpos_spring;
  /* geoms */
  const int *geom_type, *geom_contype, *geom_conaffinity, *geom_condim, *geom_bodyid, *geom_dataid, *geom_priority;
  const double *geom_size, *geom_pos, *geom_quat, *geom_friction, *geom_solmix, *geom_solref, *geom_solimp,
      *geom_margin, *geom_gap, *geom_rbound, *geom_aabb;
  const int* pair_geom;
  /* meshes (convex hull vertices) */
  const int *mesh_vertadr, *mesh_vertnum;
  const double* mesh_vert;
  /* sites */
  const int* site_bodyid;
  const double *site_pos, *site_quat;
  /* actuators */
  const int *actuator_trnid, *actuator_ctrllimited, *actuator_forcelimited, *actuator_biastype;
  const double *actuator_ctrlrange, *actuator_forcerange, *actuator_gear, *actuator_gainprm, *actuator_biasprm;
} OModel;

typedef struct {
  double dist;
  double pos[3];
  double frame[9]; /* rows: normal (geom1 -> geom2), tangent1, tangent2 */
  double friction[5];
  double solref[2];
  double solimp[5];
  double mu;
  int dim;
  int geom1, geom2;
  int efc_address;
} OContact;

typedef struct {
  double time;
  double *qpos, *qvel, *qacc, *qacc_warmstart, *ctrl, *qfrc_applied, *mocap_pos, *mocap_quat;
  /* position stage */
  double *xpos, *xquat, *xmat, *xipos, *ximat, *xanchor, *xaxis, *geom_xpos, *geom_xmat, *site_xpos, *site_xmat;
  double* cdof;  /* nv x 6: [angular; linear-at-world-origin] spatial motion axis of each dof, world frame */
  double* cinert; /* nbody x 10: I_O(6: xx,yy,zz,xy,xz,yz), h=m*c (3), m */
  double* crb;   /* nbody x 10 composite */
  double* qM;    /* sparse, nM */
  double* M;     /* dense nv x nv (own use) */
  double* L;     /* Cholesky factor of M (lower, dense) */
  /* velocity stage */
  double *cvel, *cdof_dot; /* nbody x 6, nv x 6 */
  double *qfrc_bias, *qfrc_passive, *qfrc_actuator, *actuator_force, *qfrc_smooth, *qacc_smooth, *qfrc_constraint;
  double* sensordata;
  /* collision + constraints */
  int ncon;
  OContact contact[O_MAXCON];
  int nefc, nf, nl; /* rows: nf friction-loss, nl limits, then contacts */
  int efc_type[O_MAXEFC], efc_id[O_MAXEFC], efc_state[O_MAXEFC];
  double* efc_J; /* O_MAXEFC x nv */
  double efc_pos[O_MAXEFC], efc_margin[O_MAXEFC], efc_diagApprox[O_MAXEFC], efc_D[O_MAXEFC], efc_R[O_MAXEFC],
      efc_aref[O_MAXEFC], efc_vel[O_MAXEFC], efc_frictionloss[O_MAXEFC], efc_force[O_MAXEFC], efc_KBIP[4 * O_MAXEFC];
  int solver_niter;
  int warn_flags;
} OData;

/* model / data lifecycle */
OModel* o_model_load(const void* blob, size_t nbytes);
void o_model_free(OModel* m);
OData* o_data_new(const OModel* m);
void o_data_free(OData* d);
double* o_data_field(OData* d, const char* name); /* named access for the Python side */

/* pipeline (names follow the engine calls at binding_utils.py:1091-1107) */
void o_reset_data(const OModel* m, OData* d);
void o_forward(const OModel* m, OData* d);
void o_step1(const OModel* m, OData* d);
void o_step2(const OModel* m, OData* d);
void o_step(const OModel* m, OData* d);

/* stages (exposed for tests) */
void o_model_set_body_pose(OModel* m, int body, const double* pos, const double* quat);
void o_kinematics(const OModel* m, OData* d);
void o_crb(const OModel* m, OData* d);
void o_factor_m(const OModel* m, OData* d);
void o_collision(const OModel* m, OData* d);
void o_make_constraint(const OModel* m, OData* d);
void o_com_vel(const OModel* m, OData* d);
void o_passive(const OModel* m, OData* d);
void o_rne_bias(const OModel* m, OData* d);
void o_fwd_actuation(const OModel* m, OData* d);
void o_fwd_acceleration(const OModel* m, OData* d);
void o_fwd_constraint(const OModel* m, OData* d);
void o_euler(const OModel* m, OData* d);

/* support (binding_utils.py:681-851 mj_jac*, controllers/parts/controller.py:227 mj_fullM) */
void o_jac(const OModel* m, const OData* d, double* jacp, double* jacr, const double point[3], int body);
void o_full_m(const OModel* m, const OData* d, double* dst);
void o_solve_m(const OModel* m, const OData* d, double* x, int n); /* x <- M^-1 x, n right-hand sides (row vectors) */

/* narrow-phase entry point (tests call it pairwise): returns number of contacts written */
int o_collide_pair(const OModel* m, const OData* d, int g1, int g2, OContact* out, int maxout);

#ifdef __cplusplus
}
#endif
#endif
