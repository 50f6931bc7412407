/* bik.h -- C ABI of libbik: batched differential inverse kinematics on H100 (sm_90a).
 *
 * mink has no FFI layer of its own (SURVEY.md 8b): its hot path is reached through the Python
 * classes Configuration / Task / Limit and solve_ik().  This header is what a replacement of that
 * path binds to: every entry point below names the reference function(s) it replaces.  Plain
 * pointers and sizes only; no torch / numpy / C++ types.
 *
 * Conventions
 *   - every function returns BIK_OK (0) or a negative bik_status; text via bik_last_error().
 *   - `const float* q` etc. are DEVICE pointers unless a parameter is documented "host".
 *   - descriptors (bik_task_desc, bik_limit_desc, bik_frame, model blob) are HOST memory and are
 *     copied at create time; the caller keeps ownership of everything it passes in.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls enqueue
 *     work and return; nothing synchronises unless stated.
 *   - batch layout is row-major with the instance index outermost: q[B][nq], J[B][K][nv], ...
 *   - quaternions are (w,x,y,z); poses are (qw,qx,qy,qz,x,y,z) like mink.SE3.wxyz_xyz
 *     (reference mink/lie/se3.py:24-29); twists are (v, omega) (ibid.).
 *   - model handles are immutable after creation and may be shared between streams.  A problem handle owns the K1 -> K2
 *     hand-off buffers of bik_step / bik_converge: calls on one problem handle are ordered (a call on another stream than
 *     the previous one first waits, on the device, for that call's kernels); use one problem handle per stream for overlap.
 */
#ifndef BIK_H
#define BIK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BIK_VERSION 200

typedef enum bik_status {
  BIK_OK = 0,
  BIK_ERR_INVALID = -1,     /* bad argument / malformed blob or descriptor */
  BIK_ERR_CUDA = -2,        /* CUDA runtime error (message has the cudaError string) */
  BIK_ERR_UNSUPPORTED = -3, /* model or problem outside the supported subset */
  BIK_ERR_NOMEM = -4
} bik_status;

/* Per-instance status bits written by the solve/step/check entry points.  Inside a batch these
 * replace the reference's exceptions (NotWithinConfigurationLimits, configuration.py:97-105;
 * `assert dq is not None`, solve_ik.py:103). */
#define BIK_STATUS_OUT_OF_LIMITS 1u  /* q outside [range - tol, range + tol] */
#define BIK_STATUS_QP_MAXITER    2u  /* active-set iteration cap reached, or more general rows in play than the solver holds
                                         (24 active at once, 64 inside the detection distance); dq is the last iterate */
#define BIK_STATUS_NONFINITE     4u  /* NaN/Inf met in q, targets or the factorisation */
#define BIK_STATUS_QP_INFEASIBLE 8u  /* inequality set inconsistent (lower > upper for a dof, or no feasible start): the
                                      * reference's solver returns None there and solve_ik asserts (solve_ik.py:103) */
#define BIK_STATUS_NOT_CONVERGED 16u /* bik_converge: thresholds not met within max_iters */
#define BIK_STATUS_BAD_WEIGHT    32u /* ..._weighted[_ex] entry points: a task or posture weight of the instance is outside [0, 1] or NaN; it was
                                      * clamped to [0, 1] (NaN to 0) and the step went on with the clamped value */

typedef struct bik_model bik_model;     /* flattened kinematic tree resident on one device */
typedef struct bik_problem bik_problem; /* static task + limit layout bound to a model */

/* A frame rigidly attached to a tree node (node = -1: fixed in the world).  The front end
 * resolves (name, "body"|"geom"|"site") to this once, instead of the per-call mj_name2id of
 * reference configuration.py:133,170. */
typedef struct bik_frame {
  int32_t node;
  int32_t reserved;
  double pos[3];
  double quat[4];
} bik_frame;

enum { BIK_TASK_FRAME = 0, BIK_TASK_POSTURE = 1, BIK_TASK_COM = 2, BIK_TASK_RELATIVE_FRAME = 3 };

/* One kinematic task (reference mink/tasks/task.py:54-79 holds cost/gain/lm_damping).
 *   FRAME   : FrameTask   (frame_task.py:28-45)   rows = 6, cost = position xyz | orientation xyz
 *   POSTURE : PostureTask (posture_task.py:27-50) rows = nv (never materialised as a Jacobian:
 *             J = -I with free-joint dofs zeroed, posture_task.py:137-141); dof_cost[nv] host array.
 *             DampingTask (damping_task.py:19-20) = POSTURE with gain 0 and target qpos0.
 *   COM     : ComTask     (com_task.py:25-33)     rows = 3, cost[0..2]
 *   RELATIVE_FRAME : RelativeFrameTask (relative_frame_task.py:24-45) rows = 6; pose of `frame` expressed
 *             in `root`; its target (one slot of frame_targets, in task order) is T_root<-target. */
typedef struct bik_task_desc {
  int32_t kind;
  int32_t reserved;
  bik_frame frame;
  double cost[6];
  const double* dof_cost;
  double gain;
  double lm_damping;
  bik_frame root; /* RELATIVE_FRAME only */
} bik_task_desc;

enum { BIK_LIMIT_CONFIGURATION = 0, BIK_LIMIT_VELOCITY = 1, BIK_LIMIT_COLLISION = 2 };
enum { BIK_GEOM_PLANE = 0, BIK_GEOM_SPHERE = 2, BIK_GEOM_CAPSULE = 3, BIK_GEOM_BOX = 6 };   /* mjtGeom codes */

typedef struct bik_geom {
  int32_t type;
  int32_t reserved;
  bik_frame frame;
  double size[3];
} bik_geom;

/* One inequality limit  G(q) dq <= h(q)  (reference mink/limits/limit.py:11-57).
 *   CONFIGURATION (configuration_limit.py:69-124): for each listed dof i (slide/hinge):
 *        -gain*(q_i - lower_i) <= dq_i <= gain*(upper_i - q_i);  lower/upper already include
 *        min_distance_from_limits (configuration_limit.py:50-51).
 *   VELOCITY      (velocity_limit.py:71-101):      |dq_i| <= dt * vmax_i.
 *   COLLISION     (collision_avoidance_limit.py:187-210): one row per geom pair,
 *        -n^T (Jp2 - Jp1) dq <= gain*(dist - minimum_distance)/dt + bound_relaxation, rows whose
 *        distance is >= detection_distance are inactive.  Primitive pairs only (plane, sphere,
 *        capsule, box; no plane-plane and no box-box pair). */
typedef struct bik_limit_desc {
  int32_t kind;
  int32_t n;             /* CONFIGURATION/VELOCITY: number of listed dofs; COLLISION: number of pairs */
  const int32_t* dof;    /* [n] tangent-space indices */
  const double* lower;   /* [n] CONFIGURATION */
  const double* upper;   /* [n] CONFIGURATION */
  const double* vmax;    /* [n] VELOCITY */
  double gain;
  const bik_geom* geoms; /* COLLISION */
  int32_t ngeoms;
  int32_t reserved;
  const int32_t* pairs;  /* [n][2] indices into geoms */
  double minimum_distance;
  double detection_distance;
  double bound_relaxation;
} bik_limit_desc;

/* Per-call inputs of the task layer (device pointers).  Targets are what FrameTask.set_target /
 * PostureTask.set_target / ComTask.set_target store (frame_task.py:83, posture_task.py:77,
 * com_task.py:61), one per instance. */
typedef struct bik_inputs {
  const void* q;               /* [B][nq] */
  const void* frame_targets;   /* [B][F][7]  F = number of FRAME + RELATIVE_FRAME tasks, in task-list order */
  const void* posture_targets; /* layout by posture_batched (below)  P = number of POSTURE tasks */
  const void* com_targets;     /* [B][C][3]  C = number of COM tasks */
  int32_t posture_batched;     /* layout of posture_targets, one of BIK_POSTURE_* */
  int32_t f64;                 /* element type of the four buffers: 0 float (fp32 entry points), 1 double (the ...64 ones) */
} bik_inputs;

/* bik_inputs.posture_batched.  The two sequence forms are accepted by bik_track, bik_track64, bik_track_weighted and
 * bik_track_weighted64 only: instance b on frame t uses row t of BIK_POSTURE_SEQ_SHARED and row b*T + t of
 * BIK_POSTURE_SEQ_BATCHED.  Every other entry point rejects them with BIK_ERR_INVALID. */
#define BIK_POSTURE_SHARED      0  /* [P][nq]: one target shared by the batch */
#define BIK_POSTURE_BATCHED     1  /* [B][P][nq]: one target per instance (any other value outside 2..3 is read as 1) */
#define BIK_POSTURE_SEQ_SHARED  2  /* [T][P][nq]: one target per frame, shared by the batch */
#define BIK_POSTURE_SEQ_BATCHED 3  /* [B][T][P][nq]: one target per instance and frame */

typedef struct bik_dims {
  int32_t nq, nv, nnode;
  int32_t nframe, nposture, ncom; /* F, P, C */
  int32_t nrows;                  /* K = 6F + 3C : rows of the stacked J / e */
  int32_t npairs;                 /* collision rows */
} bik_dims;

int bik_version(void);
const char* bik_last_error(void);

/* Model = what mink reads out of MjModel during mj_kinematics/mj_jac (configuration.py:63-64,145).
 * `blob` is the BIKM v1 buffer produced by mink_b200.flatten.FlatModel.to_blob(). */
int bik_model_create(const void* blob, size_t nbytes, int device, bik_model** out);
void bik_model_destroy(bik_model* model);

int bik_problem_create(const bik_model* model, const bik_task_desc* tasks, int ntasks,
                       const bik_limit_desc* limits, int nlimits, bik_problem** out);
void bik_problem_destroy(bik_problem* problem);
int bik_problem_dims(const bik_problem* problem, bik_dims* out);

/* Forward kinematics of arbitrary frames.
 * Replaces Configuration.update + get_transform_frame_to_world (configuration.py:53-64,157-185)
 * and data.subtree_com[1] (com_task.py:69).  poses [B][nframes][7]; com [B][3] or NULL.
 * `frames` is a HOST array. */
int bik_fk(const bik_model* model, int B, const float* q, const bik_frame* frames, int nframes,
           float* poses, float* com, void* stream);

/* Body-frame Jacobians of arbitrary frames: Configuration.get_frame_jacobian
 * (configuration.py:112-155).  J [B][nframes][6][nv], rows = (linear xyz, angular xyz). */
int bik_frame_jacobian(const bik_model* model, int B, const float* q, const bik_frame* frames,
                       int nframes, float* J, void* stream);

/* K1: FK + task errors + task Jacobians for every task of the problem.
 * Replaces Task.compute_error / Task.compute_jacobian of FrameTask (frame_task.py:95-146),
 * ComTask (com_task.py:71-97) and PostureTask.compute_error (posture_task.py:87-118).
 *   J         [B][K][nv]   stacked rows in task order (FRAME 6 rows, COM 3 rows)
 *   e         [B][K]
 *   e_posture [B][P][nv]   (NULL allowed when P = 0)
 *   G_coll    [B][npairs][nv], h_coll [B][npairs]  collision rows (NULL allowed when npairs = 0);
 *             inactive rows are zero with h = +inf (collision_avoidance_limit.py:192-199) */
int bik_fk_jac(const bik_problem* problem, int B, const bik_inputs* in, float dt, float* J, float* e,
               float* e_posture, float* G_coll, float* h_coll, void* stream);

/* QP objective  H = damping*I + sum_t H_t,  c = sum_t c_t  with
 * H_t = (W J)^T (W J) + mu I, c_t = -(W(-gain e))^T (W J), mu = lm_damping ||W(-gain e)||^2.
 * Replaces Task.compute_qp_objective (task.py:105-138) + _compute_qp_objective (solve_ik.py:13-22).
 *   H [B][nv][nv], c [B][nv]  (fp64) */
int bik_qp_objective(const bik_problem* problem, int B, const float* J, const float* e,
                     const float* e_posture, double damping, double* H, double* c, void* stream);

/* Box form of the configuration + velocity limits:  lo <= dq <= hi  per dof ([B][nv], +-inf where
 * unbounded).  Replaces ConfigurationLimit / VelocityLimit.compute_qp_inequalities
 * (configuration_limit.py:98-124, velocity_limit.py:99-101); G is the constant +-projection. */
int bik_limits_box(const bik_problem* problem, int B, const float* q, float dt, float* lo, float* hi,
                   void* stream);

/* K2: assemble the QP from (J, e) and solve it exactly (active set on a warp-per-problem Cholesky).
 * Replaces build_ik + qpsolvers.solve_problem (solve_ik.py:43-65,101).  dq [B][nv] is the
 * displacement BEFORE the division by dt of solve_ik.py:104.  status [B] (may be NULL). */
int bik_solve(const bik_problem* problem, int B, const float* q, const float* J, const float* e,
              const float* e_posture, const float* G_coll, const float* h_coll, float dt,
              double damping, float* dq, int32_t* status, void* stream);

/* bik_solve plus diagnostics: iters [B] (may be NULL) receives the number of active-set iterations. */
int bik_solve_ex(const bik_problem* problem, int B, const float* q, const float* J, const float* e,
                 const float* e_posture, const float* G_coll, const float* h_coll, float dt,
                 double damping, float* dq, int32_t* status, int32_t* iters, void* stream);

/* q <- q (+) dq : Configuration.integrate / integrate_inplace (configuration.py:214-236). */
int bik_integrate(const bik_model* model, int B, float* q, const float* dq, void* stream);

/* Configuration.check_limits (configuration.py:77-110): sets BIK_STATUS_OUT_OF_LIMITS per instance. */
int bik_check_limits(const bik_model* model, int B, const float* q, float tol, int32_t* status,
                     void* stream);

/* The whole solve_ik step (solve_ik.py:68-105) `nsteps` times, two launches per step:
 *   K1 (check_limits + FK + task rows, packed: only the non-zero Jacobian columns) -> K2 (QP + integrate if `integrate` != 0).
 * `in->q` is ignored; q [B][nq] is read and, when integrating, updated in place.
 * dq [B][nv] receives the last step's displacement. */
int bik_step(const bik_problem* problem, int B, float* q, const bik_inputs* in, float dt,
             double damping, int nsteps, int integrate, float* dq, int32_t* status, void* stream);

/* Same step with HOST buffers: copies q/targets to the device, runs bik_step, copies dq (and q when
 * integrating) back, and synchronises.  This is the entry point a host-only caller (the reference's
 * numpy world) binds to; h2d/d2h byte counts are returned for measurement. */
int bik_step_host(const bik_problem* problem, int B, float* q_host, const bik_inputs* in_host,
                  float dt, double damping, int nsteps, int integrate, float* dq_host,
                  int32_t* status_host, size_t* h2d_bytes, size_t* d2h_bytes);

/* Converge-until-threshold driver: the solve_ik + integrate inner loop of the reference's examples
 * (examples/quadruped_spot.py:89-104, examples/arm_aloha.py:146-169), per instance:
 *     for i in range(max_iters):  v = solve_ik(...); q = integrate(q, v, dt)
 *                                 if all frame tasks: |e[:3]| <= pos_threshold and |e[3:]| <= ori_threshold: break
 * q [B][nq] is updated in place; an instance that met the thresholds keeps its configuration while the
 * others go on.  iters [B] receives the number of steps each instance took (1..max_iters); instances
 * that never met the thresholds get BIK_STATUS_NOT_CONVERGED.  The batch loop stops as soon as no
 * instance is left (the device counter is read back every `check_every` steps).  Device buffers. */
int bik_converge(const bik_problem* problem, int B, float* q, const bik_inputs* in, float dt,
                 double damping, int max_iters, float pos_threshold, float ori_threshold,
                 int check_every, int32_t* iters, int32_t* status, void* stream);

/* The examples' outer loop (examples/arm_aloha.py:140-169): for each frame t of a target sequence, the bik_converge loop.
 * Each instance moves to its next frame as soon as it is done with the current one; for every instance b the results are
 * those of bik_converge called on frames 0..lengths[b]-1 in turn.  fp32 device buffers, as bik_converge (bik_track64: fp64).
 *   in->frame_targets [B][T][F][7], in->com_targets [B][T][C][3]; in->posture_targets as for bik_converge (the same for every
 *   frame), or a sequence: [T][P][nq] with posture_batched = BIK_POSTURE_SEQ_SHARED, [B][T][P][nq] with
 *   BIK_POSTURE_SEQ_BATCHED (frame t's row then stands where bik_converge's target stands on frame t)
 *   lengths [B] frames per instance, each in 0..T (NULL: all T); q [B][nq] in: start, out: end of each instance's last frame
 *   q_traj [B][T][nq], iters [B][T], status [B][T] (NULL allowed): per frame, as bik_converge returns them; rows past
 *   lengths[b] untouched
 *   passes: device int, number of passes the loop ran, max_b sum_t (iters[b][t] + 1) (NULL allowed)
 * BIK_CONVERGE_GRAPH=0 runs the host-polled loop: the device counter is read back every `check_every` passes. */
int bik_track(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const int32_t* lengths,
              float dt, double damping, int max_iters, float pos_threshold, float ori_threshold, int check_every,
              float* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream);

/* ---- fp64 entry points --------------------------------------------------------------------------------------------
 * The reference is fp64 end to end (numpy; mink/solve_ik.py:13-22).  These mirror the fp32 entry points above with
 * double buffers (bik_inputs.f64 = 1): the fp64 instantiations of the kernels run, on the kinematic constants at full
 * precision, and reproduce the reference to solver tolerance (~1e-8 rad) also where cost / sqrt(damping) would amplify
 * fp32 rounding past 1e-4 rad (BASELINE config 5).  A single (numpy, B = 1) Configuration of the Python front end
 * always takes them.  The fp32 entry points pick the fp64 K1 by themselves for ill-conditioned problems
 * (bik_problem_describe says which; BIK_K1_PRECISION=f32|f64 overrides). */
int bik_fk64(const bik_model* model, int B, const double* q, const bik_frame* frames, int nframes,
             double* poses, double* com, void* stream);
int bik_frame_jacobian64(const bik_model* model, int B, const double* q, const bik_frame* frames,
                         int nframes, double* J, void* stream);
int bik_fk_jac64(const bik_problem* problem, int B, const bik_inputs* in, double dt, double* J, double* e,
                 double* e_posture, double* G_coll, double* h_coll, void* stream);
int bik_qp_objective64(const bik_problem* problem, int B, const double* J, const double* e,
                       const double* e_posture, double damping, double* H, double* c, void* stream);
int bik_limits_box64(const bik_problem* problem, int B, const double* q, double dt, double* lo, double* hi,
                     void* stream);
int bik_solve64(const bik_problem* problem, int B, const double* q, const double* J, const double* e,
                const double* e_posture, const double* G_coll, const double* h_coll, double dt,
                double damping, double* dq, int32_t* status, int32_t* iters, void* stream);
int bik_integrate64(const bik_model* model, int B, double* q, const double* dq, void* stream);
int bik_check_limits64(const bik_model* model, int B, const double* q, double tol, int32_t* status,
                       void* stream);
int bik_step64(const bik_problem* problem, int B, double* q, const bik_inputs* in, double dt,
               double damping, int nsteps, int integrate, double* dq, int32_t* status, void* stream);
/* bik_converge and bik_track on fp64 buffers (q, q_traj and the targets are double; in->f64 = 1 is required): the same
 * loops, the same arguments and results, with the fp64 K1 and the thresholds compared in double as the reference compares
 * them.  The fp32 bik_converge / bik_track reject fp64 inputs, and these reject fp32 ones. */
int bik_converge64(const bik_problem* problem, int B, double* q, const bik_inputs* in, double dt, double damping,
                   int max_iters, double pos_threshold, double ori_threshold, int check_every,
                   int32_t* iters, int32_t* status, void* stream);
int bik_track64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const int32_t* lengths,
                double dt, double damping, int max_iters, double pos_threshold, double ori_threshold, int check_every,
                double* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream);

/* ---- per-instance task weights -----------------------------------------------------------------------------------------
 * The entry points above with one more argument, `weights`, right after `in`: each instance scales the costs of its own frame
 * and CoM task rows, as mink's FrameTask.set_position_cost / set_orientation_cost / ComTask.set_cost would between two
 * solve_ik calls, without building another problem.
 *   weights [B][K] (K = bik_dims.nrows; bik_track: [B][T][K], row t is used while the instance is on frame t), device memory,
 *           float or double like the other inputs (bik_inputs.f64).  Rows in the stacked order of J: per FRAME /
 *           RELATIVE_FRAME task position xyz then orientation xyz, per COM task xyz, in task order.  NULL: all ones, the
 *           results of the unweighted entry point.
 *   The cost of row r of instance b is cost_r * w[b][r]: it scales the row of J and e in H, c and the Levenberg-Marquardt
 *   term mu = lm_damping ||W(-gain e)||^2 exactly as a cost does.  A weight outside [0, 1] is clamped to [0, 1], NaN to 0,
 *   and the instance gets BIK_STATUS_BAD_WEIGHT.  PostureTask / DampingTask rows have no weights.
 *   The convergence test of bik_converge / bik_track compares the unweighted errors with the thresholds, except that a frame
 *   task whose three position weights are all 0 in an instance has its position error left out of that instance's test
 *   (orientation likewise): a fully occluded target does not hold the instance for max_iters steps. */
int bik_step_weighted(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, float dt,
                      double damping, int nsteps, int integrate, float* dq, int32_t* status, void* stream);
int bik_converge_weighted(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, float dt,
                          double damping, int max_iters, float pos_threshold, float ori_threshold, int check_every,
                          int32_t* iters, int32_t* status, void* stream);
int bik_track_weighted(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const void* weights,
                       const int32_t* lengths, float dt, double damping, int max_iters, float pos_threshold,
                       float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status, int32_t* passes,
                       void* stream);
int bik_step_weighted64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, double dt,
                        double damping, int nsteps, int integrate, double* dq, int32_t* status, void* stream);
int bik_converge_weighted64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, double dt,
                            double damping, int max_iters, double pos_threshold, double ori_threshold, int check_every,
                            int32_t* iters, int32_t* status, void* stream);
int bik_track_weighted64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const void* weights,
                         const int32_t* lengths, double dt, double damping, int max_iters, double pos_threshold,
                         double ori_threshold, int check_every, double* q_traj, int32_t* iters, int32_t* status,
                         int32_t* passes, void* stream);

/* ---- per-instance posture weights --------------------------------------------------------------------------------------
 * The ..._weighted entry points with one more argument, `posture_weights`, right after `weights`: each instance also scales
 * the per-dof costs of its own PostureTask and DampingTask, as mink's PostureTask.set_cost would between two solve_ik calls.
 * A weight of 0 on every dof of a DampingTask drops that task for the instance: one problem serves a batch in which some
 * instances have the task and others do not.
 *   posture_weights [B][P][nv] (P = bik_dims.nposture, posture-type tasks in task order as in posture_targets;
 *           bik_track_weighted_ex: [B][T][P][nv], row b*T + t is used while instance b is on frame t), device memory, float or
 *           double like the other inputs (bik_inputs.f64).  NULL: exactly what the ..._weighted entry point runs, bit for bit.
 *           Non-NULL on a problem without posture-type tasks: BIK_ERR_INVALID.
 *   `weights` as in the ..._weighted entry points, NULL for all ones.
 *   The cost of posture task p on dof d of instance b is cost[p][d] * w[b][p][d]: it scales the task's diagonal, its part of
 *   the linear term and its Levenberg-Marquardt term exactly as a cost does.  A weight of exactly 1 gives the unweighted
 *   arithmetic bit for bit.  Free-joint dofs have no posture rows, so their weights do nothing.  A weight outside [0, 1] is
 *   clamped to [0, 1], NaN to 0, and the instance (in bik_track: the frame in progress) gets BIK_STATUS_BAD_WEIGHT.  The
 *   convergence test does not change: it looks at frame errors only.
 *   Precision of K1 for fp32 callers: posture costs regularise the QP, and the automatic choice of K1's precision counts on
 *   them.  With posture_weights set it assumes every posture weight may be 0, i.e. it takes the damping alone as the
 *   regularisation, so a problem that runs K1 in fp32 without posture weights may run it in fp64 with them. */
int bik_step_weighted_ex(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights,
                         const void* posture_weights, float dt, double damping, int nsteps, int integrate, float* dq,
                         int32_t* status, void* stream);
int bik_converge_weighted_ex(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights,
                             const void* posture_weights, float dt, double damping, int max_iters, float pos_threshold,
                             float ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_weighted_ex(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const void* weights,
                          const void* posture_weights, const int32_t* lengths, float dt, double damping, int max_iters,
                          float pos_threshold, float ori_threshold, int check_every, float* q_traj, int32_t* iters,
                          int32_t* status, int32_t* passes, void* stream);
int bik_step_weighted_ex64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights,
                           const void* posture_weights, double dt, double damping, int nsteps, int integrate, double* dq,
                           int32_t* status, void* stream);
int bik_converge_weighted_ex64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights,
                               const void* posture_weights, double dt, double damping, int max_iters, double pos_threshold,
                               double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_weighted_ex64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const void* weights,
                            const void* posture_weights, const int32_t* lengths, double dt, double damping, int max_iters,
                            double pos_threshold, double ori_threshold, int check_every, double* q_traj, int32_t* iters,
                            int32_t* status, int32_t* passes, void* stream);

/* ---- per-instance joint limits ------------------------------------------------------------------------------------------
 * The ..._weighted_ex entry points with one more argument, `bounds`, right after `posture_weights`: each instance narrows the
 * problem's ConfigurationLimit bounds and VelocityLimit caps with its own, as mink's ConfigurationLimit.lower / upper and
 * VelocityLimit.limit would be changed between two solve_ik calls.  A cap of 0 (or lower == upper == q) locks a dof of one
 * instance exactly, e.g. the base of a mobile robot on the instances where it must stay put.
 *   bounds  host memory; its members are device buffers [B][nv] (tangent dofs; bik_track_bounded: one row per instance, used on
 *           every frame), float or double like the other inputs (bik_inputs.f64), each NULL for no narrowing.  A NULL `bounds`,
 *           or one whose three members are NULL, runs exactly what the ..._weighted_ex entry point runs, bit for bit.
 *           `lower` / `upper` on a problem without a ConfigurationLimit, `vmax` on one without a VelocityLimit: BIK_ERR_INVALID.
 *   `weights` and `posture_weights` as in the ..._weighted_ex entry points, each NULL for none.
 *   Narrowing only.  For instance b and dof d, every ConfigurationLimit that lists d (gives it a finite bound) gets the bounds
 *   max(lower_c, lower[b][d]) and min(upper_c, upper[b][d]) and keeps its gain; the VelocityLimit's cap of a dof it lists (a
 *   finite cap) becomes min(vmax_d, vmax[b][d]).  The values of the other dofs are not read.  So the set of bounded dofs is
 *   the problem's, and so are the leading unbounded dofs the solver eliminates once: to widen a bound per instance, build the
 *   problem with the widest bounds and narrow them.  Instance b solves the QP of a problem built with its narrowed bounds; the
 *   problem stores bounds in fp32, so where the values are exactly representable in fp32 the results are that problem's bit
 *   for bit (dq, q, iterations, status), otherwise they are used in the caller's precision.  -inf / +inf narrow nothing.  A NaN
 *   narrows nothing and sets BIK_STATUS_NONFINITE on the instance (bik_track: on the frame in progress).  Narrowing to
 *   lower > upper, or a negative cap, sets BIK_STATUS_QP_INFEASIBLE, as that problem would.
 *   BIK_STATUS_OUT_OF_LIMITS and bik_check_limits still test the model's joint range (Configuration.check_limits), and
 *   bik_limits_box / bik_step_host have no bounded form. */
typedef struct bik_bounds {
  const void* lower;   /* [B][nv] or NULL: narrows the ConfigurationLimit bounds of the dofs they list */
  const void* upper;   /* [B][nv] or NULL */
  const void* vmax;    /* [B][nv] or NULL: narrows the VelocityLimit caps of the dofs it lists */
} bik_bounds;          /* element type follows bik_inputs.f64 */
int bik_step_bounded(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                     const bik_bounds* bounds, float dt, double damping, int nsteps, int integrate, float* dq, int32_t* status, void* stream);
int bik_converge_bounded(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                         const bik_bounds* bounds, float dt, double damping, int max_iters, float pos_threshold, float ori_threshold,
                         int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_bounded(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                      const bik_bounds* bounds, const int32_t* lengths, float dt, double damping, int max_iters, float pos_threshold,
                      float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream);
int bik_step_bounded64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                       const bik_bounds* bounds, double dt, double damping, int nsteps, int integrate, double* dq, int32_t* status,
                       void* stream);
int bik_converge_bounded64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                           const bik_bounds* bounds, double dt, double damping, int max_iters, double pos_threshold, double ori_threshold,
                           int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_bounded64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const void* weights,
                        const void* posture_weights, const bik_bounds* bounds, const int32_t* lengths, double dt, double damping,
                        int max_iters, double pos_threshold, double ori_threshold, int check_every, double* q_traj, int32_t* iters,
                        int32_t* status, int32_t* passes, void* stream);

/* ---- per-instance collision avoidance ------------------------------------------------------------------------------------
 * The ..._bounded entry points with one more argument, `coll`, right after `bounds`: each instance enables its own subset of
 * the CollisionAvoidanceLimit's geom pairs and sets its own distances, as a mink user would build the limit with the pairs
 * that matter now, or change minimum_distance_from_collisions / collision_detection_distance, between two solve_ik calls.
 * With every candidate obstacle in the model, a pair mask gives each instance its own set of obstacles.
 *   coll    host memory; its members are device buffers, each NULL for the problem's own: `enabled` [B][npairs] bytes
 *           (bik_track_coll: [B][T][npairs]), `minimum_distance` and `detection_distance` [B] (bik_track_coll: [B][T]), float
 *           or double like the other inputs (bik_inputs.f64).  bik_track_coll uses row b*T + t while instance b is on frame t.
 *           A NULL `coll`, or one whose three members are NULL, runs exactly what the ..._bounded entry point runs, through
 *           the same kernels, bit for bit.  A non-NULL member on a problem without a CollisionAvoidanceLimit: BIK_ERR_INVALID.
 *   `weights`, `posture_weights` and `bounds` as in the ..._bounded entry points, each NULL for none.
 *   Pair k of instance b is used iff enabled[b][k] != 0.  A disabled pair hands the QP what a pair beyond the detection
 *   distance hands it (no constraint row), and its distance is never computed.  An instance with at least one enabled pair
 *   gives, bit for bit, what a problem built with its enabled pairs (in the same order) and its distances gives: dq, q,
 *   iterations and status.  One exception: the solver's iteration cap (60 + 2 (nv + min(npairs, 24))) counts the problem's
 *   pairs, so an instance with fewer than 24 enabled pairs may iterate longer before BIK_STATUS_QP_MAXITER than that
 *   problem would.  An instance with no enabled pair solves the QP without collision rows; it agrees with a problem built
 *   without the limit to solver tolerance, not bit for bit (that problem may take fp32 kernels and another QP path).
 *   The distances are used in the caller's precision where K1 runs in fp64, which it does for every problem with a
 *   CollisionAvoidanceLimit unless BIK_K1_PRECISION=f32 is set.  A non-finite distance falls back to the problem's value and
 *   sets BIK_STATUS_NONFINITE on the instance (bik_track_coll: on the frame in progress); no other value is refused.
 *   The limit's gain and bound_relaxation stay the problem's, and bik_fk_jac, bik_solve, bik_limits_box and bik_step_host
 *   have no collision form. */
typedef struct bik_collision {
  const uint8_t* enabled;          /* [B][npairs] (bik_track_coll: [B][T][npairs]) or NULL: pair k of instance b is used iff != 0 */
  const void* minimum_distance;    /* [B] (track: [B][T]) or NULL: replaces minimum_distance_from_collisions */
  const void* detection_distance;  /* [B] (track: [B][T]) or NULL: replaces collision_detection_distance */
} bik_collision;                   /* distances: float or double like the other inputs (bik_inputs.f64) */
int bik_step_coll(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                  const bik_bounds* bounds, const bik_collision* coll, float dt, double damping, int nsteps, int integrate, float* dq,
                  int32_t* status, void* stream);
int bik_converge_coll(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                      const bik_bounds* bounds, const bik_collision* coll, float dt, double damping, int max_iters, float pos_threshold,
                      float ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_coll(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                   const bik_bounds* bounds, const bik_collision* coll, const int32_t* lengths, float dt, double damping, int max_iters,
                   float pos_threshold, float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status,
                   int32_t* passes, void* stream);
int bik_step_coll64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                    const bik_bounds* bounds, const bik_collision* coll, double dt, double damping, int nsteps, int integrate, double* dq,
                    int32_t* status, void* stream);
int bik_converge_coll64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                        const bik_bounds* bounds, const bik_collision* coll, double dt, double damping, int max_iters, double pos_threshold,
                        double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_coll64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const void* weights,
                     const void* posture_weights, const bik_bounds* bounds, const bik_collision* coll, const int32_t* lengths, double dt,
                     double damping, int max_iters, double pos_threshold, double ori_threshold, int check_every, double* q_traj,
                     int32_t* iters, int32_t* status, int32_t* passes, void* stream);

/* ---- held targets in bik_track ------------------------------------------------------------------------------------------
 * bik_track_coll with one more argument, `hold`, right after `coll`: a task can hold the value it had at the configuration
 * the solver reached, for a run of frames, as a mink loop that calls task.set_target_from_configuration(configuration) before
 * the first frame of the run does.  Contact locking is the typical use: a foot that touches down on frame t0 keeps the pose
 * the robot's foot had when frame t0 began, for as long as the contact lasts.
 *   hold    device, [B][T][H] bytes or NULL, H = F + C + P: the F frame-like tasks (FRAME and RELATIVE_FRAME) in the order of
 *           frame_targets, then the C CoM tasks in the order of com_targets, then the P posture-type tasks in the order of
 *           posture_targets.  A NULL `hold` runs exactly what bik_track_coll runs, through the same kernels, bit for bit.
 *   `weights`, `posture_weights`, `bounds`, `coll` and `lengths` as in bik_track_coll.
 *   A run of task k for instance b is a maximal set of consecutive frames t0..t1 with hold[b][t][k] != 0.  On the first pass
 *   of frame t0, before that pass's errors are computed, the task's value at the instance's configuration (q_traj[b][t0-1],
 *   or the start q for t0 = 0) is captured: a FRAME task's world pose as bik_fk reports it, a RELATIVE_FRAME task's pose in
 *   its root (root^-1 * frame), a CoM task's CoM, a posture-type task's q.  It is stored in the caller's precision
 *   (bik_inputs.f64), as a target the caller passed would be, and is the task's target on every frame of the run in place of
 *   its row of frame_targets / com_targets / posture_targets; it is not captured again within the run.  Frames outside runs
 *   read their targets as bik_track_coll does.  So each instance gives what T bik_converge_coll calls give when the caller
 *   sets each held task's target with set_target_from_configuration before the first frame of each of its runs.  The
 *   convergence test takes a held frame task's error against the held target, and weights apply to held tasks unchanged.
 *   A hold on a posture-type task with gain 0 (a DampingTask) changes nothing.  An all-zero mask gives what bik_track_coll
 *   gives: q_traj, iters, status and passes. */
int bik_track_hold(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                   const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold, const int32_t* lengths, float dt, double damping,
                   int max_iters, float pos_threshold, float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status,
                   int32_t* passes, void* stream);
int bik_track_hold64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const void* weights,
                     const void* posture_weights, const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold,
                     const int32_t* lengths, double dt, double damping, int max_iters, double pos_threshold, double ori_threshold,
                     int check_every, double* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream);

/* ---- per-instance frame placement --------------------------------------------------------------------------------------
 * bik_step_coll / bik_converge_coll with one more argument, `placement`, right after `coll`, and bik_track_hold with it right
 * after `hold`: each instance puts each frame task's frame at its own pose on the task's tree node, as a mink user who moves
 * model.site_pos / site_quat (geom_pos / geom_quat) between solves does.  Marker retargeting (one marker placement per
 * performer), tool or TCP offsets, and fingertip contact points are the typical uses.
 *   placement  device, [B][F][7] in the inputs' precision (bik_inputs.f64), F = number of FRAME + RELATIVE_FRAME tasks in the
 *              order of frame_targets.  Row b*F + f is wxyz xyz, laid out as frame_targets: the pose of task f's frame in its
 *              tree node, what bik_task_desc.frame.quat / pos would be.  bik_track_placed uses row b*F + f on every frame.
 *              A NULL `placement` runs exactly what bik_step_coll / bik_converge_coll / bik_track_hold run, through the same
 *              kernels, bit for bit.  Non-NULL on a problem without frame-like tasks is BIK_ERR_INVALID.
 *   `weights`, `posture_weights`, `bounds`, `coll`, `hold` and `lengths` as in those entry points.
 *   Instance b runs what a problem built with frame poses row b runs.  The node stays the problem's (a placement moves a frame
 *   on its body, never onto another body), and a RELATIVE_FRAME task's root keeps the problem's placement.  A row that holds
 *   exactly what the problem image would hold for that pose (the builder divides the quaternion by its norm in double, then
 *   stores both in K1's precision) gives that problem's dq, q, iters, status and passes bit for bit; a quaternion that is not
 *   of unit length is used as given, not renormalised.  The convergence test takes the placed frames' errors; a held FRAME
 *   task captures the world pose of its placed frame, a held RELATIVE_FRAME task that frame's pose in its root.
 *   A row with a non-finite element keeps the problem's placement for that task and instance and sets BIK_STATUS_NONFINITE on
 *   the instance (bik_track_placed: on every frame the instance runs).
 *   bik_fk_jac, bik_solve, bik_limits_box and bik_step_host have no placed form. */
int bik_step_placed(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                    const bik_bounds* bounds, const bik_collision* coll, const void* placement, float dt, double damping, int nsteps,
                    int integrate, float* dq, int32_t* status, void* stream);
int bik_step_placed64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                      const bik_bounds* bounds, const bik_collision* coll, const void* placement, double dt, double damping, int nsteps,
                      int integrate, double* dq, int32_t* status, void* stream);
int bik_converge_placed(const bik_problem* problem, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                        const bik_bounds* bounds, const bik_collision* coll, const void* placement, float dt, double damping, int max_iters,
                        float pos_threshold, float ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_converge_placed64(const bik_problem* problem, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                          const bik_bounds* bounds, const bik_collision* coll, const void* placement, double dt, double damping, int max_iters,
                          double pos_threshold, double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream);
int bik_track_placed(const bik_problem* problem, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                     const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold, const void* placement, const int32_t* lengths,
                     float dt, double damping, int max_iters, float pos_threshold, float ori_threshold, int check_every, float* q_traj,
                     int32_t* iters, int32_t* status, int32_t* passes, void* stream);
int bik_track_placed64(const bik_problem* problem, int B, int T, double* q, const bik_inputs* in, const void* weights,
                       const void* posture_weights, const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold,
                       const void* placement, const int32_t* lengths, double dt, double damping, int max_iters, double pos_threshold,
                       double ori_threshold, int check_every, double* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream);

/* Measurement aid for the K2 roofline (bench.py): sustained fused-multiply-add throughput of the CUDA cores of `device`
 * in TFLOP/s (fp32 or fp64; 16 independent chains per thread, every SM filled), best of `repeats` event-timed launches. */
int bik_measure_fma_peak(int device, int use_double, int repeats, double* tflops);

/* Bytes of device scratch a problem needs for a batch of B (K1's packed task rows, collision rows, ... between K1 and K2). */
size_t bik_workspace_bytes(const bik_problem* problem, int B);

/* One-line description of how a problem is mapped onto the device (lanes per instance and visited
 * nodes in K1, coupled block size, K2 path and precision chosen for `damping`), for logs and
 * benchmark labels.  Writes at most cap bytes including the terminator; returns the full length. */
int bik_problem_describe(const bik_problem* problem, double damping, char* buf, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* BIK_H */
