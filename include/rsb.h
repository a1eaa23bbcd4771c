/* rsb.h -- C-ABI of the H100-native batched rigid-body step ("raisim batch").
 *
 * This is the drop-in boundary for the hot path raisim::World::integrate() =
 * integrate1() + integrate2() and the ArticulatedSystem state/force/PD accessors around it
 * (SURVEY.md section 8b).  The reference exposes that path as C++ classes, not a plugin ABI, and the
 * reference snapshot holds none of the headers (/root/reference/.SUBMODULES.json:2 records
 * "bytes": 0; the only consumer build recorded is /root/reference/.travis.yml:11,
 * -DRAISIM_EXAMPLE=ON).  Each entry point below therefore cites the upstream *symbol* it replaces
 * ([RECALL] in SURVEY.md: include/raisim/World.hpp, object/ArticulatedSystem/ArticulatedSystem.hpp,
 * contact/Contact.hpp); the header-only facade in include/raisim/ forwards those symbols here.
 *
 * Rules: plain C, opaque handles, int status (0 = OK, negative = error, text via rsb_last_error()),
 * no exceptions across the boundary, all buffers caller-owned.  One handle <-> one host thread.
 * All batched arrays are float32; `where` says whether a caller buffer is host or device memory.
 * `where`, `where_in` and `where_out` are RSB_HOST or RSB_DEVICE: any other value is refused with
 * RSB_ERR_INVALID before anything is enqueued.  Pageable host rows pass through a device staging
 * buffer of the batch that grows to the largest such transfer and is kept until the batch is destroyed.
 * Device work is enqueued on the batch's stream (rsb_batch_set_stream) and is asynchronous unless a
 * host buffer is read back.
 */
#ifndef RSB_H_
#define RSB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RSB_OK 0
#define RSB_ERR_INVALID (-1)
#define RSB_ERR_PARSE (-2)
#define RSB_ERR_CUDA (-3)
#define RSB_ERR_UNSUPPORTED (-4)

#define RSB_HOST 0
#define RSB_DEVICE 1

#define RSB_KMAX 8 /* contacts kept per environment (the deepest RSB_KMAX candidates) */
#define RSB_LMAX 4 /* joint-limit constraints kept per environment (the first RSB_LMAX violated joints) */

/* ArticulatedSystem::ControlMode */
#define RSB_FORCE_AND_TORQUE 0
#define RSB_PD_PLUS_FEEDFORWARD_TORQUE 1

typedef struct rsb_model rsb_model; /* immutable robot description (URDF -> tables) */
typedef struct rsb_batch rsb_batch; /* N environments of one model on one GPU        */

/* World::setTimeStep, setGravity, setERP, setContactSolverParam, setDefaultMaterial.
 * rsb_batch_set_params refuses (RSB_ERR_INVALID, naming the field; the batch keeps its parameters) a non-finite value in any float
 * field, dt <= 0, max_iter < 1, mu < 0, accel_m other than 0 or 2, accel_start < 3 with accel_m = 2, and stall_reg < 0. */
typedef struct rsb_params {
  float dt;          /* World::setTimeStep                               (default 0.0025) */
  float gravity[3];  /* World::setGravity                                (0,0,-9.81)      */
  float erp;         /* World::setERP                                    (0)              */
  float alpha_init;  /* World::setContactSolverParam(alpha_init, ...)    (1)              */
  float alpha_min;   /*                                                  (1)              */
  float alpha_decay; /*                                                  (1)              */
  int max_iter;      /*                                                  (150)            */
  float threshold;   /*                                                  (1e-6, float32)  */
  float mu;          /* World::setDefaultMaterial friction               (0.8)            */
  float restitution; /* World::setDefaultMaterial restitution            (0)              */
  float rest_threshold; /* restitution threshold velocity               (0.01)           */
  /* Stagnation exit of the Gauss-Seidel loop (NOT in the reference; stall_window = 0 restores the
   * plain maxIter behaviour): every stall_window iterations, stop if the largest impulse update has
   * not dropped below stall_ratio x its value one window earlier (then see stall_reg below).  A safety
   * net for the contact sets on which the published per-contact rule enters a limit cycle (~1 % of the
   * problems of fallen robots even with the accelerated sweeps; none of standing ones); DESIGN.md 5. */
  int stall_window;     /*                                               (8)              */
  float stall_ratio;    /*                                               (0.5)            */
  int joint_limits;     /* enforce URDF <limit lower upper> as unilateral rows of the same solve (1) */
  /* Anderson acceleration of the Gauss-Seidel sweep map (NOT in the reference; accel_m = 0 restores the plain sweeps of the
   * published method): from sweep accel_start on, the next iterate is extrapolated from the last accel_m + 1 sweep
   * outputs g_k and residuals f_k = g_k - x_k (least squares over the residual differences; history dropped when the
   * residual doubles).  Same fixed point; redundant contact sets (box feet, knee + foot on one shank) converge in a
   * third of the sweeps and quickly converging problems never reach accel_start.  DESIGN.md section 5. */
  int accel_m;          /* 0 = off, 2 = on                               (2)              */
  int accel_start;      /* first extrapolation after this sweep          (6)              */
  /* What the FIRST failed stagnation check does: with stall_reg > 0 the solve goes on with the Delassus matrix
   * G + stall_reg * mean(diag G) * I -- a slightly compliant contact set (constraint-force mixing) on which the sweeps do
   * converge -- and only a second failed check ends it; stall_reg = 0 ends it at once.  Fires on ~1 % of the steps of
   * fallen robots whose joint stops fight sticking contacts, never on standing ones (DESIGN.md section 5). */
  float stall_reg;      /*                                               (0.02)           */
} rsb_params;

/* raisim::Contact as returned by ArticulatedSystem::getContacts(): 12 words */
typedef struct rsb_contact {
  int32_t local_body;  /* Contact::getlocalBodyIndex()                                      */
  int32_t pair_index;  /* terrain feature: 0 = Ground plane, 2*cell+tri on a HeightMap;   */
                       /* self contact: -1 - the pair's second body (always < 0)           */
  float position[3];   /* Contact::getPosition()  (world)                                   */
  float normal[3];     /* Contact::getNormal()    (world, terrain -> robot; self: second -> first body) */
  float impulse[3];    /* Contact::getImpulse()   (world, on the robot)                     */
  float depth;         /* Contact::getDepth()                                               */
} rsb_contact;

/* host-side view of the model tables (doubles; arrays owned by the model) */
typedef struct rsb_model_tables {
  int nb, nq, nv, floating, ncoll, npts;
  const int *parent, *jtype, *qidx, *vidx, *depth;
  const double *jpos, *jrot, *axis, *mass, *com, *inertia, *jlimit;
  const int *cbody, *ctype;
  const double *csize, *cpos, *crot;
  const int *pt_body, *pt_coll, *pt_feat;
  const double *pt_pos, *pt_rad;
  /* contact candidates are typed: 0 = sphere of radius pt_rad at pt_pos (radius 0: box corner / cylinder rim sample), 1 = the
   * segment pt_pos .. pt_pos2 swept by pt_rad (capsule / cylinder side), 2 = the box of collision body pt_coll against terrain
   * vertices; types 1 and 2 come after the points and act on height maps only */
  const int* pt_type;
  const double* pt_pos2;
  const double* jeffort; /* [nb] URDF <limit effort> of the joint that carries the body (1e30 = none): the commanded torque saturates there */
} rsb_model_tables;

/* zero-copy device view (rows are padded: element (env, i) of X lives at X[env * X_stride + i]) */
typedef struct rsb_device_view {
  int num_envs, nq, nv, gc_stride, gv_stride;
  float *gc, *gv, *tau_ff, *ptarget, *vtarget;
  int32_t* ncontacts;
  rsb_contact* contacts; /* [num_envs][RSB_KMAX] */
} rsb_device_view;

const char* rsb_last_error(void);
int rsb_version(void);

/* ---- model: World::addArticulatedSystem(urdf) parsing half (SURVEY 3.3) ---------------------- */
int rsb_model_create_from_urdf(const char* path_or_xml, rsb_model** out);
void rsb_model_destroy(rsb_model* m);
/* binary cache of the compiled model tables (SURVEY 8f N2): skips XML parsing for fleets of workers; same-architecture file */
int rsb_model_save(const rsb_model* m, const char* path);
int rsb_model_load(const char* path, rsb_model** out);
int rsb_model_dims(const rsb_model* m, int* nq, int* nv, int* nb, int* ncoll, int* npts);
int rsb_model_get_tables(const rsb_model* m, rsb_model_tables* out);
int rsb_model_body_index(const rsb_model* m, const char* name);    /* ArticulatedSystem::getBodyIdx   */
const char* rsb_model_body_name(const rsb_model* m, int body);
int rsb_model_collision_index(const rsb_model* m, const char* name); /* getCollisionBody("LINK/k"): k-th collision body of a link */
const char* rsb_model_joint_name(const rsb_model* m, int body);
int rsb_model_frame_index(const rsb_model* m, const char* name);   /* getFrameIdxByName (link frames) */
int rsb_model_frame(const rsb_model* m, int frame, int* body, double pos[3], double rot[9]);

/* ---- batch lifetime --------------------------------------------------------------------------- */
int rsb_batch_create(const rsb_model* m, int num_envs, int device, rsb_batch** out);
void rsb_batch_destroy(rsb_batch* b);
int rsb_batch_set_stream(rsb_batch* b, void* cuda_stream);
int rsb_batch_sync(rsb_batch* b);
int rsb_batch_num_envs(const rsb_batch* b);

/* ---- world set-up ----------------------------------------------------------------------------- */
int rsb_batch_set_ground(rsb_batch* b, float z);                                   /* World::addGround    */
int rsb_batch_set_heightmap(rsb_batch* b, int x_samples, int y_samples, float x_size, float y_size,
                            float center_x, float center_y, const float* heights_host); /* World::addHeightMap */
int rsb_batch_clear_terrain(rsb_batch* b);
/* terrain atlas: upstream gives every environment its own World, hence possibly its own HeightMap; here `count` same-sized
 * maps ([count][y_samples][x_samples], host) share one batch and map_of_env[num_envs] (host) picks one per environment */
int rsb_batch_set_heightmaps(rsb_batch* b, int count, int x_samples, int y_samples, float x_size, float y_size,
                             float center_x, float center_y, const float* heights_host, const int32_t* map_of_env);
/* Terrain curriculum (legged_gym-style: an environment moves to a harder or easier map when it resets): environments
 * [env_begin, env_begin + env_count) collide with the maps map_of_env[env_count] (int32, host or device source, `where`) of the atlas
 * set by rsb_batch_set_heightmaps, from the next launch on.  No map is uploaded.  The indices are copied into the batch's staging
 * buffer (env_count words) and checked there on the device; the call waits for that check, then copies them into the atlas index in
 * stream order: launches enqueued before the call see the old assignment, later ones the new.  env_count == 0 does nothing.
 * The terrain enters neither M, h nor the poses: nothing goes stale and no step launch is added; the contact records and contact forces
 * of the last step stay as they were, and height scans read the new assignment from the call on.  Gym resets keep the assignment;
 * rsb_batch_set_heightmaps replaces it, rsb_batch_set_ground and rsb_batch_clear_terrain drop it.
 * Refused with RSB_ERR_INVALID, changing nothing: a null batch or map_of_env, a bad range or `where`, an index outside [0, count), or
 * no atlas (ground, no terrain, or the single map of rsb_batch_set_heightmap). */
int rsb_batch_set_heightmap_index(rsb_batch* b, const int32_t* map_of_env, int env_begin, int env_count, int where);
/* Maps first .. first + count - 1 of the terrain overwritten in place with heights [count][y_samples][x_samples] float32 (host or device
 * source, `where`), the samples, size and centre staying those of the terrain; any height-map terrain, the single map of
 * rsb_batch_set_heightmap being map 0.  Environments keep their map index.  The heights are copied into the batch's staging buffer,
 * which grows to count * x_samples * y_samples words, and checked there on the device, which also finds the largest height of every new
 * map; the call waits for that, then copies them over the maps in stream order (launches enqueued before the call see the old
 * heights, later ones the new).  The stage-B cull height stays the exact maximum over all maps.  count == 0 does nothing.  Like
 * rsb_batch_set_heightmap_index it adds no launch and makes nothing stale; height scans read the new heights from the call on.
 * Refused with RSB_ERR_INVALID, changing nothing: a null batch or heights, a bad `where`, first or count out of range, a height that is
 * not finite, or no height map. */
int rsb_batch_update_heightmaps(rsb_batch* b, int first, int count, const float* heights, int where);
int rsb_batch_set_params(rsb_batch* b, const rsb_params* p);
int rsb_batch_get_params(const rsb_batch* b, rsb_params* p);
int rsb_params_default(rsb_params* p);
/* friction of one collision body (index in rsb_model_tables order) against the terrain; mu < 0 = default material.
 * The per-body half of World::setMaterialPairProp / getCollisionBody(name).setMaterial, shared by all environments; per-environment
 * rows (rsb_batch_set_contact_friction) take precedence where they hold a value >= 0 */
int rsb_batch_set_collision_friction(rsb_batch* b, int collision_body, float mu);
/* Per-environment terrain friction of every collision body (World::setMaterialPairProp / setDefaultMaterial /
 * getCollisionBody(name).setMaterial, per World upstream).  rows [env_count][ncoll] float32 in the collision-body order of
 * rsb_model_tables; host or device source (`where`).  An entry mu >= 0 is the friction of that collision body's terrain contacts in that
 * environment; mu < 0 is the batch-level value, resolved at every launch: rsb_batch_set_collision_friction for that body if set, else
 * rsb_params.mu.  rows == NULL resets the range to -1.  The first call (and the first after rsb_batch_clear_contact_friction) starts
 * every environment at -1, then writes the range: no rows, rows of -1 and rows set then cleared compute the same bits.
 * Self contacts (candidates npts + j) keep their pair's friction; restitution stays per batch.  The rows live outside the model blob, so
 * rsb_batch_set_collision_friction, set_self_collision, set_params, the terrain calls and gym resets keep them.  The friction does not
 * enter M, h or the poses: nothing goes stale and no launch is added.
 * Refused with RSB_ERR_INVALID, changing nothing: a null batch, a bad range or `where`, or a value that is NaN or +-inf.  The rows are
 * checked on the device in the batch's staging buffer before any of them is committed; the call waits for that check. */
int rsb_batch_set_contact_friction(rsb_batch* b, const float* rows, int env_begin, int env_count, int where);
/* drop all per-environment friction rows: every later launch runs as if none had been set */
int rsb_batch_clear_contact_friction(rsb_batch* b);
/* Self-collision between the bodies of the robot (ArticulatedSystem collisions between its own bodies): OFF unless pairs are enabled
 * here.  pairs[n][2] are collision-body indices (rsb_model_tables / rsb_model_collision_index order), at most RSB_MAX_SELF_PAIRS; there
 * is no "all pairs" mode.  Supported: sphere-sphere, sphere-capsule, capsule-capsule, sphere-box (RSB_ERR_UNSUPPORTED, naming the pair,
 * for capsule-box, box-box and anything with a cylinder); two collision bodies of the same body are RSB_ERR_INVALID; parent-child pairs
 * are allowed; the world-welded root of a fixed-base robot acts as a static obstacle.  One contact per pair at the deepest point: normal
 * from the pair's second body to its first, position = midpoint of the two surface points, depth = penetration.  The impulse acts on the
 * first body and its negative on the second; friction mu[j] (NULL or mu[j] < 0: the default material; the per-collision-body terrain
 * friction does not apply); ERP and restitution as on terrain contacts.  Self contacts share the RSB_KMAX contacts with the terrain:
 * pair j is candidate npts + j (rsb_batch_get_contact_points), its rsb_contact has local_body = first body and
 * pair_index = -1 - second body.  n = 0 clears the pairs.  Everything is checked first: a refused call changes nothing.  A batch with
 * pairs runs the generic (not the model-specific) instance of the step kernel. */
#define RSB_MAX_SELF_PAIRS 32
int rsb_batch_set_self_collision(rsb_batch* b, const int32_t* pairs, int n, const float* mu);

/* ---- state and actuation (ArticulatedSystem::setState/getState/setPdGains/setPdTarget/
 *      setGeneralizedForce/setControlMode); buffers are tight [env_count][nq|nv] float32 ---------- */
int rsb_batch_set_state(rsb_batch* b, const float* gc, const float* gv, int env_begin, int env_count, int where);
int rsb_batch_get_state(rsb_batch* b, float* gc, float* gv, int env_begin, int env_count, int where);
/* [nv], host, all envs; per-environment actuator rows (rsb_batch_set_actuator_params) take precedence where they hold a value >= 0 */
int rsb_batch_set_pd_gains(rsb_batch* b, const float* kp, const float* kd);
int rsb_batch_set_pd_target(rsb_batch* b, const float* ptarget, const float* vtarget, int env_begin, int env_count, int where);
/* zero-copy PD targets for trainers on the same GPU: the step kernel reads rows [env][0..nq) straight from the
 * caller's device buffer (row_stride floats apart) until targets are copied in again or NULL is bound */
int rsb_batch_bind_pd_target(rsb_batch* b, const float* ptarget_device, int row_stride);
int rsb_batch_set_generalized_force(rsb_batch* b, const float* tau, int env_begin, int env_count, int where);
int rsb_batch_set_control_mode(rsb_batch* b, int mode);
/* ArticulatedSystem::setExternalForce(bodyIdx, pos, force) / setExternalTorque(bodyIdx, torque): one wrench per
 * environment on `body`, applied at point_body[3] (body frame, host pointer; NULL = body origin); force / torque are
 * [env_count][3] world-frame rows (NULL = zero).  Like upstream it acts during the next integrate() call only (all fused
 * sub-steps of that call) and is cleared afterwards. */
int rsb_batch_set_external_wrench(rsb_batch* b, int body, const float* force, const float* torque, const float* point_body,
                                  int env_begin, int env_count, int where);
/* Per-environment inertial parameters of every body (ArticulatedSystem::getMass / getBodyCOM_B / getInertia + updateMassInfo, per
 * World upstream).  rows [env_count][nb][10] float32: mass, centre of mass in the body frame (3), inertia about the centre of mass in
 * the body frame (xx, xy, xz, yy, yz, zz) -- the order of rsb_model_tables mass / com / inertia.  rows == NULL resets those
 * environments to the model's values.  Host or device source (`where`).
 * The first call (and the first after rsb_batch_clear_body_inertia) gives every environment the model's float32 values, the ones the
 * step uses without rows, then writes the range: rows equal to the model's values give results bit-identical to no rows.  Every later
 * launch of the step kernel uses the rows: integrate, integrate1, integrate2, control_step, gym_step and the kinematics pass of the
 * lazy getters (gym resets keep them).  M, h and the poses describe the new parameters from the next getter on.
 * Refused with RSB_ERR_INVALID, changing nothing: a bad range or `where`, a value that is not finite, a negative mass, or an inertia
 * that is not positive semidefinite.  The inertia test, in double precision with t = xx + yy + zz: every diagonal entry >= -1e-6 t,
 * every 2 x 2 principal minor >= -1e-6 t^2 and the determinant >= -1e-6 t^3.  The rows are checked on the device in the batch's
 * staging buffer before any of them is committed; the call waits for that check.  Collision shapes stay per batch; terrain friction
 * (rsb_batch_set_contact_friction) and gains and effort limits (rsb_batch_set_actuator_params) have rows of their own. */
int rsb_batch_set_body_inertia(rsb_batch* b, const float* rows, int env_begin, int env_count, int where);
/* drop all per-environment rows: every later launch runs exactly as if none had ever been set */
int rsb_batch_clear_body_inertia(rsb_batch* b);
/* Per-environment PD gains and actuator effort limits (ArticulatedSystem::setPdGains / setPGains / setDGains / setActuationLimits, per
 * World upstream).  rows [env_count][nv][3] float32 in the batch's gv order: kp, kd and the effort limit of every dof; host or device
 * source (`where`).  An entry < 0 is the batch-level value, resolved at every launch: kp and kd of rsb_batch_set_pd_gains (0 if it was
 * never called), the URDF <limit effort> of the joint; so a later rsb_batch_set_pd_gains still reaches the entries of -1.  An entry
 * >= 0 replaces it for that dof in that environment: kp = kd = 0 gives the dof no PD law, effort 0 lets the actuator give no torque,
 * effort +inf is no limit (stored as the batch's "none" value, so an unlimited joint computes the same bits either way).  The six
 * base dofs of a floating robot are not actuated: their entries are ignored and stored as -1.  rows == NULL resets the range to -1.
 * The first call (and the first after rsb_batch_clear_actuator_params) starts every environment at -1, then writes the range: no
 * rows, rows of -1 and rows set then cleared compute the same bits, and so do rows equal to the batch-level values.
 * The step kernel applies PD laws in RSB_PD_PLUS_FEEDFORWARD_TORQUE mode once rsb_batch_set_pd_gains was called or rows are active,
 * and rsb_batch_gym_step accepts either.  The effort limit holds in both control modes, as the URDF one does (in RSB_FORCE_AND_TORQUE
 * it saturates the feed-forward torque).  The rows live outside the model blob, so rsb_batch_set_pd_gains, set_collision_friction,
 * set_self_collision, set_params, the terrain calls and gym resets keep them.  The gains enter neither M, h nor the poses: nothing
 * goes stale and no launch is added.
 * Refused with RSB_ERR_INVALID, changing nothing: a null batch, a bad range or `where`, NaN anywhere, +-inf in kp or kd, or -inf in
 * the effort limit.  The rows are checked on the device in the batch's staging buffer before any of them is committed; the call waits
 * for that check. */
int rsb_batch_set_actuator_params(rsb_batch* b, const float* rows, int env_begin, int env_count, int where);
/* drop all per-environment actuator rows: every later launch runs as if none had been set */
int rsb_batch_clear_actuator_params(rsb_batch* b);
/* Learned actuator network (Hwangbo et al., Science Robotics 2019): the torque of each listed dof is an MLP of its own recent
 * position errors and velocities, evaluated by the step kernel at every sub-step from that sub-step's state.
 *   One network per batch, shared by dofs[n_dofs] (batch gv order; a floating robot's six base dofs are refused).
 *   Input: 2H features [e_t, e_{t-1}, ..., e_{t-H+1}, v_t, v_{t-1}, ..., v_{t-H+1}] with e = ptarget[q(d)] - gc[q(d)] (the float32
 *   subtraction of the PD law) and v = gv[d], the current ones taken at the start of the sub-step.  L hidden layers of width W, each
 *   affine then softsign x / (1 + |x|), then one linear output.  params are packed in torch.nn.Linear order: W1[W][2H], b1[W], ...,
 *   WL[W][W], bL[W], Wout[1][W], bout[1] (2HW + W + (L - 1)(W^2 + W) + W + 1 floats, host memory).  There are no scaling parameters:
 *   input normalisation and output scale fold exactly into the first and last layers (INTEGRATION.md).
 *   History: per environment and listed dof, (e, v) of the last H - 1 sub-steps.  Every launch that advances the state (integrate,
 *   integrate2, control_step, gym_step) shifts it once per sub-step, so 4 launches of 1 sub-step equal 1 launch of 4 sub-steps bit for
 *   bit; integrate1, the kinematics pass, the getters and the height scan neither evaluate the network nor shift the history.  The
 *   network and its history act in RSB_PD_PLUS_FEEDFORWARD_TORQUE mode only: in RSB_FORCE_AND_TORQUE mode the listed dofs get their
 *   feed-forward torque as every dof does and the history stays as it is.
 *   Torque: for a listed dof the network replaces the PD law (kp, kd and the velocity target of that dof are ignored).  The commanded
 *   torque tau_ff + net is explicit, constant over the sub-step (nothing is folded into the mass matrix), saturated at the dof's effort
 *   limit (URDF or rsb_batch_set_actuator_params row) and reported by rsb_batch_get_generalized_force as applied.  Unlisted dofs are
 *   unchanged.  A set network counts as PD gains for rsb_batch_gym_step.
 *   Resets: every rsb_batch_set_actuator_network call and rsb_batch_gym_reset zero all histories; a termination in rsb_batch_gym_step
 *   zeroes that environment's history.  rsb_batch_set_state does not touch it (set it with rsb_batch_set_actuator_history).
 *   n_dofs = 0 clears the network (the other arguments are then not read).  Refused with RSB_ERR_INVALID, changing nothing (the old
 *   network and history stay): a null batch, n_dofs outside [0, nv], a NULL, out-of-range, duplicated or base dof, history, layers or
 *   width out of range, NULL params with n_dofs > 0, a parameter that is not finite. */
#define RSB_ACTNET_MAX_HISTORY 4
#define RSB_ACTNET_MAX_LAYERS 4
#define RSB_ACTNET_MAX_WIDTH 32
int rsb_batch_set_actuator_network(rsb_batch* b, const int32_t* dofs, int n_dofs, int history, int layers, int width, const float* params);
/* History rows [env_count][n_dofs][2][H - 1] float32 (errors then velocities, most recent first), host or device (`where`).  rows ==
 * NULL zeroes the range.  The rows are checked on the device in the batch's staging buffer before any of them is committed; the call
 * waits for that check.  With H = 1 the rows have no words and both calls succeed without doing anything.  Refused with
 * RSB_ERR_INVALID, changing nothing: a null batch, no network, a bad range or `where`, a value that is not finite. */
int rsb_batch_set_actuator_history(rsb_batch* b, const float* rows, int env_begin, int env_count, int where);
int rsb_batch_get_actuator_history(rsb_batch* b, float* rows, int env_begin, int env_count, int where);
/* Actuation delay: a joint command takes effect a chosen number of physics sub-steps after it was issued, per environment (a real
 * robot applies a policy's command some milliseconds late; training draws the delay per environment at every episode reset).
 *   Command: at every advancing sub-step, the triple (ptarget[q(d)], vtarget[d], tau_ff[d]) the step would use for every dof d that is
 *   not one of a floating base's six, whatever its source: rsb_batch_set_pd_target, a bound buffer (rsb_batch_bind_pd_target),
 *   rsb_batch_control_step targets (pinned rows read in place included), the gym task's action * std + mean, rsb_batch_set_generalized_force.
 *   It is recorded in both control modes.
 *   Delay and history: each environment has a delay d in [0, RSB_MAX_ACTUATION_DELAY] sub-steps and a command history.  With t the
 *   advancing sub-steps since the history was last emptied, counted from 0, sub-step t applies cmd(max(t - d, 0)): after an emptying
 *   the first command holds for the first d + 1 sub-steps.  The applied command is what the implicit PD law and its saturation test,
 *   the actuator network's error and rsb_batch_get_generalized_force use.  Gains, effort limits and the network are not delayed; the
 *   batch's target rows keep the commanded values, so targets persist across launches as they do without a delay.
 *   Only launches that advance the state record a command: integrate, integrate2, control_step, gym_step.  integrate1, the kinematics
 *   pass, the getters, the frame calls and the height scan do not, so 1 launch of 4 sub-steps equals 4 launches of 1 bit for bit.
 *   Emptying: setting an environment's delay, rsb_batch_gym_reset (every environment) and a termination in rsb_batch_gym_step (that
 *   environment) empty its history; the last two keep the delay.  rsb_batch_set_state and rsb_batch_set_pd_target do not.
 * delays [env_count] int32, host or device (`where`): an entry d >= 0 sets that environment's delay and empties its history, an entry
 * -1 leaves the environment as it is (so a trainer may pass where(done, new_delay, -1) from the device).  delays == NULL sets 0 and
 * empties the whole range.  The first call, and the first after rsb_batch_clear_actuation_delay, starts every environment at delay 0
 * with an empty history; delays of 0 give results bit-identical to no delay.  The entries are checked on the device in the batch's
 * staging buffer before any is committed; the call waits for that check.  Refused with RSB_ERR_INVALID, changing nothing: a null
 * batch, a bad range or `where`, an entry < -1 or > RSB_MAX_ACTUATION_DELAY. */
#define RSB_MAX_ACTUATION_DELAY 16
int rsb_batch_set_actuation_delay(rsb_batch* b, const int32_t* delays, int env_begin, int env_count, int where);
/* drop the delays and the histories: every later launch runs exactly as if none had been set */
int rsb_batch_clear_actuation_delay(rsb_batch* b);
/* ArticulatedSystem::getGeneralizedForce(): feed-forward + PD force applied over the last integrate() */
int rsb_batch_get_generalized_force(rsb_batch* b, float* tau, int env_begin, int env_count, int where);

/* ---- the hot path: World::integrate1(), integrate2(), integrate() ----------------------------- */
int rsb_batch_integrate1(rsb_batch* b);               /* kinematics, collision, M, h (for the getters)   */
int rsb_batch_integrate2(rsb_batch* b);               /* contact solve + state integration               */
int rsb_batch_integrate(rsb_batch* b, int substeps);  /* substeps x integrate(), one fused launch        */

/* ---- read-backs (lazy getters of the reference, SURVEY 3.4): M, h and poses always describe the current state ---- */
int rsb_batch_get_mass_matrix(rsb_batch* b, int env_begin, int env_count, float* out, int where);     /* [n][nv*nv] getMassMatrix     */
int rsb_batch_get_nonlinearities(rsb_batch* b, int env_begin, int env_count, float* out, int where);  /* [n][nv]    getNonlinearities */
int rsb_batch_get_body_poses(rsb_batch* b, int env_begin, int env_count, float* rot, float* pos, int where); /* [n][nb*9],[n][nb*3] */
int rsb_batch_get_contacts(rsb_batch* b, rsb_contact* out, int32_t* counts, int env_begin, int env_count, int where); /* out [n][RSB_KMAX] */
int rsb_batch_get_contact_points(rsb_batch* b, int32_t* pt_index, int env_begin, int env_count, int where);          /* [n][RSB_KMAX] candidate-point ids */
int rsb_batch_get_solver_iterations(rsb_batch* b, int32_t* iters, int env_begin, int env_count, int where);          /* getContactSolver().getLoopCounter() */
int rsb_batch_get_diverged(rsb_batch* b, int32_t* flags, int env_begin, int env_count, int where);                   /* 1 = state went non-finite in the last step: reset it */
/* a diverged environment with an actuator network also carries NaN in its actuator history until that is set (rsb_batch_set_actuator_history) */
/* how the last contact solve of every environment ended */
#define RSB_SOLVER_CONVERGED 0           /* largest impulse update < threshold                                         */
#define RSB_SOLVER_CONVERGED_COMPLIANT 1 /* ... on the compliant contact set entered after a failed stagnation check   */
#define RSB_SOLVER_STALLED 2             /* ended by a failed stagnation check (second one when stall_reg > 0)          */
#define RSB_SOLVER_MAXITER 3             /* max_iter sweeps without reaching the threshold                              */
int rsb_batch_get_solver_status(rsb_batch* b, int32_t* status, int env_begin, int env_count, int where);
int rsb_batch_get_solver_residual(rsb_batch* b, float* resid, int env_begin, int env_count, int where);              /* largest impulse update of the last sweep (< threshold: converged) */
/* ---- frame kinematics (ArticulatedSystem::getFramePosition / getFrameOrientation / getFrameVelocity / getFrameAngularVelocity /
 *      getDenseFrameJacobian for every environment at once).  The getters are lazy like rsb_batch_get_body_poses: they describe the
 *      current state and run the kinematics pass only when the state changed through this API since the last one (one launch, plus
 *      that pass when it is due).  They leave the contact records, solver outputs, diverged flags and applied torques of the last
 *      integrate() as they were and have no effect on any later step.  After rsb_batch_integrate2() the getters' buffers hold the
 *      poses from before that step (M and h stay those of integrate1()); the frame getters then run the kinematics pass for the
 *      stepped state first, so poses and velocities always belong to one state, and M, h and the body poses describe it too from
 *      then on.  Device buffers are tight rows, written in stream order.  Host buffers are written when the call returns; they are
 *      staged through the batch's staging buffer (env_count * F floats times 18 for the states, times 6 * nv for the Jacobians):
 *      device buffers avoid it. */
#define RSB_MAX_FRAMES 64
/* Frames rigidly attached to bodies, shared by all environments: body[n] (rsb_model_body_index order), pos[n][3] in the body frame,
 * rot[n][9] row-major orientation in the body frame (NULL = identity).  rsb_model_frame() returns exactly (body, pos, rot) for the
 * URDF's link frames.  n = 0 clears.  A refused call (n < 0 or > RSB_MAX_FRAMES, a body out of range, NULL body or pos with n > 0)
 * changes nothing. */
int rsb_batch_set_frames(rsb_batch* b, const int32_t* body, const float* pos, const float* rot, int n);
/* World frame, current state: pos [n][F][3], rot [n][F][9] (R_body * rot), lin_vel [n][F][3] (velocity of the frame's point),
 * ang_vel [n][F][3] (angular velocity of its body).  A NULL output is skipped.  RSB_ERR_INVALID when no frames are set. */
int rsb_batch_get_frame_states(rsb_batch* b, int env_begin, int env_count, float* pos, float* rot, float* lin_vel, float* ang_vel, int where);
/* [n][F][6][nv] row-major: rows 0-2 translational (v_point = Jp gv), rows 3-5 rotational (omega = Jr gv).
 * Columns follow the batch's gv order; for a floating base that is [v_world | omega_world | joints].  Non-ancestor columns are 0. */
int rsb_batch_get_frame_jacobians(rsb_batch* b, int env_begin, int env_count, float* jac, int where);
/* ---- contact forces per body over a whole launch.  A launch that advances the state (rsb_batch_integrate, rsb_batch_integrate2,
 *      rsb_batch_control_step, rsb_batch_gym_step) runs `substeps` sub-steps, and the contact records above are those of the last one
 *      only.  For up to RSB_MAX_CONTACT_BODIES chosen bodies, shared by all environments, the step kernel also gathers, as the
 *      sub-steps go by:
 *        force[env][s][3]         world frame, newtons: the sum over all sub-steps of the launch and over all contacts acting on body s
 *                                 in each of them of the contact impulse on the body, times the float32 reciprocal of substeps * dt: the
 *                                 mean contact force on the body over the launch.  A terrain contact acts on its local_body with the
 *                                 impulse rsb_contact::impulse would show; a self contact with +impulse on its first body (local_body)
 *                                 and -impulse on its second (-1 - pair_index), on both when both are listed.  Joint-limit rows and
 *                                 external wrenches do not enter.
 *        steps_in_contact[env][s] the number of sub-steps of the launch in which the body had at least one contact in the environment's
 *                                 contact list (as first or second body), whatever the impulse: > 0 = touched during the launch,
 *                                 == substeps = in contact throughout.
 *      Contacts are summed in contact-list order and sub-steps in time order, one lane per body: results are bit-identical from run to
 *      run and for every launch shape.  A candidate cut by the RSB_KMAX cap carries no impulse in the solve and none here.  Each
 *      advancing launch overwrites both outputs; every other launch (rsb_batch_integrate1, the kinematics pass of the lazy getters,
 *      rsb_batch_update_kinematics, the frame getters) leaves them as they are, like the contact records.  They read zero from
 *      rsb_batch_set_contact_bodies() until the first advancing launch.  In rsb_batch_gym_step an environment that terminates and is
 *      reset keeps the forces of the step that ended it.  With no bodies set the step computes and stores nothing for this.  Upstream
 *      has no such call: there, user code sees every sub-step's getContacts() between its own World::integrate() calls. */
#define RSB_MAX_CONTACT_BODIES 32
/* body[n] in rsb_model_body_index order; a body may be listed twice.  n = 0 clears.  Refused with RSB_ERR_INVALID, changing nothing:
 * n < 0 or > RSB_MAX_CONTACT_BODIES, NULL with n > 0, a body out of range. */
int rsb_batch_set_contact_bodies(rsb_batch* b, const int32_t* body, int n);
/* force [n][S][3] float32, steps_in_contact [n][S] int32, S = the number of bodies set; a NULL output is skipped; RSB_ERR_INVALID when
 * no bodies are set.  A plain copy of a contiguous slice of the batch's rows in stream order: no launch, host or device destination. */
int rsb_batch_get_body_contact_forces(rsb_batch* b, int env_begin, int env_count, float* force, int32_t* steps_in_contact, int where);
/* ---- IMU readings over a whole launch: what an accelerometer and a gyroscope rigidly attached to a body measure, for every
 *      environment at once, gathered by the step kernel as the sub-steps go by.
 *      Sensors: up to RSB_MAX_IMUS, shared by all environments.  Sensor k is attached to body[k]: its origin is at pos[k] and its
 *      orientation is rot[k], both in the body frame (the triple rsb_model_frame returns for a URDF link frame, as for
 *      rsb_batch_set_frames).
 *      Notation: a launch that advances the state (rsb_batch_integrate, rsb_batch_integrate2, rsb_batch_control_step, rsb_batch_gym_step)
 *      runs S sub-steps; (q_s, v_s) is the state at the start of sub-step s and v_{s+1} the velocity it produces.  x_k(q) is the
 *      sensor's world point, R_k(q) = R_body(q) * rot[k] its world orientation, J_p, J_r the point and rotational Jacobians of
 *      rsb_batch_get_frame_jacobians, g = rsb_params.gravity, dt = rsb_params.dt.
 *      Per sub-step:
 *        specific force  f_s = R_k(q_s)^T [ J_p(q_s) (v_{s+1} - v_s) / dt + Jdot_p(q_s, v_s) v_s - g ]: the classical acceleration of the
 *                        sensor point that the sub-step's generalized acceleration gives at its start state, minus gravity.  The
 *                        velocity difference is the one the step forms before it adds it to v_s.
 *        angular rate    w_s = R_k(q_s)^T J_r(q_s) v_{s+1}: the rate the semi-implicit update turns the pose by over the sub-step (a
 *                        floating base's quaternion update uses exactly this omega).
 *      Output of a launch, per environment and sensor, float32 in the sensor frame: lin_acc = (sum_s f_s) * (1 / S) [m/s^2] and ang_vel =
 *      (sum_s w_s) * (1 / S) [rad/s], summed in sub-step order and multiplied by the float32 reciprocal of S.
 *      So a sensor at rest on a robot standing still reads +|g| along the sensor-frame direction opposite to gravity, a robot in free fall
 *      reads 0, and a body spinning at a constant rate w reads the centripetal -w^2 r_perp and the rate w.
 *      Each advancing launch overwrites both outputs; every other launch (rsb_batch_integrate1, the kinematics pass of the lazy getters,
 *      rsb_batch_update_kinematics, the frame getters, the height scan) leaves them as they are.  They read zero from rsb_batch_set_imus()
 *      until the first advancing launch.  In rsb_batch_gym_step an environment that terminates keeps the readings of the sub-steps that
 *      ended it: the reset comes after them.  rsb_batch_set_state changes nothing until the next launch; a reading covers its own launch
 *      only, so there is no history to reset.  A diverged environment may read NaN.  One lane per sensor and sub-steps in time order:
 *      readings are bit-identical from run to run and for every launch shape.  With no sensors set the step computes and stores
 *      nothing for this.  Noise, bias and drift are left to the caller; the sensor's orientation comes from the frame getters or gc. */
#define RSB_MAX_IMUS 8
/* body[n] in rsb_model_body_index order, pos[n][3], rot[n][9] row-major (NULL = identity).  n = 0 clears.  Refused with
 * RSB_ERR_INVALID, changing nothing: a null batch, n < 0 or > RSB_MAX_IMUS, body or pos NULL with n > 0, a body out of range, a pos or
 * rot entry that is not finite, a rot that is not a rotation (|R^T R - I| > 1e-4 in some entry, or det R <= 0, in double precision). */
int rsb_batch_set_imus(rsb_batch* b, const int32_t* body, const float* pos, const float* rot, int n);
/* lin_acc [n][I][3], ang_vel [n][I][3] float32, I = the number of sensors set; a NULL output is skipped; RSB_ERR_INVALID when no
 * sensors are set, or for a bad range or `where`.  A plain copy of a contiguous slice of the batch's rows in stream order: no launch,
 * host or device destination. */
int rsb_batch_get_imu_readings(rsb_batch* b, int env_begin, int env_count, float* lin_acc, float* ang_vel, int where);
/* ---- terrain height scans (what an upstream ENVIRONMENT builds in observe() with HeightMap::getHeight(x, y) once per point, for
 *      every environment at once).  One list of points, shared by all environments; point i hangs on body[i] at the horizontal
 *      offset xy[i][2].  Its sample is, with (p, R) the body's world pose:
 *        RSB_SCAN_YAW    p_xy + Rz(psi) offset, (cos psi, sin psi) = (R00, R10) normalised (psi = 0 when that norm is < 1e-6):
 *                        the offsets turn with the body's heading and ignore its roll and pitch;
 *        RSB_SCAN_WORLD  p_xy + offset.
 *      The height is the world z of the collision surface there: the ground's z, or the environment's own height map (terrain atlas),
 *      two triangles per cell split along P00-P11 with the narrow phase's float arithmetic, so the scan shows the surface the robot
 *      collides with.  Outside the map the sample is clamped to the nearest border point, as HeightMap::getHeight does.  A sample with
 *      a coordinate that is not finite (a diverged environment) reads NaN.  The terrain is read at call time.
 *      Poses: a point on the root of a floating-base robot takes its pose from gc (position gc[0:3], heading from the normalised
 *      quaternion), so a list of base points is one launch and never runs the kinematics pass; a point on any other body uses the
 *      kinematics pass's poses, which the call runs first when they are stale, as the frame getters do.  The scan leaves the state,
 *      contact records, contact forces, solver outputs, diverged flags and applied torques as they were and has no effect on any
 *      later step.  Host outputs are staged through the batch's staging buffer (env_count * P * 3 floats). */
#define RSB_MAX_SCAN_POINTS 1024
#define RSB_SCAN_YAW 0   /* offsets turn with the anchor body's heading */
#define RSB_SCAN_WORLD 1 /* offsets are along the world x / y axes      */
/* body[n] in rsb_model_body_index order, xy[n][2], align RSB_SCAN_YAW / RSB_SCAN_WORLD for all points.  n = 0 clears.  Refused with
 * RSB_ERR_INVALID, changing nothing: n < 0 or > RSB_MAX_SCAN_POINTS, body or xy NULL with n > 0, a body out of range, an offset that is
 * not finite, another align. */
int rsb_batch_set_height_scan(rsb_batch* b, const int32_t* body, const float* xy, int n, int align);
/* height [n][P] (world z of the surface at each sample) and xy_out [n][P][2] (the world sample location), P = the number of points
 * set; a NULL output is skipped (both NULL: nothing is launched).  RSB_ERR_INVALID when no points are set or there is no terrain. */
int rsb_batch_get_height_scan(rsb_batch* b, int env_begin, int env_count, float* height, float* xy_out, int where);
/* FK, M and h of the CURRENT state for the getters above, without touching the contact records of the last integrate()
 * (upstream's getters are lazy the same way).  The getters call it themselves when the state changed through this API;
 * call it explicitly after writing the state through rsb_batch_device_ptrs() views. */
int rsb_batch_update_kinematics(rsb_batch* b);
int rsb_batch_device_ptrs(rsb_batch* b, rsb_device_view* view);
int64_t rsb_batch_launch_count(const rsb_batch* b);   /* kernels launched by this batch so far */

/* ---- RaisimGym observation row (VectorizedEnvironment::observe), ANYmal locomotion layout:
 *      [z, R^T e_z (3), joint q (nq-7), R^T v (3), R^T w (3), joint rates (nv-6)]  -> ob_dim = nq+nv-3 -- */
int rsb_batch_ob_dim(const rsb_batch* b);
int rsb_batch_observe(rsb_batch* b, float* obs, int env_begin, int env_count, int where);
/* VectorizedEnvironment::step() for the whole batch in one call: targets in, `substeps` fused
 * World::integrate() calls, observation rows out (either pointer may be NULL to skip that leg) */
int rsb_batch_control_step(rsb_batch* b, const float* ptarget, const float* vtarget, int where_in, int substeps, float* obs, int where_out);

/* ---- terrain generation (raisim::TerrainProperties, World::addHeightMap(centerX, centerY, terrainProperties)) ------ */
typedef struct rsb_terrain_properties {
  int x_samples, y_samples;      /* TerrainProperties::xSamples, ySamples */
  double x_size, y_size;         /* xSize, ySize [m]                       */
  double frequency;              /* base frequency of the noise [1/m]      */
  double z_scale;                /* zScale                                 */
  int fractal_octaves;           /* fractalOctaves                         */
  double fractal_lacunarity;     /* fractalLacunarity                      */
  double fractal_gain;           /* fractalGain                            */
  double step_size;              /* stepSize (0 = smooth)                  */
  double height_offset;          /* heightOffset                           */
  uint32_t seed;                 /* seed                                   */
} rsb_terrain_properties;
int rsb_terrain_generate(const rsb_terrain_properties* p, float* heights_out /* [y_samples][x_samples] */);

/* height-map files: World::addHeightMap(raisimHeightMapFileName, centerX, centerY) -- text, header "xSamples ySamples xSize
 * ySize" then the heights, x fastest -- and World::addHeightMap(pngFileName, centerX, centerY, xSize, ySize, heightScale,
 * heightOffset) -- 8/16-bit PNG, height = pixel * scale + offset.  heights == NULL only reports the sample counts. */
int rsb_heightmap_read_text(const char* path, int* x_samples, int* y_samples, double* x_size, double* y_size, float* heights, int capacity);
int rsb_heightmap_read_png(const char* path, double height_scale, double height_offset, int* x_samples, int* y_samples, float* heights, int capacity);

/* ---- multi-GPU inside one process (SURVEY 8e): one rsb_batch per GPU, NCCL all-gather of the observation rows ----
 *      (NCCL is bound at run time; bench.py uses torch.distributed for the same collective, one process per GPU) */
typedef struct rsb_comm rsb_comm;
int rsb_comm_init(rsb_batch** batches, int ndev, rsb_comm** out);             /* ncclCommInitAll over the batches' devices */
int rsb_comm_allgather_obs(rsb_comm* c, float* const* obs_all_per_device);     /* observe + ncclAllGather on every device     */
void rsb_comm_destroy(rsb_comm* c);

/* ---- multi-GPU, one process per GPU: the observation all-gather FUSED into the step kernel over NVLink peer memory ----
 * Every rank allocates two gathered-rows buffers [world * num_envs][ob_dim] and one counter row unsigned[world]
 * (rsb_peer_buffer_create: cudaMalloc + CUDA IPC handle), ships the 64-byte handles to its peers over any host channel
 * (torch.distributed / MPI / a pipe), maps theirs (rsb_peer_buffer_open) and hands all pointers to its batch.  From then on
 * a control step that returns observation rows on the device also stores every finished row straight into every rank's
 * buffer (parity = control step & 1) while the kernel is still running, and bumps a counter on every rank as each CTA ends;
 * the last CTA of the launch stays until every rank's counter shows its rows of this step, so the launch completes when the
 * gathered rows are complete (bounded: a dead peer traps).  rsb_batch_wait_observation_peers() tells which of the two buffers
 * holds the rows of the last step.  No NCCL call on the data path.  Every rank must step the same number of times. */
int rsb_peer_buffer_create(int device, size_t bytes, void** dev_ptr, unsigned char* handle64 /* may be NULL */);
int rsb_peer_buffer_open(int device, const unsigned char* handle64, void** dev_ptr);
int rsb_peer_buffer_close(void* dev_ptr);
int rsb_peer_buffer_destroy(void* dev_ptr);
int rsb_batch_set_observation_peers(rsb_batch* b, int world, int rank, void* const* obs_all /* [2 * world] */, void* const* flags /* [world] */);
int rsb_batch_wait_observation_peers(rsb_batch* b, int* buffer_parity /* may be NULL */);

/* ---- RaisimGym task on the device (raisimGymTorch VectorizedEnvironment.hpp / envs/rsg_anymal/Environment.hpp,
 *      [RECALL]): pTarget = action * std + mean; reward = torque_coeff * |tau|^2 + forward_vel_coeff * min(4, v_body_x);
 *      an episode terminates on any contact whose local body is not in foot_bodies (reward += terminal_reward, state reset) -- */
int rsb_batch_gym_configure(rsb_batch* b, const float* gc_init, const float* gv_init, const float* action_mean, const float* action_std,
                            const int32_t* foot_bodies, int n_foot, float torque_coeff, float forward_vel_coeff, float terminal_reward);
int rsb_batch_gym_reset(rsb_batch* b);                                             /* VectorizedEnvironment::reset() */
/* ::step() + ::observe() in ONE launch of the step kernel: action rows -> PD targets, `substeps` x World::integrate(), reward,
 * isTerminalState(), reset() of the terminated environments, observation rows of the resulting state.  Needs rsb_batch_set_pd_gains(),
 * active per-environment actuator rows (rsb_batch_set_actuator_params) or an actuator network (rsb_batch_set_actuator_network). */
int rsb_batch_gym_step(rsb_batch* b, const float* action, int where_in, int substeps, float* obs, float* reward, unsigned char* done,
                       int where_out);

#ifdef __cplusplus
}
#endif
#endif /* RSB_H_ */
