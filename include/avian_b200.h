/*
 * avian_b200.h — C ABI of libavian_b200.so, the H100-native replacement for the avian3d substep hot path.
 *
 * The reference (avianphysics/avian @ 5bef382) has no FFI: its hot path is three Bevy plugins
 * (`IntegratorPlugin`, `BroadPhasePlugin`, `SolverPlugin` + `XpbdSolverPlugin`).  A thin Rust shim
 * (INTEGRATION.md) snapshots the ECS component columns those plugins read into the column structs
 * below once per physics step, calls the entry points here, and scatters the results back.
 *
 * Each entry point cites the reference system(s) it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every function returns an AvnStatus (0 = ok, < 0 = error); nothing throws or aborts across the ABI;
 *     avn_last_error() returns a human-readable message for the last failing call on that context.
 *   - the caller owns all host buffers; they must stay valid until the call returns.  Buffers obtained
 *     from avn_alloc_pinned() are page-locked, which makes the host<->device copies asynchronous DMA.
 *   - the library owns all device memory.  One call in flight per context; a context is not thread-safe,
 *     but any host thread may call (the context binds its CUDA device on entry).
 *   - "scalar" columns are `float` when the context was created with scalar_bits = 32 and `double` when
 *     scalar_bits = 64 (reference features `f32` / `f64`, crates/avian3d/Cargo.toml:14-77).
 *   - Vec3 columns are packed [n][3], quaternions are packed [n][4] in glam order x,y,z,w, symmetric 3x3
 *     matrices are packed [n][6] = m00,m01,m02,m11,m12,m22 (glam_matrix_extras::SymmetricMat3).
 *   - there is NO CPU fallback: if no CUDA device is usable avn_create() fails with AVN_ERR_CUDA.
 */
#ifndef AVIAN_B200_H
#define AVIAN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AVN_ABI_VERSION 1u

/* src/dynamics/solver/constraint_graph.rs:39-48 */
#define AVN_GRAPH_COLOR_COUNT 24
#define AVN_COLOR_OVERFLOW 23
#define AVN_DYNAMIC_COLOR_COUNT 20
/* ContactManifold::prune_points keeps at most 4 points in 3D (src/collision/contact_types/mod.rs:478-566). */
#define AVN_MAX_MANIFOLD_POINTS 4
/* A contact/joint body that has no solver body and no column entry (static, zero velocity). */
#define AVN_NO_BODY (-1)

typedef enum AvnStatus {
    AVN_OK = 0,
    AVN_ERR_INVALID_ARGUMENT = -1,
    AVN_ERR_CUDA = -2,
    AVN_ERR_OUT_OF_MEMORY = -3,
    AVN_ERR_UNSUPPORTED = -4,
    AVN_ERR_CAPACITY = -5,
    AVN_ERR_NCCL = -6
} AvnStatus;

/* RigidBody (src/dynamics/rigid_body/mod.rs). Static entries are optional: they carry pose for joints and
 * LinearVelocity for contact tangents but are SolverBody::DUMMY inside the solver (solver_body/mod.rs:93-104). */
typedef enum AvnBodyKind { AVN_BODY_DYNAMIC = 0, AVN_BODY_KINEMATIC = 1, AVN_BODY_STATIC = 2 } AvnBodyKind;

/* LockedAxes bit layout (src/dynamics/rigid_body/locked_axes.rs; same bits as SolverBodyFlags, solver_body/mod.rs:133-146). */
#define AVN_LOCK_TRANSLATION_X 0x20u
#define AVN_LOCK_TRANSLATION_Y 0x10u
#define AVN_LOCK_TRANSLATION_Z 0x08u
#define AVN_LOCK_ROTATION_X 0x04u
#define AVN_LOCK_ROTATION_Y 0x02u
#define AVN_LOCK_ROTATION_Z 0x01u

/* integration_flags bits: marker components integrator/mod.rs:168-195 */
#define AVN_CUSTOM_VELOCITY_INTEGRATION 0x1u
#define AVN_CUSTOM_POSITION_INTEGRATION 0x2u

/* AabbIntervalFlags, src/collision/broad_phase.rs:187-196 */
#define AVN_AABB_IS_INACTIVE 0x01u
#define AVN_AABB_CONTACT_EVENTS 0x02u
#define AVN_AABB_GENERATE_CONSTRAINTS 0x04u
#define AVN_AABB_CUSTOM_FILTER 0x08u
#define AVN_AABB_MODIFY_CONTACTS 0x10u
/* Multi-GPU x-slab partition (SURVEY 8e): the interval is a copy of one owned by the next slab ("halo").  It is only ever the LATER
 * element of a pair: the sweep never starts from it, so pairs between two halo intervals are left to the slab that owns them.  Not a
 * reference flag; single-GPU callers never set it. */
#define AVN_AABB_HALO 0x80u
/* An interval that reaches far beyond its own slab (a ground slab) is not swept by its owner alone: it carries AVN_AABB_SPLIT_I in
 * every slab it reaches and pairs, as the earlier element, only with intervals that slab owns (never with AVN_AABB_HALO ones).  In
 * the slabs that do not own it it also carries AVN_AABB_NOT_J: it is never the later element there. */
#define AVN_AABB_SPLIT_I 0x40u
#define AVN_AABB_NOT_J 0x20u

/* Flag bits of an emitted pair (what collect_collision_pairs stores on ContactEdge / ContactPair,
 * broad_phase.rs:443-468) plus NEEDS_HOOK: the shim must still call CollisionHooks::filter_pairs for it
 * (broad_phase.rs:431-439), in list order, and drop the pair when the hook says no. */
#define AVN_PAIR_CONTACT_EVENTS 0x01u
#define AVN_PAIR_MODIFY_CONTACTS 0x02u
#define AVN_PAIR_GENERATE_CONSTRAINTS 0x04u
#define AVN_PAIR_NEEDS_HOOK 0x08u

typedef struct AvnContext AvnContext;

typedef struct AvnConfig {
    uint32_t abi_version;     /* AVN_ABI_VERSION */
    int32_t device;           /* CUDA device ordinal */
    uint32_t scalar_bits;     /* 32 (feature f32) or 64 (feature f64) */
    uint32_t flags;           /* AVN_CFG_* */
} AvnConfig;

/* Evaluate sin/cos of Quat::from_scaled_axis in double and round (bit-compatible with a correctly rounded
 * libm; default).  Without it the f32 path uses the CUDA sinf/cosf (<= 1 ulp). */
#define AVN_CFG_FAST_TRIG 0x1u

/* ---- step parameters: resources read by the three plugins -------------------------------------------- */
typedef struct AvnStepParams {
    double dt;                /* Time<Physics>::delta_secs_f64()  (src/schedule/mod.rs:247-260) */
    double h;                 /* Time<Substeps>::delta_secs_f64() (solver/schedule.rs:195-200)  */
    uint32_t substeps;        /* SubstepCount (solver/schedule.rs:187-191) */
    uint32_t restitution_iterations; /* SolverConfig (solver/plugin.rs:291-302) */
    double gravity[3];        /* Gravity (integrator/mod.rs:150-162) */
    double contact_damping_ratio;
    double contact_frequency_factor;
    double max_overlap_solve_speed;
    double warm_start_coefficient;
    double restitution_threshold;
    double length_unit;       /* PhysicsLengthUnit (solver/plugin.rs:200-207) */
    uint32_t match_contacts;  /* NarrowPhaseConfig::match_contacts: warm starting enabled (plugin.rs:432) */
    uint32_t solver_iterations; /* EXTENSION, reference semantics = 1: repeats the biased solve pass (SURVEY D2) */
} AvnStepParams;

/* ---- bodies: Appendix B of SURVEY.md; queries at solver_body/plugin.rs:174-185, integrator/mod.rs:261-268 */
typedef struct AvnBodyColumns {
    uint32_t count;
    uint32_t _pad;
    const uint8_t* kind;              /* AvnBodyKind */
    void* position;                   /* [n][3] in/out  Position */
    void* rotation;                   /* [n][4] in/out  Rotation */
    void* linear_velocity;            /* [n][3] in/out  LinearVelocity */
    void* angular_velocity;           /* [n][3] in/out  AngularVelocity */
    const void* inverse_mass;         /* [n]     ComputedMass::inverse() */
    const void* inverse_inertia_local;/* [n][6]  ComputedAngularInertia::inverse() (local frame) */
    const void* center_of_mass;       /* [n][3]  ComputedCenterOfMass (local); NULL = zero */
    const uint8_t* locked_axes;       /* NULL = none */
    const int8_t* dominance;          /* NULL = 0 */
    const void* linear_damping;       /* [n] NULL = 0 */
    const void* angular_damping;      /* [n] NULL = 0 */
    const void* gravity_scale;        /* [n] NULL = 1 */
    const void* linear_acceleration;  /* [n][3] VelocityIntegrationData::linear_increment as written by ForcePlugin
                                         (an acceleration until UpdateVelocityIncrements); NULL = 0 */
    const void* angular_acceleration; /* [n][3] NULL = 0 */
    const void* max_linear_speed;     /* [n] MaxLinearSpeed; NULL or +inf = absent */
    const void* max_angular_speed;    /* [n] MaxAngularSpeed; NULL or +inf = absent */
    const uint8_t* integration_flags; /* NULL = 0 */
} AvnBodyColumns;

/* ---- contact manifolds, grouped by graph colour (ConstraintGraph.colors[c].manifold_handles order,
 *      solver/plugin.rs:389-434; ContactManifold/ContactPoint at contact_types/mod.rs:342-378,603-660) ---- */
typedef struct AvnManifoldColumns {
    uint32_t count;                                     /* M */
    uint32_t point_count;                               /* P = point_offsets[M] */
    uint32_t color_offsets[AVN_GRAPH_COLOR_COUNT + 1];  /* colour c owns manifolds [off[c], off[c+1]) */
    const int32_t* body1;             /* [M] index into AvnBodyColumns or AVN_NO_BODY */
    const int32_t* body2;
    const void* normal;               /* [M][3] */
    const void* friction;             /* [M] */
    const void* restitution;          /* [M] */
    const void* tangent_velocity;     /* [M][3] NULL = 0 */
    const uint32_t* point_offsets;    /* [M+1], at most AVN_MAX_MANIFOLD_POINTS per manifold */
    const void* anchor1;              /* [P][3] */
    const void* anchor2;              /* [P][3] */
    const void* penetration;          /* [P] */
    const void* normal_speed;         /* [P] */
    void* warm_start_normal_impulse;  /* [P]    in/out (store_contact_impulses, plugin.rs:741-750) */
    void* warm_start_tangent_impulse; /* [P][2] in/out */
    void* normal_impulse;             /* [P]    out: ContactPoint::normal_impulse (total) */
} AvnManifoldColumns;

/* ---- joints: five typed arrays in the reference's solve order (xpbd/plugin.rs:58-86), each in ECS table
 *      order.  Frames are the already-localised ones (update_local_frames in joints/{fixed,revolute,...}.rs). ------------------ */
typedef enum AvnJointType {
    AVN_JOINT_FIXED = 0,
    AVN_JOINT_REVOLUTE = 1,
    AVN_JOINT_SPHERICAL = 2,
    AVN_JOINT_PRISMATIC = 3,
    AVN_JOINT_DISTANCE = 4,
    AVN_JOINT_TYPE_COUNT = 5
} AvnJointType;

typedef struct AvnJointColumns {
    uint32_t count;
    uint32_t _pad;
    const int32_t* body1;             /* [J] index into AvnBodyColumns (static bodies need an entry: pose is read) */
    const int32_t* body2;
    const void* local_anchor1;        /* [J][3] */
    const void* local_anchor2;        /* [J][3] */
    const void* local_basis1;         /* [J][4] (unused by Distance); NULL = identity */
    const void* local_basis2;
    const void* axis;                 /* [J][3] hinge_axis / twist_axis / slider_axis; NULL = type default (Z / Y / X) */
    const uint8_t* limit_enabled;     /* [J] bit0: angle_limit | swing_limit | prismatic limits ; bit1: twist_limit.
                                         Distance joints always use limit (min,max). NULL = 0 */
    const void* limit_min;            /* [J] */
    const void* limit_max;            /* [J] */
    const void* limit2_min;           /* [J] spherical twist_limit */
    const void* limit2_max;
    /* compliances, NULL = 0.  meaning per type:
     *   fixed:     c0 point      c1 angle
     *   revolute:  c0 point      c1 align     c2 limit
     *   spherical: c0 point      c1 swing     c2 twist
     *   prismatic: c0 align(pos) c1 angle     c2 limit (unused by the reference solve, kept for layout)
     *   distance:  c0 compliance */
    const void* compliance0;
    const void* compliance1;
    const void* compliance2;
    const uint8_t* damping_enabled;   /* [J] JointDamping present; NULL = none */
    const void* damping_linear;       /* [J] */
    const void* damping_angular;      /* [J] */
    void* force;                      /* [J][3] out: JointForces::force  (xpbd/plugin.rs:242-260); NULL = skip */
    void* torque;                     /* [J][3] out */
} AvnJointColumns;

typedef struct AvnJointSet {
    AvnJointColumns types[AVN_JOINT_TYPE_COUNT];
} AvnJointSet;

/* ---- broad phase: AabbIntervals (broad_phase.rs:176-202), in the PERSISTENT interval order (previous
 *      frame's sorted order, then newly added colliders appended, broad_phase.rs:296-315) -------------- */
typedef struct AvnAabbColumns {
    uint32_t count;                   /* C */
    uint32_t retained_count;          /* out (written by upload and again by download): intervals that stay in the list = entries of order_out.
                                         Intervals whose AABB has a NaN or infinite component are dropped, as update_aabb_intervals' retain
                                         does (broad_phase.rs:243-245): they form no pairs and are absent from order_out */
    const uint32_t* collider;         /* [C] Entity::index() of the collider */
    const uint32_t* body;             /* [C] Entity::index() of ColliderOf::body */
    const void* aabb_min;             /* [C][3] ColliderAabb::min */
    const void* aabb_max;             /* [C][3] */
    const uint32_t* memberships;      /* [C] CollisionLayers; NULL = 1 (default layer) */
    const uint32_t* filters;          /* [C] NULL = 0xFFFFFFFF */
    const uint8_t* flags;             /* [C] AVN_AABB_* */
    uint32_t* order_out;              /* [C] out: new persistent order, as indices into these columns (retained_count entries); NULL = skip */
    /* pairs already in ContactGraph::pair_set (contact_graph.rs:95): PairKey u64, any order */
    const uint64_t* existing_pairs;
    uint64_t existing_pair_count;
    /* body pairs (PairKey of body Entity::index()) whose joints disable collision (broad_phase.rs:423-428) */
    const uint64_t* joint_disabled_body_pairs;
    uint64_t joint_disabled_pair_count;
} AvnAabbColumns;

typedef struct AvnPairList {
    uint64_t capacity;                /* in: elements available in each array below */
    uint64_t count;                   /* out: pairs found (may exceed capacity -> AVN_ERR_CAPACITY, arrays hold the prefix) */
    uint32_t* collider1;              /* [capacity] out: Entity::index() (i before j in the sorted order) */
    uint32_t* collider2;
    uint32_t* body1;
    uint32_t* body2;
    uint8_t* flags;                   /* AVN_PAIR_* */
} AvnPairList;

/* Device-time per phase in milliseconds of the last avn_solver_step / avn_broadphase call, named after
 * SolverDiagnostics (src/dynamics/solver/diagnostics.rs:13-39) and CollisionDiagnostics (collision/diagnostics.rs:13-20). */
typedef struct AvnTimings {
    float h2d_ms;
    float prepare_ms;          /* prepare_solver_bodies + prepare_joints + prepare_constraints + update_velocity_increments */
    float substep_loop_ms;     /* integrate_velocities .. joint damping, all substeps */
    float finalize_ms;         /* apply_restitution + finalize + store_impulses */
    float d2h_ms;
    float broad_phase_ms;
    float total_ms;
    uint32_t kernel_launches;  /* kernels launched by the last call */
    uint32_t contact_constraint_count;
    uint32_t joint_levels;
    uint32_t active_colors;
    uint32_t launch_mode;      /* AVN_LAUNCH_*: how the last solver stage was launched (a refused cooperative launch falls back to phases) */
} AvnTimings;
#define AVN_LAUNCH_PHASES 0u        /* one kernel launch per phase (~500 per step) */
#define AVN_LAUNCH_MEGA_BARRIER 1u  /* one persistent cooperative kernel, grid barriers between colours */
#define AVN_LAUNCH_MEGA_WAVE 2u     /* one persistent cooperative kernel, per-body event counters instead of barriers */

/* lifecycle ------------------------------------------------------------------------------------------- */
AvnStatus avn_create(const AvnConfig* config, AvnContext** out_ctx);
void avn_destroy(AvnContext* ctx);
const char* avn_last_error(const AvnContext* ctx); /* ctx may be NULL: error of the last failed avn_create */
uint32_t avn_abi_version(void);

/* pinned host memory for the column buffers */
AvnStatus avn_alloc_pinned(AvnContext* ctx, size_t bytes, void** out_ptr);
AvnStatus avn_free_pinned(AvnContext* ctx, void* ptr);

/*
 * One full solver stage of a physics step.  Replaces, in order:
 *   prepare_solver_bodies (solver_body/plugin.rs:173-251), prepare_xpbd_joint<T> x5 (xpbd/plugin.rs:125-142),
 *   update_contact_softness + prepare_contact_constraints (solver/plugin.rs:326-448),
 *   pre_process_velocity_increments (integrator/mod.rs:260-313),
 *   run_substep_schedule (solver/schedule.rs:194-213): integrate_velocities, clamp_velocities, warm_start,
 *     solve_contacts<true>, integrate_positions, solve_contacts<false>, solve_xpbd_joint<T> x5,
 *     project_linear/angular_velocity, joint_damping<T> x5,
 *   solve_restitution (solver/plugin.rs:630-718), writeback_solver_bodies (solver_body/plugin.rs:255-284),
 *   writeback_joint_forces (xpbd/plugin.rs:242-260), store_contact_impulses (solver/plugin.rs:722-755).
 * Host buffers in, host buffers out (copies are inside the call).  manifolds / joints may be NULL.
 */
AvnStatus avn_solver_step(AvnContext* ctx, const AvnStepParams* params, AvnBodyColumns* bodies,
                          AvnManifoldColumns* manifolds, AvnJointSet* joints);

/* The same stage split in three so a caller can keep the snapshot resident in HBM:
 *   upload (H2D only) -> run (kernels only, repeatable: every run restarts from the uploaded snapshot)
 *   -> download (D2H of the last run's results into the column buffers given to upload). */
AvnStatus avn_solver_upload(AvnContext* ctx, const AvnStepParams* params, AvnBodyColumns* bodies,
                            AvnManifoldColumns* manifolds, AvnJointSet* joints);
AvnStatus avn_solver_run(AvnContext* ctx);
AvnStatus avn_solver_download(AvnContext* ctx);

/* ---- one coupled scene over several GPUs: the x-slab partition (SURVEY.md 8e, BASELINE north_star "single all-gather of boundary
 *      state per substep where the scene spans GPUs").  Not a reference interface: the reference is single-process. -------------
 * Each rank uploads its own bodies and constraints plus copies ("ghosts") of the remote bodies its constraints touch.  A body held
 * by more than one rank is a BOUNDARY body; it has one slot in a table every rank agrees on.  Per substep each rank launches
 * avn_solver_run_range for that substep, packs for every boundary body it holds the velocity change its own constraints caused
 * (relative to the velocity right after integrate_velocities, which every holder computes identically) and, if it owns the body,
 * the body's delta_position / delta_rotation, into its own packed table (one record per held boundary body); the tables are all-gathered (NCCL, by the caller, on the stream avn_get_stream
 * returns); avn_solver_boundary_apply sets v = v_ref + sum over ranks in rank order of their changes and takes the owner's deltas.
 * Impulses therefore cross a cut once per substep instead of once per constraint: results match the single-GPU step to solver
 * tolerance, not to 1e-5; a scene whose constraints do not cross a cut is reproduced bit for bit. */
#define AVN_RUN_PREPARE 0x1u      /* prepare bodies / constraints: must be part of the first launch after an upload */
#define AVN_RUN_RESTITUTION 0x2u  /* solve_restitution after the substeps of this launch */
#define AVN_RUN_FINALIZE 0x4u     /* writeback_solver_bodies + store_contact_impulses: must be part of the last launch */

typedef struct AvnBoundary {
    uint32_t count;               /* boundary bodies held by this rank: record k of this rank's table belongs to body[k] */
    uint32_t record_count;        /* records per rank's table = the largest `count` of any rank (all-gather needs equal sizes) */
    uint32_t rank, world;
    const int32_t* body;          /* [count] index into the uploaded AvnBodyColumns */
    const int32_t* source;        /* [count][world] record of body[k] in rank r's table, or -1 when rank r does not hold it */
    const int32_t* owner_rank;    /* [count] the rank whose delta_position / delta_rotation are authoritative */
} AvnBoundary;
/* scalars per record of the exchange table (4 rows of 4): a table is record_count * AVN_BOUNDARY_RECORD_SCALARS scalars,
 * the gathered tables world times that, rank-major.  Only held bodies travel: the table is as large as the busiest rank's list. */
#define AVN_BOUNDARY_RECORD_SCALARS 16

AvnStatus avn_solver_run_range(AvnContext* ctx, uint32_t first_substep, uint32_t substep_count, uint32_t run_flags);
AvnStatus avn_solver_set_boundary(AvnContext* ctx, const AvnBoundary* boundary);   /* after upload; NULL / count 0 clears it */
AvnStatus avn_solver_boundary_snapshot(AvnContext* ctx);                           /* v_ref = current velocity (before a restitution launch) */
AvnStatus avn_solver_boundary_pack(AvnContext* ctx, void* device_table);           /* DEVICE pointer */
AvnStatus avn_solver_boundary_apply(AvnContext* ctx, const void* device_gathered); /* DEVICE pointer */
AvnStatus avn_solver_needs_restitution(AvnContext* ctx, int* out_nonzero);         /* any uploaded restitution coefficient != 0 */
/* the context's CUDA stream (a cudaStream_t) so that the caller's collective can be ordered with the launches above */
AvnStatus avn_get_stream(AvnContext* ctx, void** out_stream);

/* ---- the communicator: one process per GPU, one AvnContext per process, one NCCL communicator per context (SURVEY.md 8b).  NCCL is bound
 *      at run time (dlopen "libnccl.so.2", or the name in AVN_NCCL_LIB): a host that never calls avn_comm_init with world > 1 needs no NCCL.
 *      One rank calls avn_comm_unique_id and hands the AVN_COMM_ID_BYTES bytes to the others over any channel the host has (a file, a socket,
 *      MPI, torch.distributed's store); then EVERY rank calls avn_comm_init with the same bytes (collective).  Errors: AVN_ERR_NCCL. */
#define AVN_COMM_ID_BYTES 128
AvnStatus avn_comm_unique_id(AvnContext* ctx, void* out_id /* [AVN_COMM_ID_BYTES] */);
AvnStatus avn_comm_init(AvnContext* ctx, uint32_t rank, uint32_t world, const void* unique_id /* NULL allowed when world == 1 */);
AvnStatus avn_comm_destroy(AvnContext* ctx);
/* all-gather of bytes_per_rank bytes of DEVICE memory from every rank into recv_device (world * bytes_per_rank, rank-major), enqueued on the
 * context's stream (pair lists of the slab broad phase, results of the owned rows) */
AvnStatus avn_comm_all_gather(AvnContext* ctx, const void* send_device, void* recv_device, size_t bytes_per_rank);
/*
 * The whole partitioned solver stage of this rank, inside the library: after avn_solver_upload (this rank's share) and
 * avn_solver_set_boundary, runs for every substep  avn_solver_run_range -> pack -> ncclAllGather of the packed tables -> apply  on the
 * context's stream, the restitution launch + one more exchange when any rank uploaded a non-zero coefficient (agreed with one all-reduce),
 * and the finalize launch.  Follow with avn_solver_download.  With a communicator of one rank (or no boundary) it equals avn_solver_run.
 * The exchange tables live in the library; nothing crosses the host.
 */
AvnStatus avn_solver_step_partitioned(AvnContext* ctx);

/*
 * Sweep-and-prune pair generation.  Replaces collect_collision_pairs / sweep_and_prune (broad_phase.rs:343-474)
 * over the intervals that update_aabb_intervals / add_new_aabb_intervals maintain (broad_phase.rs:214-315).
 * The emitted list is exactly the sequence of ContactGraph::add_edge_and_key_with calls the reference makes
 * (same pairs, same order); pairs flagged AVN_PAIR_NEEDS_HOOK still need the host filter_pairs callback.
 */
AvnStatus avn_broadphase(AvnContext* ctx, AvnAabbColumns* aabbs, AvnPairList* out_pairs);
/* split form: the AvnAabbColumns struct itself (not only its buffers) must stay valid until avn_broadphase_download returns */
AvnStatus avn_broadphase_upload(AvnContext* ctx, AvnAabbColumns* aabbs);
AvnStatus avn_broadphase_run(AvnContext* ctx);
AvnStatus avn_broadphase_download(AvnContext* ctx, AvnPairList* out_pairs);

/* ---- collider AABBs (SURVEY.md 8f "next #2"): update_aabb for the shapes the device knows ------------------------------- */
/* AVN_SHAPE_CAPSULE: Collider::capsule(radius, length), dims = [radius, length / 2, unused]; the segment runs from (0, -length/2, 0) to
 * (0, +length/2, 0) in the collider frame.  The AABB update, the narrow phase, the contact store, the spatial queries (colliders and query
 * shapes), move and slide (obstacles and characters) and swept CCD (with AVN_CCD_CAPSULES) take capsules.
 * AVN_SHAPE_CONVEX_HULL: Collider::convex_hull / the parts of Collider::convex_decomposition, dims = [hull index, unused, unused] into the
 * context's hull table (avn_set_convex_hulls).  The index is stored in the column scalar: integral, non-negative and below the table's hull
 * count.  The AABB update, the narrow phase, the contact store, the spatial queries (colliders and query shapes) and move and slide (obstacles
 * and characters) and swept CCD (with AVN_CCD_HULLS) take hulls. */
typedef enum AvnShape { AVN_SHAPE_CUBOID = 0, AVN_SHAPE_SPHERE = 1, AVN_SHAPE_CAPSULE = 2, AVN_SHAPE_CONVEX_HULL = 3 } AvnShape;

/* ---- convex hulls: the table AVN_SHAPE_CONVEX_HULL colliders index (parry's ConvexPolyhedron: points, faces as vertex loops) ---------- */
#define AVN_HULL_MAX_VERTICES 64u        /* per hull; the device kernels' fixed buffers are sized from these three */
#define AVN_HULL_MAX_FACES 128u          /* per hull */
#define AVN_HULL_MAX_FACE_VERTICES 32u   /* per face loop */
#define AVN_HULL_MAX_COUNT (1u << 24)    /* hulls per table: every index is exact in an f32 dims column */
/* The relative tolerance of the table checks: a face is planar, and a hull convex, when no vertex lies more than
 * AVN_HULL_REL_TOL * size above a face plane (size = the diagonal of the hull's local vertex box); a face's area must exceed
 * (AVN_HULL_REL_TOL * size)^2, and the vertex mean must lie more than AVN_HULL_REL_TOL * size below every face plane. */
#define AVN_HULL_REL_TOL 1e-6
typedef struct AvnConvexHulls {
    uint32_t hull_count, _pad;
    const uint32_t* vertex_offsets;    /* [hull_count + 1] CSR into vertices */
    const void* vertices;              /* [V][3] column scalar, hull-local and already scaled (Collider::shape_scaled) */
    const uint32_t* face_offsets;      /* [hull_count + 1] CSR into the faces (loop_offsets' rows) */
    const uint32_t* loop_offsets;      /* [F + 1] CSR into loop */
    const uint32_t* loop;              /* [L] hull-local vertex indices, each face counter-clockwise seen from outside */
} AvnConvexHulls;
/* Checks the table on the host and, when it is accepted, derives in double (face normals by Newell's method, plane offsets, the unique
 * edges with the two faces each separates, each hull's vertex mean and bounding radius) and uploads it; every later avn_update_aabbs,
 * avn_narrow_phase and avn_contacts_step of the context reads it.  NULL clears the table.  AVN_ERR_INVALID_ARGUMENT, before anything is
 * stored (a refused call changes nothing), for: missing columns, more than AVN_HULL_MAX_COUNT hulls, decreasing offsets, a vertex index out
 * of range, more than AVN_HULL_MAX_VERTICES vertices, AVN_HULL_MAX_FACES faces or AVN_HULL_MAX_FACE_VERTICES vertices on one face, a face
 * loop of fewer than 3 or with a repeated vertex, two coincident vertices, an open or non-manifold surface (every directed edge once and its
 * reverse once, V - E + F = 2), a zero-area, non-planar or inward-wound face, and a non-convex hull (tolerances: AVN_HULL_REL_TOL).
 * A shape column that names a hull while no table is set, or an index at or past the hull count, is AVN_ERR_INVALID_ARGUMENT from
 * avn_update_aabbs, avn_narrow_phase and avn_contacts_step, before anything is copied. */
AvnStatus avn_set_convex_hulls(AvnContext* ctx, const AvnConvexHulls* hulls);

typedef struct AvnAabbParams {
    double dt;                         /* Time::delta (full step, collider/backend.rs:536) */
    double contact_tolerance;          /* PhysicsLengthUnit * NarrowPhaseConfig::contact_tolerance (default 0.005) */
    double default_speculative_margin; /* PhysicsLengthUnit * NarrowPhaseConfig::default_speculative_margin (default Scalar::MAX: pass +inf) */
} AvnAabbParams;

typedef struct AvnColliderColumns {
    uint32_t count;
    uint32_t _pad;
    const uint8_t* shape;              /* [C] AvnShape */
    const void* dims;                  /* [C][3] cuboid half extents / sphere radius in [0] / capsule [radius, half length] (scaled shape) */
    const void* position;              /* [C][3] collider Position */
    const void* rotation;              /* [C][4] collider Rotation */
    const void* linear_velocity;       /* [C][3] the velocity update_aabb uses: the collider's own LinearVelocity, or its body's velocity at
                                          the collider offset (backend.rs:560-580); NULL = 0 */
    const void* angular_velocity;      /* [C][3] NULL = 0 */
    const void* collision_margin;      /* [C] CollisionMargin; NULL = 0 */
    const void* speculative_margin;    /* [C] SpeculativeMargin (+inf for SweptCcd); NULL = the default */
    void* aabb_min;                    /* [C][3] out: ColliderAabb::min */
    void* aabb_max;                    /* [C][3] out */
} AvnColliderColumns;

/*
 * Replaces update_aabb::<Collider> (src/collision/collider/backend.rs:498-625) for cuboid, sphere and capsule colliders: swept AABB from the
 * current pose to the pose after dt (rotation advanced by Quat::from_scaled_axis + fast_renormalize, translation clamped to the
 * speculative margin), grown by contact_tolerance + collision margin.  AVN_ERR_INVALID_ARGUMENT, before anything is computed, for a shape
 * above AVN_SHAPE_CONVEX_HULL, a capsule with a negative radius or half length, or a hull index the table does not hold (avn_narrow_phase
 * and avn_contacts_step check the same).  A hull's AABB is parry's ConvexPolyhedron::aabb: every vertex moved by the pose, min / max.
 */
AvnStatus avn_update_aabbs(AvnContext* ctx, const AvnAabbParams* params, AvnColliderColumns* colliders);

/* ---- contact manifolds, the stand-alone geometry stage (SURVEY.md 8f "next #1"): one manifold of at most 4 points per listed pair of
 *      cuboid / sphere colliders.  Stands where NarrowPhase::update calls contact_manifolds (narrow_phase/system_param.rs:437-830,
 *      collider/parry/contact_query.rs:156-261); the arithmetic is this repository's generator (csrc/narrow_math.hpp — parry3d is not
 *      vendored), shared with the host fixture.  avn_contacts_step runs the same geometry on the rows of the contact store. -------------- */
typedef struct AvnNarrowParams {
    double dt;                         /* Time::delta (narrow_phase/mod.rs:289) */
    double contact_tolerance;          /* PhysicsLengthUnit * NarrowPhaseConfig::contact_tolerance */
} AvnNarrowParams;

typedef struct AvnNarrowInput {
    uint32_t pair_count, collider_count, body_count, _pad;
    const uint32_t* collider1;         /* [pairs] row of the collider columns below (avn_contacts_step ignores the pair arrays) */
    const uint32_t* collider2;
    const uint32_t* body1;             /* [pairs] row of the body velocity columns */
    const uint32_t* body2;
    const uint8_t* shape;              /* [C] AvnShape; NULL = cuboid */
    const void* dims;                  /* [C][3] cuboid half extents / sphere radius in [0] / capsule [radius, half length] */
    const void* position;              /* [C][3] collider Position (world pose; without body frames a collider sits at its body's origin and
                                          the centre of mass at that origin, see avn_contacts_set_body_frames) */
    const void* rotation;              /* [C][4] */
    const void* linear_velocity;       /* [B][3] */
    const void* angular_velocity;      /* [B][3] */
    const void* aabb_min;              /* [C][3] optional: pairs whose AABBs are disjoint are reported in `disjoint` and skipped */
    const void* aabb_max;
} AvnNarrowInput;

typedef struct AvnRawManifolds {      /* fixed stride: 4 point slots per pair, unused slots zero */
    uint8_t* point_count;              /* [pairs] 0..4 (0 = not touching within the speculative margin) */
    uint8_t* disjoint;                 /* [pairs] optional */
    void* normal;                      /* [pairs][3] from collider1 to collider2 */
    void* anchor1;                     /* [pairs][4][3] */
    void* anchor2;
    void* penetration;                 /* [pairs][4] */
    void* normal_speed;                /* [pairs][4] */
} AvnRawManifolds;

AvnStatus avn_narrow_phase(AvnContext* ctx, const AvnNarrowParams* params, const AvnNarrowInput* input, AvnRawManifolds* out);

/* ---- body frames: several colliders per body, offset from the body origin, with the centre of mass off the origin (ColliderOf,
 *      ComputedCenterOfMass).  With frames set, avn_narrow_phase and avn_contacts_step return anchors relative to each body's centre of mass,
 *      as update_contacts does (narrow_phase/system_param.rs:540-570, 731-747):
 *        anchor = (witness relative to the collider + (collider position - body position)) - body rotation * center_of_mass
 *      and take the normal speed, the speculative keep rule and match_contacts from those anchors.  The input's position / rotation stay the
 *      colliders' world poses, and body1 / body2 (or the contact store's rows) name the bodies. -------------------------------------------- */
typedef struct AvnBodyFrames {
    uint32_t body_count, _pad;         /* must equal AvnNarrowInput::body_count of the calls that use the frames */
    const void* position;              /* [B][3] body Position: the origin the collider offsets are measured from */
    const void* rotation;              /* [B][4] body Rotation */
    const void* center_of_mass;        /* [B][3] ComputedCenterOfMass, local; NULL = 0 */
} AvnBodyFrames;
/* Copies the frames on the host; every later avn_contacts_step / avn_narrow_phase of the context uses them until the next call.  NULL (or
 * never called) = a collider at its body's origin and the centre of mass at that origin, bit for bit as before.  Static bodies need a frame
 * too: a static side's anchor enters initial_separation.  AVN_ERR_INVALID_ARGUMENT without position or rotation; a call that uses the frames
 * refuses an input whose body_count differs, before anything is copied.  AVN_ERR_UNSUPPORTED while swept CCD is configured: swept CCD
 * assumes a collider at its body's origin, so avn_ccd_configure refuses a configuration while frames are set, and the two never meet.
 * A refused call changes nothing. */
AvnStatus avn_contacts_set_body_frames(AvnContext* ctx, const AvnBodyFrames* frames);

/* ---- the ContactGraph and the ConstraintGraph on the device (SURVEY.md 8f "next #3"): after this nothing of the contact pipeline lives on
 *      the host.  Replaces, for the pairs the device narrow phase covers,
 *        ContactGraph::add_edge_and_key_with          (collision/contact_types/contact_graph.rs:521-565; ids: data_structures/id_pool.rs:43-52)
 *        the status-change loop of NarrowPhase::update (collision/narrow_phase/system_param.rs:136-389: removal of separated pairs,
 *                                                       started / stopped touching)
 *        ConstraintGraph::push_manifold / pop_manifold (dynamics/solver/constraint_graph.rs:163-296)
 *      with the reference's results: the same ContactId for every pair, the same colour for every manifold (the greedy colouring is
 *      order dependent; the device reproduces the sequential order with a dependency wavefront, csrc/contacts.cu).  The order of the
 *      manifolds INSIDE a colour is ascending ContactId instead of the reference's swap_remove order — it does not influence the solve;
 *      the overflow colour, which is solved serially, keeps the reference's list order. ------------------------------------------------ */
typedef struct AvnContactGraphConfig {
    uint32_t body_count, collider_count;
    const uint8_t* body_kind;          /* [B] AvnBodyKind: static bodies never enter a colour's body set */
    const double* friction;            /* [C] per collider; a pair's coefficient is the mean of its colliders' (NULL = 0.5) */
    const double* restitution;         /* [C] (NULL = 0) */
} AvnContactGraphConfig;
AvnStatus avn_contacts_configure(AvnContext* ctx, const AvnContactGraphConfig* config);

typedef struct AvnContactStep {
    uint32_t rows_high_water;          /* ContactIds in use: [0, rows_high_water) */
    uint32_t rows_live;                /* pairs in the ContactGraph after this step */
    uint32_t pairs_added, pairs_removed, started_touching, stopped_touching;
    uint32_t manifold_count;           /* manifolds in the ConstraintGraph = length of the colour-major list */
    uint32_t colouring_rounds;         /* dependency levels the greedy colouring needed this step */
    uint32_t any_restitution;
    uint32_t _pad;
    uint32_t color_offsets[AVN_GRAPH_COLOR_COUNT + 1];
} AvnContactStep;
#define AVN_CONTACTS_TAKE_BROADPHASE_PAIRS 0x1u   /* add the new pairs of the context's last avn_broadphase_run (read in device memory) */
#define AVN_CONTACTS_SHAPES_UNCHANGED 0x2u        /* input->shape and input->dims equal the previous call's: not copied again (nor checked) */
/* One step of the contact pipeline on the device: (new pairs ->) rows, geometry + match_contacts for every live row, the status loop, the
 * graphs, the colour-major list.  input: the collider / body columns of AvnNarrowInput (pair arrays ignored).  From the first call on the
 * contact store's pair set is the broad phase's "existing pairs" set (AvnAabbColumns::existing_pairs may stay NULL). */
AvnStatus avn_contacts_step(AvnContext* ctx, const AvnNarrowParams* params, const AvnNarrowInput* input, uint32_t match_contacts, double length_unit,
                            uint32_t flags, AvnContactStep* out);
/* The solver stage fed entirely from the device: manifolds from the contact rows, the constraint graph from the last avn_contacts_step.
 * Then avn_solver_run / avn_solver_download (bodies only) as usual. */
AvnStatus avn_solver_upload_resident(AvnContext* ctx, const AvnStepParams* params, AvnBodyColumns* bodies, AvnJointSet* joints);
/* Optional, any pipeline: start copying the body columns of the NEXT avn_solver_upload* / avn_solver_step call to the device now, on a second
 * stream, so that the copy overlaps the stages that run before the solver (broad phase, contact pipeline).  The next upload must be given the
 * same column pointers (otherwise it simply copies again); the host columns must not change in between.
 * AVN_BODIES_STATIC_UNCHANGED: the columns that describe the bodies (kind, locked_axes, dominance, integration_flags, inverse_mass,
 * inverse_inertia_local, center_of_mass, dampings, gravity_scale, max speeds) equal those of the previous upload of the same number of
 * bodies; only position, rotation, velocities and accelerations are copied. */
#define AVN_BODIES_STATIC_UNCHANGED 0x1u
AvnStatus avn_solver_prefetch_bodies(AvnContext* ctx, AvnBodyColumns* bodies, uint32_t flags);
/* After avn_broadphase_run in the device-resident pipeline: waits for the run, writes order_out / retained_count of the uploaded columns and
 * returns the number of new pairs; the pairs themselves stay on the device for avn_contacts_step. */
AvnStatus avn_broadphase_download_order(AvnContext* ctx, uint64_t* out_pair_count);
/* the graphs as the device holds them (tests, tools): per row [capacity] colliders, live / touching flags, colour (-1 = not in the
 * constraint graph); edge_list [manifold_count] = the colour-major list.  Any pointer may be NULL. */
AvnStatus avn_contacts_download_graph(AvnContext* ctx, uint32_t capacity, uint32_t* collider1, uint32_t* collider2, uint8_t* live, uint8_t* touching,
                                      int8_t* colour, uint32_t* edge_list);
/* the impulses of the rows as the last solve left them (tests, tools), in the context's scalar type: per row [capacity][4] warm-start normal,
 * [capacity][4][2] warm-start tangent, [capacity][4] normal impulse; min(capacity, rows) rows are written.  Any pointer may be NULL. */
AvnStatus avn_contacts_download_impulses(AvnContext* ctx, uint32_t capacity, void* warm_start_normal, void* warm_start_tangent, void* normal_impulse);

/* ---- the contact pipeline's output to the application: collision events, sensors, removal of colliders, contact reports.  All of it works on
 *      the ContactGraph of avn_contacts_step; before the first avn_contacts_step of the context (before avn_contacts_configure for
 *      avn_contacts_set_sensors) these calls return AVN_ERR_UNSUPPORTED.  Nothing changes for a caller that never makes them.
 *      Lists use the capacity protocol of the hit lists: on AVN_ERR_CAPACITY `count` is the required size and nothing else was written.
 *      Stated deviation: inside one removal call the rows of the removed colliders are visited in ascending ContactId, where the reference walks
 *      the collider's edge list (the order of the queued CollisionEnds and of the overflow colour's swap_removes). -------------------------- */
typedef struct AvnCollisionEvents {   /* CollisionStart / CollisionEnd (collision/collision_events.rs:171, :268) */
    uint64_t capacity;                 /* in: entries the arrays hold */
    uint64_t count;                    /* out: entries of the list (AVN_ERR_CAPACITY when > capacity) */
    uint32_t* collider1;               /* [capacity] out; any array may be NULL (not wanted) */
    uint32_t* collider2;
    uint32_t* body1;
    uint32_t* body2;
    uint8_t* flags;                    /* the pair's AVN_PAIR_* flags: CONTACT_EVENTS = an events-enabled pair, GENERATE_CONSTRAINTS clear = a sensor pair */
} AvnCollisionEvents;

typedef struct AvnContactReport {     /* one entry per touching pair, ascending ContactId; scalars in the context's type; any array may be NULL */
    uint64_t capacity;
    uint64_t count;
    uint32_t* contact_id;
    uint32_t* collider1;
    uint32_t* collider2;
    uint32_t* body1;
    uint32_t* body2;
    uint8_t* flags;                    /* AVN_PAIR_* */
    uint8_t* point_count;
    void* normal;                      /* [n][3] manifold normal, from collider1 to collider2 */
    void* total_normal_impulse;        /* ContactManifold::total_normal_impulse: the points' normal_impulse summed in slot order */
    void* max_normal_impulse;          /* ContactManifold::max_normal_impulse (0 when no point) */
    void* max_penetration;             /* penetration of find_deepest_contact (contact_types/mod.rs:318-327) */
} AvnContactReport;
#define AVN_REPORT_EVENTS_ONLY 0x1u   /* only pairs with AVN_PAIR_CONTACT_EVENTS */

/* The Sensor column (Collider::is_sensor): a row generates constraints only when its broad-phase flags do and neither collider is a sensor
 * (narrow_phase/system_param.rs:583-599).  Sensor rows are narrow-phased, touch, produce events and appear in reports (with zero impulses); they
 * never take a colour and never link islands.  Plays the On<Add, Sensor> / On<Remove, Sensor> observers (narrow_phase/mod.rs:614-668): every
 * collider whose flag changed goes through remove_collider at once, and the next broad phase finds its pairs again with the new flags.  A call
 * before any row exists only stores the column.  sensor: [collider_count], NULL = none; collider_count must equal avn_contacts_configure's
 * (AVN_ERR_INVALID_ARGUMENT otherwise).  avn_contacts_configure clears the column. */
AvnStatus avn_contacts_set_sensors(AvnContext* ctx, uint32_t collider_count, const uint8_t* sensor);
/* remove_collider (narrow_phase/mod.rs:399-459) for each listed collider, on the device, now: every live row that names one of them queues a
 * CollisionEnd when it was touching, leaves its colour (the overflow colour keeps its swap_remove order), applies remove_contact to its island
 * when it was a touching, constraint-generating contact and islands are configured (islands/mod.rs:594-667), and is freed.  The colour-major
 * list, the colour offsets and the pair set are rebuilt: avn_solver_upload_resident and the next broad phase see the new graph.  Despawned
 * colliders, ColliderDisabled.  A collider >= the configured count is AVN_ERR_INVALID_ARGUMENT and nothing is removed.  Waking the islands of
 * the removed collider's body stays with the caller (AvnIslandsStep::wake). */
AvnStatus avn_contacts_remove_colliders(AvnContext* ctx, uint32_t n, const uint32_t* colliders);
/* The collision events of the last avn_contacts_step; repeatable until the next step.  Every transition is listed with its pair flags, events
 * enabled or not: the caller writes CollisionStart / CollisionEnd for the AVN_PAIR_CONTACT_EVENTS entries and updates CollidingEntities from all
 * of them (system_param.rs:155-321).
 *   started: rows that started touching, ascending ContactId (the order of the reference's status loop);
 *   ended:   first the CollisionEnds of the removals since the previous step (touching rows, call order), then the rows that stopped touching
 *            or whose AABBs separated while touching, ascending ContactId.
 * Either list may be NULL. */
AvnStatus avn_contacts_events(AvnContext* ctx, AvnCollisionEvents* started, AvnCollisionEvents* ended);
/* ContactPair::total_normal_impulse / max_normal_impulse (contact_types/mod.rs:227-277) of the touching pairs as the last solve left them:
 * call it after avn_solver_run.  Geometry from this step's narrow phase, impulses from store_contact_impulses (solver/plugin.rs:722-754).  A row
 * that was not solved this step (a sensor pair) reports 0 impulses, as the reference's fresh points do; a row that is asleep
 * (avn_islands_apply) is listed with the impulses of its last solve.  flags: AVN_REPORT_*. */
AvnStatus avn_contacts_report(AvnContext* ctx, uint32_t flags, AvnContactReport* out);

/* ---- simulation islands and sleeping on the device (SURVEY.md 8f "next #4").  Replaces the bookkeeping and the decisions of
 *        PhysicsIslands::add_contact / remove_contact / add_joint / merge_islands / split_island   (dynamics/solver/islands/mod.rs:513-1270)
 *        update_sleeping_states, wake_islands_with_sleeping_disabled, sleep_islands                 (dynamics/solver/islands/sleeping.rs:164-292)
 *      Islands are PERSISTENT like the reference's: merged when a touching, constraint-generating contact (or a joint) links two of them,
 *      marked (constraints_removed) when such a contact goes, and split lazily — one island per step, the one holding the sleepiest body
 *      that wants to sleep — by recomputing its connected components.  The contact events come from the last avn_contacts_step of this
 *      context (the rows on the device); the body velocities are the solver's results of the same step.  Output: island label and Sleeping
 *      flag per body.  APPLYING a decision is opt-in (avn_islands_apply below): the library then plays the SleepIslands / WakeIslands commands
 *      on its own rows, graphs and solver stage, and the shim only mirrors the flags (`Sleeping` component, AVN_AABB_IS_INACTIVE).
 *      One deviation, stated: the reference tracks the split candidate as an island id that a merge can retire (when the candidate is the
 *      smaller island of the merge); here the candidate is the sleepiest BODY, and the island that holds it one step later is split. -------- */
typedef struct AvnIslandsConfig {
    uint32_t body_count, joint_count;
    const uint8_t* body_kind;            /* [B] AvnBodyKind: static bodies have no island */
    const float* sleep_threshold_linear; /* [B] SleepThreshold::linear  (NULL = 0.15; negative = never sleeps) */
    const float* sleep_threshold_angular;/* [B] SleepThreshold::angular (NULL = 0.15) */
    const uint8_t* sleeping_disabled;    /* [B] SleepingDisabled marker (NULL = none) */
    const uint32_t* joint_body1;         /* [J] bodies linked by joints (PhysicsIslands::add_joint) */
    const uint32_t* joint_body2;
    float time_to_sleep;                 /* TimeToSleep (default 0.5 s) */
    float length_unit;                   /* PhysicsLengthUnit */
} AvnIslandsConfig;
/* Islands start as one per non-static body, linked by the joints and — when the contact store already holds touching pairs — by those. */
AvnStatus avn_islands_configure(AvnContext* ctx, const AvnIslandsConfig* config);

typedef struct AvnIslandsStep {
    float delta_secs;                    /* in: Time::delta_secs of the step */
    uint32_t _pad;
    const void* linear_velocity;         /* in: [B][3] SolverBody velocities after the solve (column scalar type) */
    const void* angular_velocity;        /* in: [B][3] */
    const uint8_t* wake;                 /* in: [B] optional: bodies the application touched (wake_on_changed): their islands wake up */
    uint32_t* island;                    /* out: [B] island label = smallest body index of the island (0xFFFFFFFF for static bodies); NULL = skip */
    uint8_t* sleeping;                   /* out: [B] 1 = the body's island sleeps; NULL = skip */
    float* sleep_timer;                  /* out: [B] SleepTimer; NULL = skip */
    uint32_t island_count, sleeping_islands, islands_put_to_sleep, islands_woken, split_bodies, merges;   /* out */
} AvnIslandsStep;
/* Once per step, after avn_contacts_step and the solver stage of the same step (it consumes that step's contact events). */
AvnStatus avn_islands_step(AvnContext* ctx, AvnIslandsStep* step);

/* ---- applying sleeping and waking on the device (SleepIslands::apply / WakeIslands::apply, islands/sleeping.rs:354-533; opt-in).
 *      State: one `asleep` byte per contact row and one per body.  When an island is put to sleep every touching row of its bodies leaves the
 *      ConstraintGraph (ContactGraph::sleep_entity_with, contact_graph.rs:765-826) and keeps its manifold, matched anchors and impulses
 *      untouched: avn_contacts_step neither narrow-phases nor classifies an asleep row, so it produces no event.  A body that is asleep enters the
 *      solver stage of avn_solver_upload_resident as AVN_BODY_STATIC (no SolverBody: not integrated, not written back; its velocities stay as
 *      they are — the reference does not zero them either).  When the island wakes the rows are pushed back (wake_entity_with, :702-763) and
 *      the solve warm-starts from the impulses of the last solve before the sleep.  An edge follows EITHER endpoint, as in the reference: a
 *      touching sensor pair between a sleeping body and an awake body of another island sleeps with the first and is not updated until one of
 *      the two islands wakes.  avn_contacts_report lists asleep rows with the impulses of their last solve; avn_contacts_remove_colliders and
 *      avn_contacts_set_sensors remove them like any other row.  The broad phase is not changed: the caller sets AVN_AABB_IS_INACTIVE on the
 *      intervals of the bodies whose `sleeping` flag the last avn_islands_step returned.
 *      Stated deviations: woken rows are pushed, and rows put to sleep leave the overflow colour, in ascending ContactId (the reference walks each
 *      island's body list and each collider's edge list).  The colouring is the sequential greedy result for that order and conflict-free,
 *      but after a wake a manifold may hold another colour than in the reference, and the colours are the Gauss-Seidel order.
 *      Order of one step:  avn_contacts_step -> avn_islands_wake -> avn_solver_upload_resident / run / download -> avn_islands_step. -------- */
/* enable != 0: from now on the decisions are applied.  AVN_ERR_UNSUPPORTED before avn_islands_configure (whose body count must equal
 * avn_contacts_configure's) and while avn_ccd_configure holds a body list (avn_ccd_configure is refused the same way while application is on).
 * enable == 0: every sleeping island is woken first, then the context behaves as if the call had never been made; only between steps
 * (AVN_ERR_INVALID_ARGUMENT between avn_contacts_step and the avn_islands_step that ends the step).
 * While application is on avn_contacts_configure and avn_islands_configure return AVN_ERR_UNSUPPORTED: turn it off, reconfigure, turn it on. */
AvnStatus avn_islands_apply(AvnContext* ctx, uint32_t enable);

typedef struct AvnIslandsWake {
    uint32_t islands_woken;              /* islands woken by this call */
    uint32_t rows_woken;                 /* contact rows that left the sleeping set */
    uint32_t rows_asleep, bodies_asleep; /* now */
    uint32_t manifold_count;             /* of the list the solver will read */
    uint32_t colouring_rounds;           /* of the woken rows' pushes; 0 when no island woke (the list is avn_contacts_step's) */
    uint32_t color_offsets[AVN_GRAPH_COLOR_COUNT + 1];   /* the colour-major list as the solver will read it (AvnContactStep's values are stale after a wake) */
} AvnIslandsWake;
/* The narrow-phase half of the island step (system_param.rs:253-258 queues WakeIslands, applied before the solver of the same step): links the
 * islands of the contacts that started touching, wakes the sleeping islands they reach and the islands of the bodies marked in `wake`
 * ([B] or NULL), and pushes the woken islands' rows after the step's own changes.  Once per step between avn_contacts_step and
 * avn_solver_upload_resident, which returns AVN_ERR_INVALID_ARGUMENT when application is on and this call was skipped.  avn_islands_step then
 * skips what was done here.  AVN_ERR_UNSUPPORTED while application is off. */
AvnStatus avn_islands_wake(AvnContext* ctx, const uint8_t* wake, AvnIslandsWake* out);
/* tests, tools: row_asleep [capacity], body_asleep [body_count]; either may be NULL */
AvnStatus avn_contacts_download_sleeping(AvnContext* ctx, uint32_t capacity, uint8_t* row_asleep, uint32_t body_count, uint8_t* body_asleep);

/* ---- spatial queries (SpatialQueryPlugin, src/lib.rs:839; spatial_query/pipeline.rs): a collider tree rebuilt on the device by every
 *      avn_query_update, then batched ray casts and AABB intersection tests against it.  Cuboid, sphere, capsule and convex hull colliders.
 *      The per-shape arithmetic is this repository's own (avian_b200/csrc/query_math.hpp, shared with the host fixture; parry3d is not
 *      vendored), so results equal the host brute force over every collider bit for bit, independent of the tree.  Conventions:
 *        - a ray is origin + t * direction, t in units of |direction| (pass a unit Dir3); a hit counts when 0 <= t <= max_distance;
 *        - shapes are closed; origin inside and solid -> t = 0, normal 0; origin inside and hollow -> the exit, outward normal there;
 *        - cuboid normal: outward normal of the entering face (largest entering slab parameter, ties to the lowest local axis); a direction
 *          component that is exactly 0 leaves its axis unconstrained when the origin is inside that slab and misses otherwise;
 *        - capsule: tight AABB = the posed segment ends' min / max grown by the radius; normal = unit(hit - closest segment point); a
 *          radius-0 capsule is a closed segment (avian_b200/csrc/query_math.hpp, DESIGN.md §7j);
 *        - convex hull (avian_b200/csrc/hull_query_math.hpp, DESIGN.md §7l): tight AABB = the posed vertices' min / max; the ray test,
 *          containment and projection from inside use the table's face planes; normal = the posed face normal of the entering face (largest
 *          entering parameter, ties to the lowest face); the index is checked against the context's hull table (avn_set_convex_hulls) as
 *          avn_contacts_step checks it, a hull without a table is refused, and under AVN_QUERY_SHAPES_UNCHANGED the kept column's largest index
 *          is checked against the current table.  Replacing the table (avn_set_convex_hulls) makes every query and avn_move_and_slide against
 *          a tree that holds a hull fail with AVN_ERR_INVALID_ARGUMENT until the next avn_query_update;
 *        - filter (SpatialQueryFilter::test, query_filter.rs:97-101): (memberships & mask) != 0 and not in the ray's excluded list;
 *        - AABB test: inclusive compares (Aabb::intersects) against the collider's tight AABB (compute_aabb) rounded to the column scalar,
 *          no filter, as pipeline.rs:709-729;
 *        - the rotation is the quaternion's, normalised: the AABB and the ray test see the same box for a quaternion of any nonzero length;
 *        - colliders with a non-finite pose or dims or a zero quaternion are never reported; negative dims are refused; rays with a
 *          non-finite origin, direction or max_distance hit nothing.
 *      Stated deviations: the closest hit is the lexicographic minimum of (t, collider index), where the reference takes the first in tree
 *      order; ray_hits keeps the max_hits NEAREST hits sorted by (t, collider index) — RayHits::iter_sorted order — where the reference keeps
 *      the first max_hits in tree order, unordered (pipeline.rs:213-216); the two sets are equal when a ray has no more than max_hits hits.
 *      Shape casts, point projection and point / shape intersections (cuboid, sphere, capsule and hull query shapes) are further down, with their own
 *      conventions.  Not covered: target_distance != 0, other shapes, predicates and the *_callback early exits, several GPUs. ------------- */
typedef struct AvnQueryColliders {
    uint32_t count;
    uint32_t _pad;
    const uint8_t* shape;              /* [C] AvnShape */
    const void* dims;                  /* [C][3] cuboid half extents / sphere radius in [0] */
    const void* position;              /* [C][3] collider Position */
    const void* rotation;              /* [C][4] collider Rotation */
    const uint32_t* memberships;       /* [C] CollisionLayers::memberships; NULL = 1 (the default layer) */
} AvnQueryColliders;
#define AVN_QUERY_SHAPES_UNCHANGED 0x1u   /* shape, dims and memberships equal the previous update's (same count): not copied again */

typedef struct AvnRayBatch {
    uint32_t count;
    uint32_t exclude_count;            /* length of exclude[] */
    const void* origin;                /* [n][3] */
    const void* direction;             /* [n][3] */
    const void* max_distance;          /* [n] */
    const uint8_t* solid;              /* [n] NULL = all solid */
    const uint32_t* max_hits;          /* [n] ray_hits only: 0 = none, 0xFFFFFFFF = all; NULL = all */
    const uint32_t* mask;              /* [n] SpatialQueryFilter::mask; NULL = all layers */
    const uint32_t* exclude_offsets;   /* [n + 1] CSR of excluded collider indices (excluded_entities, RayCaster::ignore_self); NULL = none */
    const uint32_t* exclude;           /* [exclude_count] */
} AvnRayBatch;

typedef struct AvnRayClosest {         /* per ray */
    int32_t* collider;                 /* [n] out: collider index, -1 = no hit */
    void* distance;                    /* [n] out (0 when no hit) */
    void* normal;                      /* [n][3] out (0 when no hit) */
} AvnRayClosest;

typedef struct AvnHitList {            /* CSR: the hits of query i are [offsets[i], offsets[i+1]) */
    uint64_t capacity;                 /* in: entries collider / distance / normal can hold */
    uint64_t count;                    /* out: total hits; above capacity -> AVN_ERR_CAPACITY and nothing else is written */
    uint64_t* offsets;                 /* [n + 1] out */
    uint32_t* collider;                /* [capacity] out */
    void* distance;                    /* [capacity] out, ray hits only (NULL = not wanted) */
    void* normal;                      /* [capacity][3] out, ray hits only (NULL = not wanted) */
} AvnHitList;

/* Replaces update_spatial_query_pipeline / SpatialQueryPipeline::update (spatial_query/system_param.rs:80-82, pipeline.rs:96-133): the
 * tree over every collider passed, rebuilt from scratch (LBVH: Morton codes, Karras hierarchy, bottom-up refit).  Collider index = row. */
AvnStatus avn_query_update(AvnContext* ctx, const AvnQueryColliders* colliders, uint32_t flags);
/* Replaces SpatialQueryPipeline::cast_ray (pipeline.rs:156-180), one query per ray.  Before any update: AVN_ERR_INVALID_ARGUMENT. */
AvnStatus avn_query_cast_ray(AvnContext* ctx, const AvnRayBatch* rays, AvnRayClosest* out);
/* Replaces SpatialQueryPipeline::ray_hits (pipeline.rs:182-216) and the raycast system's RayHits (ray_caster.rs:250-309): per ray its
 * max_hits nearest hits in (t, collider index) order. */
AvnStatus avn_query_ray_hits(AvnContext* ctx, const AvnRayBatch* rays, AvnHitList* out);
/* Replaces SpatialQueryPipeline::aabb_intersections_with_aabb (pipeline.rs:690-729): per query box the colliders whose tight AABB it
 * touches, ascending by index.  min / max: [n][3] in the column scalar. */
AvnStatus avn_query_aabb_intersections(AvnContext* ctx, uint32_t count, const void* min, const void* max, AvnHitList* out);

/* ---- shape casts, point projection, point and shape intersections (pipeline.rs:315-826, ShapeCaster shape_caster.rs:335-400) against
 *      the tree of the last avn_query_update.  Same arithmetic sharing as above (query_math.hpp), so results equal the host brute force bit
 *      for bit.  Conventions:
 *        - a cast moves the query shape along direction; distances are in units of |direction|.  The TOI is the smallest t in
 *          [0, max_distance] at which the closed shapes intersect.  Sphere-sphere: a solid ray cast against radius rA + rB.  Sphere-cuboid:
 *          the centre against the box rounded by the radius (exact piecewise quadratic).  Cuboid-cuboid: moving separating-axis test over
 *          the 15 axes (A's faces, B's faces, A_i x B_j; exactly-zero axes skipped); the entering axis is the largest interval start, ties
 *          to the lowest axis;
 *        - outputs (ShapeHitData): point1 / normal1 on the hit collider, normal1 outward (towards the cast shape); point2 / normal2 =
 *          -normal1 on the cast shape at its TOI pose.  Box-box face contacts report the clipped incident-face vertex nearest to the
 *          reference face; edge contacts the closest points of the two edges;
 *        - origin penetration (touching or overlapping at t = 0) is a hit at t = 0, normal along the axis of least penetration (boxes), the
 *          nearest face of a box holding the sphere's centre, or the centre difference (+y for coincident centres).
 *          AVN_CAST_IGNORE_ORIGIN_PENETRATION drops such a collider when direction . normal1 > 0; AVN_CAST_NO_CONTACT_ON_PENETRATION
 *          writes its points and normals as 0;
 *        - target_distance must be 0 (ShapeCaster's default): any other value is refused with AVN_ERR_INVALID_ARGUMENT;
 *        - project_point: cuboid = clamp in its frame, sphere = centre + r * unit(p - centre); the surface counts as inside; inside and solid
 *          -> the point itself, is_inside = 1; inside and hollow -> the nearest face (ties to the lowest axis, then the + side), +y from a
 *          sphere's centre; the closest collider is the lexicographic minimum of (distance, collider index);
 *        - point intersections: closed containment; shape intersections: exact SAT for two cuboids (touching intersects), closest point for
 *          sphere-cuboid, centre distance for two spheres; both apply the filter;
 *        - query shapes with a non-finite pose, dims, direction or max_distance or a zero quaternion hit nothing; non-finite points project
 *          onto nothing and lie in nothing; negative dims and unknown shapes are refused; a sphere of radius 0 is legal.
 *      Stated deviations: closest = minimum of (t, collider index) where the reference takes the first in tree order; shape_hits keeps the
 *      max_hits nearest sorted by (t, collider index) — the same set as the reference's repeated cast with the previous hits excluded
 *      (shape_caster.rs:372-399, pipeline.rs:524-554), since each collider's TOI does not depend on the others; only ties are ordered
 *      differently (by index instead of tree order); point and shape intersections are ascending by index, where the reference returns
 *      tree order. -------------------------------------------------------------------------------------------------------------------- */
#define AVN_CAST_IGNORE_ORIGIN_PENETRATION 0x1u   /* ShapeCastConfig::ignore_origin_penetration */
#define AVN_CAST_NO_CONTACT_ON_PENETRATION 0x2u   /* !ShapeCastConfig::compute_contact_on_penetration */

typedef struct AvnShapeBatch {
    uint32_t count;
    uint32_t exclude_count;            /* length of exclude[] */
    const uint8_t* shape;              /* [n] AvnShape */
    const void* dims;                  /* [n][3] cuboid half extents / sphere radius in [0] */
    const void* position;              /* [n][3] */
    const void* rotation;              /* [n][4] */
    const void* direction;             /* [n][3] casts only */
    const void* max_distance;          /* [n] casts only */
    const void* target_distance;       /* [n] casts only; NULL = 0; must be 0 */
    const uint32_t* flags;             /* [n] casts only: AVN_CAST_*; NULL = 0 */
    const uint32_t* max_hits;          /* [n] shape_hits only: 0 = none, 0xFFFFFFFF = all; NULL = all */
    const uint32_t* mask;              /* [n] SpatialQueryFilter::mask; NULL = all layers */
    const uint32_t* exclude_offsets;   /* [n + 1] CSR of excluded collider indices; NULL = none */
    const uint32_t* exclude;           /* [exclude_count] */
} AvnShapeBatch;

typedef struct AvnPointBatch {
    uint32_t count;
    uint32_t exclude_count;
    const void* point;                 /* [n][3] */
    const uint8_t* solid;              /* [n] project_point only; NULL = all solid */
    const uint32_t* mask;              /* [n] NULL = all layers */
    const uint32_t* exclude_offsets;   /* [n + 1] NULL = none */
    const uint32_t* exclude;           /* [exclude_count] */
} AvnPointBatch;

typedef struct AvnShapeClosest {       /* per cast */
    int32_t* collider;                 /* [n] out: collider index, -1 = no hit */
    void* distance;                    /* [n] out (0 when no hit) */
    void* point1;                      /* [n][3] out, on the collider (0 when no hit) */
    void* point2;                      /* [n][3] out, on the cast shape */
    void* normal1;                     /* [n][3] out */
    void* normal2;                     /* [n][3] out */
} AvnShapeClosest;

typedef struct AvnShapeHitList {       /* CSR as AvnHitList; the per-hit columns other than collider may be NULL (not wanted) */
    uint64_t capacity;
    uint64_t count;                    /* out: total hits; above capacity -> AVN_ERR_CAPACITY and nothing else is written */
    uint64_t* offsets;                 /* [n + 1] out */
    uint32_t* collider;                /* [capacity] out */
    void* distance;                    /* [capacity] out */
    void* point1;                      /* [capacity][3] out */
    void* point2;
    void* normal1;
    void* normal2;
} AvnShapeHitList;

typedef struct AvnPointProjection {    /* per point */
    int32_t* collider;                 /* [n] out: closest collider, -1 = none */
    void* point;                       /* [n][3] out: the projection (0 when none) */
    uint8_t* is_inside;                /* [n] out */
} AvnPointProjection;

/* Replaces SpatialQueryPipeline::cast_shape (pipeline.rs:335-375): per query shape the closest hit.  Before any update: AVN_ERR_INVALID_ARGUMENT. */
AvnStatus avn_query_cast_shape(AvnContext* ctx, const AvnShapeBatch* shapes, AvnShapeClosest* out);
/* Replaces SpatialQueryPipeline::shape_hits (pipeline.rs:443-554) and the shapecast system's ShapeHits (shape_caster.rs:335-400): per query
 * shape its max_hits nearest hits in (t, collider index) order. */
AvnStatus avn_query_shape_hits(AvnContext* ctx, const AvnShapeBatch* shapes, AvnShapeHitList* out);
/* Replaces SpatialQueryPipeline::project_point (pipeline.rs:570-615). */
AvnStatus avn_query_project_point(AvnContext* ctx, const AvnPointBatch* points, AvnPointProjection* out);
/* Replaces SpatialQueryPipeline::point_intersections (pipeline.rs:628-683): per point the colliders containing it, ascending by index. */
AvnStatus avn_query_point_intersections(AvnContext* ctx, const AvnPointBatch* points, AvnHitList* out);
/* Replaces SpatialQueryPipeline::shape_intersections (pipeline.rs:744-826): per query shape the colliders it intersects, ascending by index.
 * The cast-only columns of the batch are ignored. */
AvnStatus avn_query_shape_intersections(AvnContext* ctx, const AvnShapeBatch* shapes, AvnHitList* out);

/* ---- move and slide (MoveAndSlide::move_and_slide, character_controller/move_and_slide.rs:464-609, velocity_project.rs:122-324) for
 *      kinematic characters, against the tree of the last avn_query_update: one device thread per character runs the whole loop — an
 *      initial depenetration, up to move_and_slide_iterations rounds of shape cast (AVN_CAST_IGNORE_ORIGIN_PENETRATION), pull-back by
 *      skin_width / max(dir . -normal1, DOT_EPSILON), plane collection (the configured planes, the sweep hit's plane, every intersection at
 *      2 * skin_width, similar planes (f32 dot >= plane_similarity_dot_threshold) keeping the more blocking normal) and the cone projection
 *      of the velocity — then a final depenetration (Gauss-Seidel over the intersections at skin_width, planes deeper than
 *      penetration_rejection_threshold skipped, stop when the summed error < max_depenetration_error; all three scaled by length_unit).
 *      The per-character algorithm is avian_b200/csrc/move_math.hpp, shared with the host fixture, so results equal the host brute force
 *      bit for bit.  Dir is f32 in both builds, as in the reference: the sweep direction, the plane normals and the similarity dot product
 *      are f32 also for 64-bit columns.  Obstacles: the colliders that pass the character's filter (mask, exclusion list: exclude the
 *      character's own collider there) and are not marked in `ignored` (sensors, colliders without a body), both for the cast and the
 *      intersections.  A character with a non-finite pose, velocity or dims or a zero quaternion is returned unmoved with no hits.
 *      Stated deviations: on_hit cannot run on the device — every hit is accepted and nothing edits the normal, position or velocity; the
 *      closest sweep hit is the lowest (t, collider index), not the first in tree order; intersections are visited in ascending collider
 *      index, not tree order; hit_toi reports the TOI, where MoveHitData::collision_distance is the requested movement length (:777);
 *      characters are cuboids, spheres, capsules and convex hulls (capsule conventions: avian_b200/csrc/query_math.hpp, DESIGN.md §7j; hulls:
 *      avian_b200/csrc/hull_query_math.hpp, DESIGN.md §7l, their indices checked against the context's hull table). ------------- */
#define AVN_MOVE_MAX_PLANES 32

/* MoveAndSlideConfig, one per call.  The reference's defaults: skin_width 0.01, max_depenetration_error 0.0001,
 * penetration_rejection_threshold 0.5, plane_similarity_dot_threshold 0.99619469809 (cos 5 degrees), 4 iterations, 16 depenetration
 * iterations, 20 planes. */
typedef struct AvnMoveConfig {
    double delta_time;
    double length_unit;                 /* PhysicsLengthUnit */
    double skin_width;
    double max_depenetration_error;
    double penetration_rejection_threshold;
    double plane_similarity_dot_threshold;
    uint32_t move_and_slide_iterations;
    uint32_t depenetration_iterations;  /* 0 = no depenetration */
    uint32_t max_planes;                /* <= AVN_MOVE_MAX_PLANES */
    uint32_t collider_count;            /* entries of ignored; must equal the tree's collider count when ignored is set */
    const uint8_t* ignored;             /* [collider_count] nonzero = not an obstacle (sensors, colliders without a body); NULL = none */
} AvnMoveConfig;

typedef struct AvnMoveBatch {           /* one character per entry */
    uint32_t count;
    uint32_t exclude_count;             /* length of exclude[] */
    const uint8_t* shape;               /* [n] AvnShape */
    const void* dims;                   /* [n][3] cuboid half extents / sphere radius in [0] */
    const void* position;               /* [n][3] */
    const void* rotation;               /* [n][4] */
    const void* velocity;               /* [n][3] desired velocity */
    const uint32_t* mask;               /* [n] SpatialQueryFilter::mask; NULL = all layers */
    const uint32_t* exclude_offsets;    /* [n + 1] CSR of excluded collider indices; NULL = none */
    const uint32_t* exclude;            /* [exclude_count] */
    const uint32_t* plane_offsets;      /* [n + 1] CSR of MoveAndSlideConfig::planes per character (e.g. the ground), at most max_planes each; NULL = none */
    const void* planes;                 /* [plane_offsets[n]][3] nonzero, finite; normalised in f32 (Dir::new) */
} AvnMoveBatch;

typedef struct AvnMoveResult {
    void* position;                     /* [n][3] out: MoveAndSlideOutput::position */
    void* velocity;                     /* [n][3] out: MoveAndSlideOutput::projected_velocity */
    /* [n][move_and_slide_iterations] out, fixed stride; collider -1 = no sweep hit in that iteration (the other columns 0 there).
     * Any of these may be NULL (not wanted). */
    int32_t* hit_collider;
    void* hit_distance;                 /* the safe distance moved (MoveHitData::distance) */
    void* hit_toi;                      /* the TOI of the cast */
    void* hit_point;                    /* [..][3] point1, on the hit collider (world) */
    void* hit_normal;                   /* [..][3] normal1, outward from the hit collider */
    float kernel_ms;                    /* out: device time of the move kernel */
    uint32_t _pad;
} AvnMoveResult;

/* Before any update: AVN_ERR_INVALID_ARGUMENT.  Refused with AVN_ERR_INVALID_ARGUMENT: negative dims, unknown shapes, a bad exclusion CSR,
 * max_planes above AVN_MOVE_MAX_PLANES, more initial planes than max_planes, non-finite or zero initial planes, a NaN config value, an
 * `ignored` column whose count is not the tree's. */
AvnStatus avn_move_and_slide(AvnContext* ctx, const AvnMoveConfig* config, const AvnMoveBatch* batch, AvnMoveResult* out);

/* ---- swept continuous collision detection (SweptCcd, dynamics/ccd/mod.rs:523-780) on the device-resident solver stage ----------------
 *      Replaces solve_swept_ccd, which the reference runs after the substeps and before solve_restitution: for every SweptCcd body, in the
 *      order of the configured list, every collider adjacent to its own collider in the ContactGraph (every live contact row, touching or
 *      not) is a candidate.  Filters in the reference's order: a dynamic body 2 is skipped unless include_dynamic; the pair is skipped when
 *      |w1 - w2|^2 < angular_threshold^2 and |v1 - v2|^2 < linear_threshold^2.  The sweep is Linear when body 1 is Linear and body 2 has no
 *      configured entry or is Linear too, otherwise NonLinear.  A TOI counts when 0 < toi < min_toi (min_toi starts at dt); a TOI of exactly
 *      0 is cast again against a ball of radius prediction_distance at body 2's pose.  The body of the smallest TOI is the hit; then
 *      m = min_toi * 1.0001 and, for body 1 and for body 2 when it has a SolverBody (dynamic or kinematic): delta_position = m * v
 *      (overwritten), delta_rotation = from_scaled_axis(w * m) * delta_rotation.  Velocities are never changed.  The writes happen in the
 *      order of the configured list, so a body hit by several CCD bodies ends with the last one's delta_position.
 *      Assumptions, as the narrow phase makes them: a collider sits at its body's origin and its pose is the body's pose before the step; the
 *      body columns and the collider rows of the contact pipeline (avn_contacts_configure / avn_contacts_step) describe the same bodies.
 *      Geometry: cuboid and sphere colliders, capsules with AVN_CCD_CAPSULES and convex hulls with AVN_CCD_HULLS; conventions in
 *      avian_b200/csrc/ccd_math.hpp (linear: the shape casts of the spatial queries; non-linear: conservative advancement to
 *      eps = 1e-4 * length_unit, at most 64 iterations).
 *      Stated deviation: equal TOIs go to the lowest ContactId, where the reference keeps the first in ContactGraph adjacency order.
 *      Runs inside avn_solver_run when the upload came from the contact store (avn_solver_upload_resident): the step becomes
 *      prepare + substeps -> CCD pass -> restitution + finalize.  While CCD is configured, avn_solver_run_range,
 *      avn_solver_step_partitioned and a run after avn_solver_upload / avn_solver_step return AVN_ERR_UNSUPPORTED. */
typedef enum AvnSweepMode { AVN_SWEEP_LINEAR = 0, AVN_SWEEP_NON_LINEAR = 1 } AvnSweepMode;

#define AVN_CCD_CAPSULES 0x1u           /* AvnCcdConfig.flags: capsule colliders take part (see avn_ccd_configure) */
#define AVN_CCD_HULLS 0x4u              /* AvnCcdConfig.flags: convex hull colliders take part (see avn_ccd_configure) */

typedef struct AvnCcdConfig {
    uint32_t count;                    /* SweptCcd bodies, in query order */
    uint32_t flags;                    /* AVN_CCD_* bits; 0 = cuboid and sphere colliders only */
    const int32_t* body;               /* [n] index into AvnBodyColumns; no body twice */
    const uint32_t* collider;          /* [n] the body's own collider: a row of the contact pipeline's collider columns */
    const uint8_t* mode;               /* [n] AvnSweepMode; NULL = AVN_SWEEP_NON_LINEAR (SweptCcd::default) */
    const uint8_t* include_dynamic;    /* [n] NULL = 1 */
    const double* linear_threshold;    /* [n] NULL = 0 */
    const double* angular_threshold;   /* [n] NULL = 0 */
    double prediction_distance;        /* NarrowPhaseConfig::default_speculative_margin * PhysicsLengthUnit (default Scalar::MAX: pass +inf) */
} AvnCcdConfig;

typedef struct AvnCcdResult {          /* per configured body, the last step's pass; any pointer may be NULL */
    void* min_toi;                     /* [n] column scalar: the smallest accepted TOI before the overshoot, dt when nothing was hit */
    int32_t* hit_body;                 /* [n] the body hit, -1 = none */
    int32_t* hit_contact;              /* [n] ContactId of the hit, -1 = none */
    uint32_t* candidates;              /* [n] candidates that passed the filters (TOIs computed) */
    uint32_t* hits;                    /* [n] candidates with an accepted TOI (0 < toi < dt) */
    float pass_ms;                     /* out: device time of the pass */
    uint32_t total_candidates;         /* out */
} AvnCcdResult;

/* Persists across steps; NULL or count == 0 clears it.  Needs avn_contacts_configure first (bodies and colliders are checked against its counts).
 * Refused with AVN_ERR_INVALID_ARGUMENT: a flag bit other than AVN_CCD_CAPSULES and AVN_CCD_HULLS, bodies or colliders out of range, a body
 * listed twice, NaN thresholds, an unknown mode.  Capsules: without AVN_CCD_CAPSULES, a contact store whose shape column holds a capsule is
 * refused with AVN_ERR_UNSUPPORTED here, and so are avn_solver_upload_resident and avn_solver_run once a later avn_contacts_step brings one
 * in.  With it, capsules are swept like the other shapes (exact capsule casts in Linear mode, exact capsule distances in NonLinear mode).
 * Convex hulls: the same with AVN_CCD_HULLS, independently of AVN_CCD_CAPSULES (a store holding both shapes needs both bits).  With it, hulls
 * are swept with the exact hull casts of the spatial queries (Linear) and exact hull distances (NonLinear) over the context's hull table.
 * The pass reads the table the last avn_contacts_step used: once avn_set_convex_hulls has replaced it, avn_solver_run returns
 * AVN_ERR_INVALID_ARGUMENT before launching anything while the store holds a hull, until the next avn_contacts_step.  Body frames stay
 * refused whatever the flags. */
AvnStatus avn_ccd_configure(AvnContext* ctx, const AvnCcdConfig* config);
/* The results of the last step that ran the pass (AVN_ERR_INVALID_ARGUMENT before any). */
AvnStatus avn_ccd_download(AvnContext* ctx, AvnCcdResult* out);

AvnStatus avn_get_timings(const AvnContext* ctx, AvnTimings* out);

/*
 * Host-only helper (needs no context and no GPU): the order-preserving level schedule the solver stage uses for
 * joints.  The reference solves joints serially in type order then table order (xpbd/plugin.rs:58-86, 145-189);
 * out_level[g] (g = index in that global order) is the parallel phase joint g runs in: joints of one level touch
 * disjoint written bodies, and every joint runs after all earlier joints it shares a written body with.
 */
AvnStatus avn_joint_levels(const AvnBodyColumns* bodies, const AvnJointSet* joints, uint32_t* out_level, uint32_t* out_level_count);

#ifdef __cplusplus
}
#endif
#endif /* AVIAN_B200_H */
