// Host-side plumbing shared by the ABI translation units: error reporting, grow-only device buffers.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/avian_b200.h"
#include "hull_table.hpp"
#include "shape_column.hpp"

namespace avn {

struct ErrorSink {
    std::string msg;
    AvnStatus fail(AvnStatus code, const char* fmt, ...) {
        char buf[1024];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof buf, fmt, ap);
        va_end(ap);
        msg = buf;
        return code;
    }
};

#define AVN_CUDA(expr)                                                                                        \
    do {                                                                                                      \
        cudaError_t _e = (expr);                                                                              \
        if (_e != cudaSuccess)                                                                                \
            return err_->fail(_e == cudaErrorMemoryAllocation ? AVN_ERR_OUT_OF_MEMORY : AVN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, \
                              cudaGetErrorString(_e), __FILE__, __LINE__);                                   \
    } while (0)

// grow-only device allocation
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    ~DevBuf() { if (p) cudaFree(p); }
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T> T* as() const { return static_cast<T*>(p); }
};

// The context's convex hull table (avn_set_convex_hulls) on the device.  dev holds device pointers; count() is 0 while no table is set.  The
// AABB updater, the narrow phase, the contact store, the query tree and swept CCD hold a pointer to it.
struct HullTable {
    bool set = false;
    uint64_t generation = 0;   // incremented by every avn_set_convex_hulls that changes the table; the query tree and swept CCD check it
    hm::Table dev{};
    DevBuf vert, plane, centre, radius, voff, foff, loff, loop, eoff, edge;
    uint32_t count() const { return set ? dev.count : 0; }
};

// the context's communicator (comm.cu): NCCL bound at run time; a communicator of one needs no NCCL at all
struct CommBase {
    virtual ~CommBase() {}
    virtual AvnStatus unique_id(void* out_id) = 0;
    virtual AvnStatus init(uint32_t rank, uint32_t world, const void* id) = 0;
    virtual AvnStatus shutdown() = 0;
    virtual int rank() const = 0;
    virtual int world() const = 0;
    virtual AvnStatus all_gather(const void* send_dev, void* recv_dev, size_t bytes_per_rank) = 0;   // on the context's stream
    virtual AvnStatus all_reduce_max_i32(int* dev, size_t count) = 0;
};
CommBase* make_comm(cudaStream_t stream, ErrorSink* err);

struct ContactsBase;
struct CcdBase;
struct CcdRows;
struct SolverBase {
    virtual ~SolverBase() {}
    virtual AvnStatus upload(const AvnStepParams* prm, AvnBodyColumns* bodies, AvnManifoldColumns* manifolds, AvnJointSet* joints) = 0;
    // the same fed from the contact store: the rows (ContactsBase::view / outputs) and the colour-major list (ContactsBase::graph_view) are on the
    // device, nothing of the constraints crosses the bus
    virtual AvnStatus upload_resident(const AvnStepParams* prm, AvnBodyColumns* bodies, ContactsBase* contacts, AvnJointSet* joints) = 0;
    virtual AvnStatus run() = 0;
    virtual AvnStatus run_range(uint32_t first, uint32_t count, uint32_t flags) = 0;
    virtual AvnStatus set_boundary(const AvnBoundary* bnd) = 0;
    virtual AvnStatus boundary_snapshot() = 0;
    virtual AvnStatus boundary_pack(void* device_table) = 0;
    virtual AvnStatus boundary_apply(const void* device_gathered) = 0;
    // the whole partitioned stage of one rank: launches substep by substep with the boundary exchange over `comm` in between
    virtual AvnStatus step_partitioned(CommBase* comm) = 0;
    virtual int needs_restitution() const = 0;
    // start the host-to-device copy of the next upload's body columns on a second stream (overlaps whatever runs before the solver stage)
    virtual AvnStatus prefetch_bodies(AvnBodyColumns* bodies, uint32_t flags) = 0;
    virtual AvnStatus download() = 0;
    virtual void timings(AvnTimings* t) const = 0;
    // the context's CCD pass and the contact store it reads: avn_solver_run runs the pass between the substeps and restitution when the pass is
    // configured and the upload came from the contact store
    virtual void attach_ccd(CcdBase* ccd, ContactsBase* contacts) = 0;
};
// the new pairs of the last broad-phase run where the run left them (device memory); count is known on the host after the run settled
struct DevicePairs {
    uint64_t count = 0;
    const uint32_t* c1 = nullptr; const uint32_t* c2 = nullptr; const uint32_t* b1 = nullptr; const uint32_t* b2 = nullptr;
    const uint8_t* flags = nullptr;
};

struct BroadphaseBase {
    virtual ~BroadphaseBase() {}
    virtual AvnStatus upload(AvnAabbColumns* aabbs) = 0;
    virtual AvnStatus run() = 0;
    virtual AvnStatus download(AvnPairList* out) = 0;
    // device-resident pipeline: the pairs stay on the device (the contact store takes them from there); only the persistent order and the
    // pair count go to the host
    virtual AvnStatus device_pairs(DevicePairs* out) = 0;
    virtual AvnStatus download_order(uint64_t* out_pair_count) = 0;
    // ContactGraph::pair_set kept by the contact store on the device: used as the "existing pairs" set of every later upload that
    // brings no host key list (table == NULL switches back)
    virtual void set_existing_device(const uint64_t* table, uint64_t mask) = 0;
    virtual void timings(AvnTimings* t) const = 0;
};

struct AabbBase {
    virtual ~AabbBase() {}
    virtual AvnStatus update(const AvnAabbParams* prm, AvnColliderColumns* colliders) = 0;
    virtual void attach_hulls(const HullTable* hulls) = 0;
};
AabbBase* make_aabb_updater(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err);

// The body frames of avn_contacts_set_body_frames: a host copy of the caller's columns in the column scalar, which every later
// avn_contacts_step / avn_narrow_phase uses until the next call (the contact store keeps it).
struct BodyFrames {
    uint32_t body_count = 0;
    std::vector<unsigned char> position, rotation, com;   // [B][3], [B][4], [B][3] scalars; com empty = 0
};

struct NarrowBase {
    virtual ~NarrowBase() {}
    // frames: NULL = a collider at its body's origin, the centre of mass at that origin
    virtual AvnStatus run(const AvnNarrowParams* prm, const AvnNarrowInput* in, AvnRawManifolds* out, const BodyFrames* frames) = 0;
    virtual void attach_hulls(const HullTable* hulls) = 0;
};
NarrowBase* make_narrow(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err);

// the spatial-query tree and its batched queries (queries.cu)
struct QueriesBase {
    virtual ~QueriesBase() {}
    virtual AvnStatus update(const AvnQueryColliders* colliders, uint32_t flags) = 0;
    virtual AvnStatus cast_ray(const AvnRayBatch* rays, AvnRayClosest* out) = 0;
    virtual AvnStatus ray_hits(const AvnRayBatch* rays, AvnHitList* out) = 0;
    virtual AvnStatus aabb_intersections(uint32_t count, const void* min, const void* max, AvnHitList* out) = 0;
    virtual AvnStatus cast_shape(const AvnShapeBatch* shapes, AvnShapeClosest* out) = 0;
    virtual AvnStatus shape_hits(const AvnShapeBatch* shapes, AvnShapeHitList* out) = 0;
    virtual AvnStatus project_point(const AvnPointBatch* points, AvnPointProjection* out) = 0;
    virtual AvnStatus point_intersections(const AvnPointBatch* points, AvnHitList* out) = 0;
    virtual AvnStatus shape_intersections(const AvnShapeBatch* shapes, AvnHitList* out) = 0;
    virtual AvnStatus move_and_slide(const AvnMoveConfig* config, const AvnMoveBatch* batch, AvnMoveResult* out) = 0;
    // the context's hull table: hull colliders, query shapes and characters index it; a tree holding a hull is refused once it is replaced
    virtual void attach_hulls(const HullTable* hulls) = 0;
};
QueriesBase* make_queries(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err);

struct ContactsBase {
    virtual ~ContactsBase() {}
    struct RowColumns {             // device pointers of the row columns (ContactId-indexed, 4 point slots per row, column scalar type)
        uint32_t rows = 0;          // allocated rows
        const uint8_t* point_count = nullptr;
        const void* normal = nullptr; const void* anchor1 = nullptr; const void* anchor2 = nullptr; const void* penetration = nullptr;
        const void* normal_speed = nullptr;
        void* warm_start_normal_impulse = nullptr; void* warm_start_tangent_impulse = nullptr; void* normal_impulse = nullptr;
    };
    virtual void view(RowColumns* out) = 0;                                  // what the solver reads
    virtual void outputs(void** ws_n, void** ws_t, void** nimp) = 0;         // device pointers store_contact_impulses writes
    virtual AvnStatus download_impulses(uint32_t capacity, void* ws_n, void* ws_t, void* nimp) = 0;
    // ---- the ContactGraph + ConstraintGraph on the device (contacts.cu)
    virtual AvnStatus configure(const AvnContactGraphConfig* cfg) = 0;
    // start the host-to-device copy of step()'s collider / body columns on a second stream (before the broad phase is waited for)
    virtual AvnStatus prefetch_inputs(const AvnNarrowParams* prm, const AvnNarrowInput* in, uint32_t match_contacts, double length_unit, uint32_t flags) = 0;
    virtual AvnStatus step(const AvnNarrowParams* prm, const AvnNarrowInput* in, uint32_t match_contacts, double length_unit, const DevicePairs* new_pairs,
                           AvnContactStep* out) = 0;
    struct ResidentGraph {          // device pointers of the colour-major list the last step() built
        uint32_t count = 0, any_restitution = 0;
        uint32_t color_offsets[AVN_GRAPH_COLOR_COUNT + 1] = {};
        const uint32_t* edge = nullptr; const int32_t* body1 = nullptr; const int32_t* body2 = nullptr;
        const void* friction = nullptr; const void* restitution = nullptr;
    };
    virtual AvnStatus graph_view(ResidentGraph* out) = 0;
    virtual void pair_set(const uint64_t** table, uint64_t* mask) = 0;
    virtual AvnStatus download_graph(uint32_t capacity, uint32_t* c1, uint32_t* c2, uint8_t* live, uint8_t* touching, int8_t* colour, uint32_t* edge_list) = 0;
    // ---- the pipeline's output to the application: sensors, removal of colliders, collision events, contact reports (contacts.cu)
    virtual AvnStatus set_sensors(uint32_t collider_count, const uint8_t* sensor) = 0;
    virtual AvnStatus remove_colliders(uint32_t n, const uint32_t* colliders) = 0;
    virtual AvnStatus events(AvnCollisionEvents* started, AvnCollisionEvents* ended) = 0;
    virtual AvnStatus report(uint32_t flags, AvnContactReport* out) = 0;
    // ---- persistent simulation islands + sleeping decisions (contacts.cu)
    virtual AvnStatus islands_configure(const AvnIslandsConfig* cfg) = 0;
    virtual AvnStatus islands_step(AvnIslandsStep* step) = 0;
    // ---- applied sleeping (contacts.cu): the switch, the narrow-phase half of the island step, and what the solver stage needs of it
    virtual AvnStatus islands_apply(uint32_t enable) = 0;
    virtual AvnStatus islands_wake(const uint8_t* wake, AvnIslandsWake* out) = 0;
    virtual AvnStatus download_sleeping(uint32_t capacity, uint8_t* row_asleep, uint32_t body_count, uint8_t* body_asleep) = 0;
    struct AsleepBodies {           // body_asleep: device column [count], NULL while application is off
        const uint8_t* body_asleep = nullptr;
        uint32_t count = 0;
        bool wake_skipped = false;  // avn_islands_wake has not run for the current contact step
    };
    virtual void asleep_bodies(AsleepBodies* out) = 0;
    // ---- the rows and collider shapes swept CCD visits (ccd.cu)
    virtual void ccd_rows(CcdRows* out) = 0;
    // ---- the shape column of a step: checked on the host when step() is going to copy it (not under AVN_CONTACTS_SHAPES_UNCHANGED), before
    //      any state changes; has_capsule: the column of the last accepted step holds a capsule (swept CCD refuses it unless configured with
    //      AVN_CCD_CAPSULES, and launches its capsule TOI kernel only when it holds one)
    virtual AvnStatus check_shapes(const AvnNarrowInput* in, uint32_t flags) = 0;
    virtual bool has_capsule() const = 0;
    // has_hull: the column on the device holds a convex hull (swept CCD refuses it unless configured with AVN_CCD_HULLS; its rows run in the
    // hull kernels).  The hull table is the context's (attach_hulls); a step under AVN_CONTACTS_SHAPES_UNCHANGED checks the kept column's
    // largest hull index against it, and every step records the table's generation for swept CCD (CcdRows::hull_generation).
    virtual bool has_hull() const = 0;
    virtual void attach_hulls(const HullTable* hulls) = 0;
    // ---- body frames (avn_contacts_set_body_frames): checked and copied on the host (NULL clears them); body_frames() = NULL when none are set
    virtual AvnStatus set_body_frames(const AvnBodyFrames* frames) = 0;
    virtual const BodyFrames* body_frames() const = 0;
};
ContactsBase* make_contacts(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err);

// ---- swept CCD (ccd.cu): what the pass reads from the contact store and from the solver's step state (device pointers, column scalar)
struct CcdRows {
    uint32_t rows = 0;                 // ContactIds in use: [0, rows)
    uint32_t bodies = 0, colliders = 0;   // avn_contacts_configure's counts (0 before it)
    const uint32_t* c1 = nullptr; const uint32_t* c2 = nullptr; const uint32_t* b1 = nullptr; const uint32_t* b2 = nullptr;
    const uint8_t* live = nullptr;
    const uint8_t* shape = nullptr;    // [C] of the last avn_contacts_step (NULL = cuboid)
    const void* dims = nullptr;        // [C][3]
    bool has_capsule = false;          // the shape column holds a capsule
    bool has_hull = false;             // the shape column holds a convex hull
    uint64_t hull_generation = 0;      // HullTable::generation at the last avn_contacts_step (the table its hull kernels read)
};
struct CcdSolverState {
    int B = 0;
    double dt = 0, length_unit = 1;
    const uint8_t* kind = nullptr;     // NULL = dynamic
    const void* position = nullptr; const void* rotation = nullptr; const void* com = nullptr;   // pre-step pose, local centre of mass (NULL = 0)
    void* vel = nullptr;               // Vec4 rows {lin}{ang} per body (solver_dev.cuh)
    void* dlt = nullptr;               // Vec4 rows {delta_position}{delta_rotation}
};
struct CcdBase {
    virtual ~CcdBase() {}
    virtual AvnStatus configure(const AvnCcdConfig* cfg, const CcdRows& rows) = 0;
    virtual bool active() const = 0;
    virtual bool capsules() const = 0;   // configured with AVN_CCD_CAPSULES
    virtual bool hulls() const = 0;      // configured with AVN_CCD_HULLS
    // the context's hull table, which the hull TOI kernel reads; table_changed: the pass would run that kernel and the table is no longer
    // the one the last contact step used (avn_set_convex_hulls since)
    virtual void attach_hulls(const HullTable* hulls) = 0;
    virtual bool table_changed(const CcdRows& rows) const = 0;
    // enqueued on the context's stream; adds its kernel launches to *launches
    virtual AvnStatus run(const CcdSolverState& st, const CcdRows& rows, uint32_t* launches) = 0;
    virtual AvnStatus download(AvnCcdResult* out) = 0;
};
CcdBase* make_ccd(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err);

SolverBase* make_solver(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err, uint32_t cfg_flags, int device);
BroadphaseBase* make_broadphase(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err, int device);

}  // namespace avn
