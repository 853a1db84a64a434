// extern "C" surface of libavian_b200.so (declared in include/avian_b200.h).
#include <cstring>
#include <memory>
#include <mutex>
#include <new>

#include "context.hpp"
#include "hull_math.hpp"
#include "joint_schedule.hpp"

struct AvnContext {
    int device = 0;
    uint32_t scalar_bits = 32;
    cudaStream_t stream = nullptr;
    avn::ErrorSink err;
    std::unique_ptr<avn::SolverBase> solver;
    std::unique_ptr<avn::BroadphaseBase> broadphase;
    std::unique_ptr<avn::AabbBase> aabbs;
    std::unique_ptr<avn::NarrowBase> narrow;
    std::unique_ptr<avn::ContactsBase> contacts;
    std::unique_ptr<avn::QueriesBase> queries;
    std::unique_ptr<avn::CommBase> comm;
    std::unique_ptr<avn::CcdBase> ccd;
    avn::HullTable hulls;              // avn_set_convex_hulls; read by aabbs, narrow, contacts, queries and ccd
    AvnTimings last{};
};

namespace {
std::string g_create_error;
std::mutex g_create_mutex;

AvnStatus create_fail(AvnStatus code, const std::string& msg) {
    std::lock_guard<std::mutex> lk(g_create_mutex);
    g_create_error = msg;
    return code;
}
bool bind(AvnContext* ctx) { return cudaSetDevice(ctx->device) == cudaSuccess; }

// "nothing throws or aborts across the ABI": every entry point that reaches C++ code which may allocate (std::vector, std::string, new) runs
// inside this guard; an exception becomes a status code and a message.
template <class F>
AvnStatus guarded(AvnContext* ctx, F&& body) noexcept {
    if (!ctx) return AVN_ERR_INVALID_ARGUMENT;
    try {
        if (!bind(ctx)) return ctx->err.fail(AVN_ERR_CUDA, "cudaSetDevice failed");
        return body();
    } catch (const std::bad_alloc&) {
        try { return ctx->err.fail(AVN_ERR_OUT_OF_MEMORY, "host allocation failed"); } catch (...) { return AVN_ERR_OUT_OF_MEMORY; }
    } catch (const std::exception& e) {
        try { return ctx->err.fail(AVN_ERR_INVALID_ARGUMENT, "internal error: %s", e.what()); } catch (...) { return AVN_ERR_INVALID_ARGUMENT; }
    } catch (...) {
        return AVN_ERR_INVALID_ARGUMENT;
    }
}
thread_local char t_create_error[512];
}  // namespace

extern "C" {

uint32_t avn_abi_version(void) { return AVN_ABI_VERSION; }

AvnStatus avn_create(const AvnConfig* config, AvnContext** out_ctx) {
    if (!config || !out_ctx) return create_fail(AVN_ERR_INVALID_ARGUMENT, "config and out_ctx are required");
    *out_ctx = nullptr;
    cudaStream_t stream = nullptr;
    try {
        if (config->abi_version != AVN_ABI_VERSION) return create_fail(AVN_ERR_INVALID_ARGUMENT, "ABI version mismatch");
        if (config->scalar_bits != 32 && config->scalar_bits != 64) return create_fail(AVN_ERR_INVALID_ARGUMENT, "scalar_bits must be 32 or 64");
        int count = 0;
        cudaError_t e = cudaGetDeviceCount(&count);
        if (e != cudaSuccess || count == 0)
            return create_fail(AVN_ERR_CUDA, std::string("no usable CUDA device (this library has no CPU fallback): ") + cudaGetErrorString(e));
        if (config->device < 0 || config->device >= count) return create_fail(AVN_ERR_INVALID_ARGUMENT, "device ordinal out of range");
        if ((e = cudaSetDevice(config->device)) != cudaSuccess) return create_fail(AVN_ERR_CUDA, cudaGetErrorString(e));
        cudaDeviceProp prop;
        if ((e = cudaGetDeviceProperties(&prop, config->device)) != cudaSuccess) return create_fail(AVN_ERR_CUDA, cudaGetErrorString(e));
        if (prop.major != 9 || prop.minor != 0)
            return create_fail(AVN_ERR_UNSUPPORTED, std::string("kernels are built for sm_90a only; device is ") + prop.name + " (sm_" +
                                                        std::to_string(prop.major) + std::to_string(prop.minor) + ")");
        auto ctx = std::make_unique<AvnContext>();
        ctx->device = config->device;
        ctx->scalar_bits = config->scalar_bits;
        if ((e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)) != cudaSuccess) return create_fail(AVN_ERR_CUDA, cudaGetErrorString(e));
        ctx->stream = stream;
        ctx->solver.reset(avn::make_solver(config->scalar_bits, ctx->stream, &ctx->err, config->flags, config->device));
        ctx->broadphase.reset(avn::make_broadphase(config->scalar_bits, ctx->stream, &ctx->err, config->device));
        ctx->aabbs.reset(avn::make_aabb_updater(config->scalar_bits, ctx->stream, &ctx->err));
        ctx->narrow.reset(avn::make_narrow(config->scalar_bits, ctx->stream, &ctx->err));
        ctx->contacts.reset(avn::make_contacts(config->scalar_bits, ctx->stream, &ctx->err));
        ctx->queries.reset(avn::make_queries(config->scalar_bits, ctx->stream, &ctx->err));
        ctx->comm.reset(avn::make_comm(ctx->stream, &ctx->err));
        ctx->ccd.reset(avn::make_ccd(config->scalar_bits, ctx->stream, &ctx->err));
        if (!ctx->solver || !ctx->broadphase || !ctx->aabbs || !ctx->narrow || !ctx->contacts || !ctx->queries || !ctx->ccd) {
            ctx.reset();   // the members hold the stream: release them before it goes
            cudaStreamDestroy(stream);
            return create_fail(AVN_ERR_UNSUPPORTED, "scalar type not available");
        }
        ctx->solver->attach_ccd(ctx->ccd.get(), ctx->contacts.get());
        ctx->aabbs->attach_hulls(&ctx->hulls);
        ctx->narrow->attach_hulls(&ctx->hulls);
        ctx->contacts->attach_hulls(&ctx->hulls);
        ctx->queries->attach_hulls(&ctx->hulls);
        ctx->ccd->attach_hulls(&ctx->hulls);
        *out_ctx = ctx.release();
        return AVN_OK;
    } catch (...) {
        if (stream) cudaStreamDestroy(stream);
        try { return create_fail(AVN_ERR_OUT_OF_MEMORY, "host allocation failed in avn_create"); } catch (...) { return AVN_ERR_OUT_OF_MEMORY; }
    }
}

void avn_destroy(AvnContext* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    ctx->comm.reset();
    ctx->solver.reset();
    ctx->ccd.reset();
    ctx->broadphase.reset();
    ctx->aabbs.reset();
    ctx->narrow.reset();
    ctx->contacts.reset();
    ctx->queries.reset();
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* avn_last_error(const AvnContext* ctx) {
    if (ctx) return ctx->err.msg.c_str();
    std::lock_guard<std::mutex> lk(g_create_mutex);   // copied under the lock: the returned pointer stays valid for this thread
    std::strncpy(t_create_error, g_create_error.c_str(), sizeof t_create_error - 1);
    t_create_error[sizeof t_create_error - 1] = 0;
    return t_create_error;
}

AvnStatus avn_alloc_pinned(AvnContext* ctx, size_t bytes, void** out_ptr) {
    if (!ctx || !out_ptr) return AVN_ERR_INVALID_ARGUMENT;
    if (!bind(ctx)) return ctx->err.fail(AVN_ERR_CUDA, "cudaSetDevice failed");
    cudaError_t e = cudaHostAlloc(out_ptr, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) return ctx->err.fail(AVN_ERR_OUT_OF_MEMORY, "cudaHostAlloc(%zu): %s", bytes, cudaGetErrorString(e));
    return AVN_OK;
}

AvnStatus avn_free_pinned(AvnContext* ctx, void* ptr) {
    if (!ctx) return AVN_ERR_INVALID_ARGUMENT;
    if (!ptr) return AVN_OK;
    cudaError_t e = cudaFreeHost(ptr);
    if (e != cudaSuccess) return ctx->err.fail(AVN_ERR_CUDA, "cudaFreeHost: %s", cudaGetErrorString(e));
    return AVN_OK;
}

AvnStatus avn_solver_upload(AvnContext* ctx, const AvnStepParams* params, AvnBodyColumns* bodies, AvnManifoldColumns* manifolds, AvnJointSet* joints) {
    return guarded(ctx, [&] { return ctx->solver->upload(params, bodies, manifolds, joints); });
}
AvnStatus avn_solver_run(AvnContext* ctx) {
    return guarded(ctx, [&] { return ctx->solver->run(); });
}
AvnStatus avn_solver_run_range(AvnContext* ctx, uint32_t first_substep, uint32_t substep_count, uint32_t run_flags) {
    return guarded(ctx, [&] { return ctx->solver->run_range(first_substep, substep_count, run_flags); });
}
AvnStatus avn_solver_set_boundary(AvnContext* ctx, const AvnBoundary* boundary) {
    return guarded(ctx, [&] { return ctx->solver->set_boundary(boundary); });
}
AvnStatus avn_solver_boundary_snapshot(AvnContext* ctx) {
    return guarded(ctx, [&] { return ctx->solver->boundary_snapshot(); });
}
AvnStatus avn_solver_boundary_pack(AvnContext* ctx, void* device_table) {
    return guarded(ctx, [&] { return ctx->solver->boundary_pack(device_table); });
}
AvnStatus avn_solver_boundary_apply(AvnContext* ctx, const void* device_gathered) {
    return guarded(ctx, [&] { return ctx->solver->boundary_apply(device_gathered); });
}
AvnStatus avn_solver_needs_restitution(AvnContext* ctx, int* out_nonzero) {
    if (!ctx || !out_nonzero) return AVN_ERR_INVALID_ARGUMENT;
    *out_nonzero = ctx->solver->needs_restitution();
    return AVN_OK;
}
AvnStatus avn_solver_step_partitioned(AvnContext* ctx) {
    return guarded(ctx, [&] { return ctx->solver->step_partitioned(ctx->comm.get()); });
}
AvnStatus avn_comm_unique_id(AvnContext* ctx, void* out_id) {
    return guarded(ctx, [&] { return ctx->comm->unique_id(out_id); });
}
AvnStatus avn_comm_init(AvnContext* ctx, uint32_t rank, uint32_t world, const void* unique_id) {
    return guarded(ctx, [&] { return ctx->comm->init(rank, world, unique_id); });
}
AvnStatus avn_comm_destroy(AvnContext* ctx) {
    return guarded(ctx, [&] { return ctx->comm->shutdown(); });
}
AvnStatus avn_comm_all_gather(AvnContext* ctx, const void* send_device, void* recv_device, size_t bytes_per_rank) {
    return guarded(ctx, [&] { return ctx->comm->all_gather(send_device, recv_device, bytes_per_rank); });
}
AvnStatus avn_get_stream(AvnContext* ctx, void** out_stream) {
    if (!ctx || !out_stream) return AVN_ERR_INVALID_ARGUMENT;
    *out_stream = (void*)ctx->stream;
    return AVN_OK;
}
AvnStatus avn_solver_download(AvnContext* ctx) {
    return guarded(ctx, [&] {
        AvnStatus st = ctx->solver->download();
        ctx->solver->timings(&ctx->last);
        return st;
    });
}
AvnStatus avn_solver_step(AvnContext* ctx, const AvnStepParams* params, AvnBodyColumns* bodies, AvnManifoldColumns* manifolds, AvnJointSet* joints) {
    AvnStatus st = avn_solver_upload(ctx, params, bodies, manifolds, joints);
    if (st != AVN_OK) return st;
    if ((st = avn_solver_run(ctx)) != AVN_OK) return st;
    return avn_solver_download(ctx);
}

AvnStatus avn_broadphase_upload(AvnContext* ctx, AvnAabbColumns* aabbs) {
    return guarded(ctx, [&] { return ctx->broadphase->upload(aabbs); });
}
AvnStatus avn_broadphase_run(AvnContext* ctx) {
    return guarded(ctx, [&] { return ctx->broadphase->run(); });
}
AvnStatus avn_broadphase_download(AvnContext* ctx, AvnPairList* out_pairs) {
    return guarded(ctx, [&] {
        AvnStatus st = ctx->broadphase->download(out_pairs);
        ctx->broadphase->timings(&ctx->last);
        return st;
    });
}
AvnStatus avn_broadphase(AvnContext* ctx, AvnAabbColumns* aabbs, AvnPairList* out_pairs) {
    AvnStatus st = avn_broadphase_upload(ctx, aabbs);
    if (st != AVN_OK) return st;
    if ((st = avn_broadphase_run(ctx)) != AVN_OK) return st;
    return avn_broadphase_download(ctx, out_pairs);
}

AvnStatus avn_update_aabbs(AvnContext* ctx, const AvnAabbParams* params, AvnColliderColumns* colliders) {
    return guarded(ctx, [&] { return ctx->aabbs->update(params, colliders); });
}

AvnStatus avn_narrow_phase(AvnContext* ctx, const AvnNarrowParams* params, const AvnNarrowInput* input, AvnRawManifolds* out) {
    return guarded(ctx, [&] { return ctx->narrow->run(params, input, out, ctx->contacts->body_frames()); });
}

AvnStatus avn_set_convex_hulls(AvnContext* ctx, const AvnConvexHulls* hulls) {
    return guarded(ctx, [&]() -> AvnStatus {
        avn::HullTable& t = ctx->hulls;
        if (!hulls) { t.set = false; ++t.generation; return AVN_OK; }
        const uint32_t H = hulls->hull_count;
        if (H > AVN_HULL_MAX_COUNT) return ctx->err.fail(AVN_ERR_INVALID_ARGUMENT, "set_convex_hulls: %u hulls, at most AVN_HULL_MAX_COUNT", H);
        if (!hulls->vertex_offsets || !hulls->vertices || !hulls->face_offsets || !hulls->loop_offsets || !hulls->loop)
            return ctx->err.fail(AVN_ERR_INVALID_ARGUMENT, "set_convex_hulls: vertex_offsets, vertices, face_offsets, loop_offsets and loop are required");
        const size_t V = hulls->vertex_offsets[H];
        std::vector<double> vert(3 * V);
        for (size_t i = 0; i < 3 * V; ++i)
            vert[i] = ctx->scalar_bits == 64 ? static_cast<const double*>(hulls->vertices)[i] : double(static_cast<const float*>(hulls->vertices)[i]);
        hm::HullSet set;
        uint32_t at = 0;
        if (const char* why = hm::derive_hulls(H, hulls->vertex_offsets, vert.data(), hulls->face_offsets, hulls->loop_offsets, hulls->loop, &set, &at))
            return ctx->err.fail(AVN_ERR_INVALID_ARGUMENT, "set_convex_hulls: hull %u: %s", at, why);
        // the previous table may still be read by work on the stream: let it finish before its buffers are replaced.  Every reader of the
        // table runs on the context's stream, so the copies go there too (a synchronous cudaMemcpy runs on the legacy default stream, which
        // a non-blocking stream does not wait for), and the call waits for them before the table is marked set and the host copy is freed
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        auto put = [&](avn::DevBuf& buf, const void* src, size_t bytes) -> const void* {
            if (e != cudaSuccess) return nullptr;
            if ((e = buf.ensure(bytes ? bytes : 1)) != cudaSuccess) return nullptr;
            if (bytes) e = cudaMemcpyAsync(buf.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream);
            return buf.p;
        };
        t.set = false;   // a failed upload leaves no table
        ++t.generation;
        hm::Table d{};
        d.count = H;
        d.vert = static_cast<const double*>(put(t.vert, set.vert.data(), set.vert.size() * sizeof(double)));
        d.plane = static_cast<const double*>(put(t.plane, set.plane.data(), set.plane.size() * sizeof(double)));
        d.centre = static_cast<const double*>(put(t.centre, set.centre.data(), set.centre.size() * sizeof(double)));
        d.radius = static_cast<const double*>(put(t.radius, set.radius.data(), set.radius.size() * sizeof(double)));
        d.voff = static_cast<const uint32_t*>(put(t.voff, set.voff.data(), set.voff.size() * sizeof(uint32_t)));
        d.foff = static_cast<const uint32_t*>(put(t.foff, set.foff.data(), set.foff.size() * sizeof(uint32_t)));
        d.loff = static_cast<const uint32_t*>(put(t.loff, set.loff.data(), set.loff.size() * sizeof(uint32_t)));
        d.loop = static_cast<const uint32_t*>(put(t.loop, set.loop.data(), set.loop.size() * sizeof(uint32_t)));
        d.eoff = static_cast<const uint32_t*>(put(t.eoff, set.eoff.data(), set.eoff.size() * sizeof(uint32_t)));
        d.edge = static_cast<const uint32_t*>(put(t.edge, set.edge.data(), set.edge.size() * sizeof(uint32_t)));
        const cudaError_t done = cudaStreamSynchronize(ctx->stream);   // also when a copy failed: `set` is freed on return
        if (e == cudaSuccess) e = done;
        if (e != cudaSuccess)
            return ctx->err.fail(e == cudaErrorMemoryAllocation ? AVN_ERR_OUT_OF_MEMORY : AVN_ERR_CUDA, "set_convex_hulls: upload failed: %s", cudaGetErrorString(e));
        t.dev = d;
        t.set = true;
        return AVN_OK;
    });
}

AvnStatus avn_contacts_configure(AvnContext* ctx, const AvnContactGraphConfig* config) { return guarded(ctx, [&] { return ctx->contacts->configure(config); }); }
AvnStatus avn_contacts_step(AvnContext* ctx, const AvnNarrowParams* params, const AvnNarrowInput* input, uint32_t match_contacts, double length_unit, uint32_t flags,
                            AvnContactStep* out) {
    return guarded(ctx, [&] {
        avn::DevicePairs pairs;
        const bool take = (flags & AVN_CONTACTS_TAKE_BROADPHASE_PAIRS) != 0;
        // this step's collider / body columns start moving to the device before the broad phase is waited for; a shape column that is
        // going to be copied is checked first, so a refused step changes nothing
        if (params && input && out) {
            const avn::BodyFrames* frames = ctx->contacts->body_frames();
            if (frames && frames->body_count != input->body_count)
                return ctx->err.fail(AVN_ERR_INVALID_ARGUMENT, "contacts_step: the body frames have %u bodies, the input %u", frames->body_count, input->body_count);
            AvnStatus st = ctx->contacts->check_shapes(input, flags);
            if (st != AVN_OK) return st;
            st = ctx->contacts->prefetch_inputs(params, input, match_contacts, length_unit, flags);
            if (st != AVN_OK) return st;
        }
        if (take) {
            AvnStatus st = ctx->broadphase->device_pairs(&pairs);
            if (st != AVN_OK) return st;
        }
        AvnStatus st = ctx->contacts->step(params, input, match_contacts, length_unit, take ? &pairs : nullptr, out);
        if (st != AVN_OK) return st;
        // ContactGraph::pair_set stays on the device: the next broad phase filters against it
        const uint64_t* table = nullptr;
        uint64_t mask = 0;
        ctx->contacts->pair_set(&table, &mask);
        ctx->broadphase->set_existing_device(table, mask);
        return AVN_OK;
    });
}
AvnStatus avn_contacts_set_body_frames(AvnContext* ctx, const AvnBodyFrames* frames) {
    return guarded(ctx, [&] {
        if (frames && ctx->ccd->active())
            return ctx->err.fail(AVN_ERR_UNSUPPORTED, "contacts_set_body_frames: swept CCD is configured (avn_ccd_configure); it assumes a collider at its body's origin");
        return ctx->contacts->set_body_frames(frames);
    });
}
AvnStatus avn_solver_upload_resident(AvnContext* ctx, const AvnStepParams* params, AvnBodyColumns* bodies, AvnJointSet* joints) {
    return guarded(ctx, [&] { return ctx->solver->upload_resident(params, bodies, ctx->contacts.get(), joints); });
}
AvnStatus avn_solver_prefetch_bodies(AvnContext* ctx, AvnBodyColumns* bodies, uint32_t flags) {
    return guarded(ctx, [&] { return ctx->solver->prefetch_bodies(bodies, flags); });
}
AvnStatus avn_broadphase_download_order(AvnContext* ctx, uint64_t* out_pair_count) { return guarded(ctx, [&] { return ctx->broadphase->download_order(out_pair_count); }); }
AvnStatus avn_contacts_download_graph(AvnContext* ctx, uint32_t capacity, uint32_t* collider1, uint32_t* collider2, uint8_t* live, uint8_t* touching, int8_t* colour,
                                      uint32_t* edge_list) {
    return guarded(ctx, [&] { return ctx->contacts->download_graph(capacity, collider1, collider2, live, touching, colour, edge_list); });
}
// the pipeline's output to the application (contacts.cu): a removal rebuilds the pair set, which the next broad phase filters against
AvnStatus avn_contacts_set_sensors(AvnContext* ctx, uint32_t collider_count, const uint8_t* sensor) {
    return guarded(ctx, [&] {
        AvnStatus st = ctx->contacts->set_sensors(collider_count, sensor);
        const uint64_t* table = nullptr;
        uint64_t mask = 0;
        ctx->contacts->pair_set(&table, &mask);
        ctx->broadphase->set_existing_device(table, mask);
        return st;
    });
}
AvnStatus avn_contacts_remove_colliders(AvnContext* ctx, uint32_t n, const uint32_t* colliders) {
    return guarded(ctx, [&] {
        AvnStatus st = ctx->contacts->remove_colliders(n, colliders);
        const uint64_t* table = nullptr;
        uint64_t mask = 0;
        ctx->contacts->pair_set(&table, &mask);
        ctx->broadphase->set_existing_device(table, mask);
        return st;
    });
}
AvnStatus avn_contacts_events(AvnContext* ctx, AvnCollisionEvents* started, AvnCollisionEvents* ended) {
    return guarded(ctx, [&] { return ctx->contacts->events(started, ended); });
}
AvnStatus avn_contacts_report(AvnContext* ctx, uint32_t flags, AvnContactReport* out) {
    return guarded(ctx, [&] { return ctx->contacts->report(flags, out); });
}
AvnStatus avn_islands_configure(AvnContext* ctx, const AvnIslandsConfig* config) { return guarded(ctx, [&] { return ctx->contacts->islands_configure(config); }); }
AvnStatus avn_islands_step(AvnContext* ctx, AvnIslandsStep* step) { return guarded(ctx, [&] { return ctx->contacts->islands_step(step); }); }
AvnStatus avn_islands_apply(AvnContext* ctx, uint32_t enable) {
    return guarded(ctx, [&] {
        if (enable && ctx->ccd->active())
            return ctx->err.fail(AVN_ERR_UNSUPPORTED, "islands_apply: swept CCD is configured (avn_ccd_configure); sleeping bodies are not swept against");
        return ctx->contacts->islands_apply(enable);
    });
}
AvnStatus avn_islands_wake(AvnContext* ctx, const uint8_t* wake, AvnIslandsWake* out) { return guarded(ctx, [&] { return ctx->contacts->islands_wake(wake, out); }); }
AvnStatus avn_contacts_download_sleeping(AvnContext* ctx, uint32_t capacity, uint8_t* row_asleep, uint32_t body_count, uint8_t* body_asleep) {
    return guarded(ctx, [&] { return ctx->contacts->download_sleeping(capacity, row_asleep, body_count, body_asleep); });
}
AvnStatus avn_contacts_download_impulses(AvnContext* ctx, uint32_t capacity, void* warm_start_normal, void* warm_start_tangent, void* normal_impulse) {
    return guarded(ctx, [&] { return ctx->contacts->download_impulses(capacity, warm_start_normal, warm_start_tangent, normal_impulse); });
}

// spatial queries (queries.cu): SpatialQueryPipeline::update / cast_ray / ray_hits / aabb_intersections_with_aabb
AvnStatus avn_query_update(AvnContext* ctx, const AvnQueryColliders* colliders, uint32_t flags) {
    return guarded(ctx, [&] { return ctx->queries->update(colliders, flags); });
}
AvnStatus avn_query_cast_ray(AvnContext* ctx, const AvnRayBatch* rays, AvnRayClosest* out) {
    return guarded(ctx, [&] { return ctx->queries->cast_ray(rays, out); });
}
AvnStatus avn_query_ray_hits(AvnContext* ctx, const AvnRayBatch* rays, AvnHitList* out) {
    return guarded(ctx, [&] { return ctx->queries->ray_hits(rays, out); });
}
AvnStatus avn_query_aabb_intersections(AvnContext* ctx, uint32_t count, const void* min, const void* max, AvnHitList* out) {
    return guarded(ctx, [&] { return ctx->queries->aabb_intersections(count, min, max, out); });
}
// SpatialQueryPipeline::cast_shape / shape_hits / project_point / point_intersections / shape_intersections
AvnStatus avn_query_cast_shape(AvnContext* ctx, const AvnShapeBatch* shapes, AvnShapeClosest* out) {
    return guarded(ctx, [&] { return ctx->queries->cast_shape(shapes, out); });
}
AvnStatus avn_query_shape_hits(AvnContext* ctx, const AvnShapeBatch* shapes, AvnShapeHitList* out) {
    return guarded(ctx, [&] { return ctx->queries->shape_hits(shapes, out); });
}
AvnStatus avn_query_project_point(AvnContext* ctx, const AvnPointBatch* points, AvnPointProjection* out) {
    return guarded(ctx, [&] { return ctx->queries->project_point(points, out); });
}
AvnStatus avn_query_point_intersections(AvnContext* ctx, const AvnPointBatch* points, AvnHitList* out) {
    return guarded(ctx, [&] { return ctx->queries->point_intersections(points, out); });
}
AvnStatus avn_query_shape_intersections(AvnContext* ctx, const AvnShapeBatch* shapes, AvnHitList* out) {
    return guarded(ctx, [&] { return ctx->queries->shape_intersections(shapes, out); });
}
// MoveAndSlide::move_and_slide against the query tree
AvnStatus avn_move_and_slide(AvnContext* ctx, const AvnMoveConfig* config, const AvnMoveBatch* batch, AvnMoveResult* out) {
    return guarded(ctx, [&] { return ctx->queries->move_and_slide(config, batch, out); });
}

// swept CCD (ccd.cu): solve_swept_ccd inside avn_solver_run
AvnStatus avn_ccd_configure(AvnContext* ctx, const AvnCcdConfig* config) {
    return guarded(ctx, [&] {
        const uint32_t known = AVN_CCD_CAPSULES | AVN_CCD_HULLS;
        if (config && config->count && (config->flags & ~known))
            return ctx->err.fail(AVN_ERR_INVALID_ARGUMENT, "ccd_configure: unknown flags 0x%x (only AVN_CCD_CAPSULES and AVN_CCD_HULLS)", config->flags & ~known);
        avn::ContactsBase::AsleepBodies asleep;
        ctx->contacts->asleep_bodies(&asleep);
        if (asleep.body_asleep && config && config->count)
            return ctx->err.fail(AVN_ERR_UNSUPPORTED, "ccd_configure: sleeping is applied on this context (avn_islands_apply); sleeping bodies are not swept against");
        if (config && config->count && !(config->flags & AVN_CCD_CAPSULES) && ctx->contacts->has_capsule())
            return ctx->err.fail(AVN_ERR_UNSUPPORTED, "ccd_configure: the contact store's shape column holds a capsule; capsule times of impact are not implemented");
        if (config && config->count && !(config->flags & AVN_CCD_HULLS) && ctx->contacts->has_hull())
            return ctx->err.fail(AVN_ERR_UNSUPPORTED, "ccd_configure: the contact store's shape column holds a convex hull; hull times of impact are not implemented");
        if (config && config->count && ctx->contacts->body_frames())
            return ctx->err.fail(AVN_ERR_UNSUPPORTED, "ccd_configure: body frames are set (avn_contacts_set_body_frames); swept CCD assumes a collider at its body's origin");
        avn::CcdRows rows;
        ctx->contacts->ccd_rows(&rows);
        return ctx->ccd->configure(config, rows);
    });
}
AvnStatus avn_ccd_download(AvnContext* ctx, AvnCcdResult* out) {
    return guarded(ctx, [&] { return ctx->ccd->download(out); });
}

AvnStatus avn_get_timings(const AvnContext* ctx, AvnTimings* out) {
    if (!ctx || !out) return AVN_ERR_INVALID_ARGUMENT;
    *out = ctx->last;
    return AVN_OK;
}

AvnStatus avn_joint_levels(const AvnBodyColumns* bodies, const AvnJointSet* joints, uint32_t* out_level, uint32_t* out_level_count) {
    if (!bodies || !joints) return AVN_ERR_INVALID_ARGUMENT;
    try {
    avn::JointSchedule sch;
    std::string error;
    AvnStatus st = avn::build_joint_schedule(*bodies, *joints, sch, error);
    if (st != AVN_OK) return create_fail(st, error);
    if (out_level)
        for (size_t g = 0; g < sch.level_of_global.size(); ++g) out_level[g] = uint32_t(sch.level_of_global[g]);
    if (out_level_count) *out_level_count = uint32_t(sch.n_levels);
    return AVN_OK;
    } catch (...) {
        return AVN_ERR_OUT_OF_MEMORY;
    }
}

}  // extern "C"
