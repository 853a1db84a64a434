/* The device-resident step through the C ABI alone (no Python, no torch): what the Rust shim of INTEGRATION.md does per PhysicsSchedule run,
 * written in C so that it can be compiled against include/avian_b200.h and linked with libavian_b200.so in the CPU test suite
 * (tests/test_abi_cpu.py::test_c_example_compiles_and_links).  Columns are the caller's (pinned, avn_alloc_pinned) SoA buffers. */
#include <stdio.h>
#include <string.h>

#include "avian_b200.h"

typedef struct World {
    AvnBodyColumns bodies;        /* Position, Rotation, velocities, mass properties ... (solver_body/plugin.rs:174-185) */
    AvnAabbColumns aabbs;         /* AabbIntervals in the persistent order (broad_phase.rs:176-202) */
    AvnNarrowInput colliders;     /* collider poses + AABBs in collider order, body velocities */
    AvnStepParams params;
    AvnIslandsStep islands;
    int static_columns_uploaded;
} World;

/* once, and again whenever bodies / colliders are added or change kind or material */
static int configure(AvnContext* ctx, const World* w, const double* friction, const double* restitution) {
    AvnContactGraphConfig gc;
    memset(&gc, 0, sizeof gc);
    gc.body_count = w->bodies.count;
    gc.collider_count = w->colliders.collider_count;
    gc.body_kind = w->bodies.kind;
    gc.friction = friction;
    gc.restitution = restitution;
    if (avn_contacts_configure(ctx, &gc) != AVN_OK) return -1;
    AvnIslandsConfig ic;
    memset(&ic, 0, sizeof ic);
    ic.body_count = w->bodies.count;
    ic.body_kind = w->bodies.kind;
    ic.time_to_sleep = 0.5f;
    ic.length_unit = 1.0f;
    return avn_islands_configure(ctx, &ic) == AVN_OK ? 0 : -1;
}

/* one PhysicsSchedule run: BroadPhase -> NarrowPhase -> Solver -> Sleeping */
static int step(AvnContext* ctx, World* w, AvnContactStep* stats) {
    uint64_t new_pairs = 0;
    AvnNarrowParams np;
    np.dt = w->params.dt;
    np.contact_tolerance = 0.005;
    const uint32_t keep = w->static_columns_uploaded;
    if (avn_broadphase_upload(ctx, &w->aabbs) != AVN_OK) return -1;          /* collect_collision_pairs (broad_phase.rs:373-487) */
    if (avn_broadphase_run(ctx) != AVN_OK) return -1;
    if (avn_solver_prefetch_bodies(ctx, &w->bodies, keep ? AVN_BODIES_STATIC_UNCHANGED : 0u) != AVN_OK) return -1;
    if (avn_contacts_step(ctx, &np, &w->colliders, w->params.match_contacts, w->params.length_unit,
                          AVN_CONTACTS_TAKE_BROADPHASE_PAIRS | (keep ? AVN_CONTACTS_SHAPES_UNCHANGED : 0u), stats) != AVN_OK) return -1;
    if (avn_broadphase_download_order(ctx, &new_pairs) != AVN_OK) return -1;  /* aabbs.order_out: next step's persistent order */
    if (avn_solver_upload_resident(ctx, &w->params, &w->bodies, NULL) != AVN_OK) return -1;
    if (avn_solver_run(ctx) != AVN_OK) return -1;                            /* run_substep_schedule + restitution + writeback */
    if (avn_solver_download(ctx) != AVN_OK) return -1;                       /* Position, Rotation, velocities back in the columns */
    w->islands.delta_secs = (float)w->params.dt;
    w->islands.linear_velocity = w->bodies.linear_velocity;
    w->islands.angular_velocity = w->bodies.angular_velocity;
    if (avn_islands_step(ctx, &w->islands) != AVN_OK) return -1;            /* island labels + Sleeping flags for the shim to apply */
    w->static_columns_uploaded = 1;
    return 0;
}

int main(void) {
    AvnConfig cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.abi_version = AVN_ABI_VERSION;
    cfg.scalar_bits = 32;
    AvnContext* ctx = NULL;
    if (avn_create(&cfg, &ctx) != AVN_OK) {          /* no CPU fallback: fails without an H100 */
        fprintf(stderr, "avn_create: %s\n", avn_last_error(NULL));
        return 1;
    }
    World w;
    memset(&w, 0, sizeof w);                          /* an empty world: zero bodies, zero colliders */
    AvnContactStep stats;
    int rc = 0;
    uint8_t no_kind = 0;
    w.bodies.kind = &no_kind;
    w.params.dt = 1.0 / 60.0; w.params.h = w.params.dt / 8; w.params.substeps = 8;
    if (configure(ctx, &w, NULL, NULL) != 0 || step(ctx, &w, &stats) != 0) {
        fprintf(stderr, "%s\n", avn_last_error(ctx));
        rc = 1;
    }
    avn_destroy(ctx);
    return rc;
}
