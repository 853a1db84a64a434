// The shape-column check shared by the library's units (the AABB update, the narrow phase, the contact store, the spatial queries) and the
// host fixture: host code only, no CUDA, so the fixture's g++ build includes it as the library does.
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/avian_b200.h"

namespace avn {

// The shape column of a collider set on the host, before anything is copied (a refused call changes nothing): every value at most
// AVN_SHAPE_CAPSULE (AVN_SHAPE_CONVEX_HULL where hulls are implemented: hull_count != NULL), a capsule's radius and half length not negative,
// and a hull's index integral and below *hull_count.  NULL shape = all cuboids.  Returns NULL or the reason, with the first offending collider
// in *at; *any_capsule / *any_hull (optional) tell whether the column holds a capsule / a hull, *max_hull the largest hull index it names.
inline const char* check_shape_column(const uint8_t* shape, const void* dims, size_t count, uint32_t scalar_bits, size_t* at, bool* any_capsule = nullptr,
                                      const uint32_t* hull_count = nullptr, bool* any_hull = nullptr, uint32_t* max_hull = nullptr) {
    if (any_capsule) *any_capsule = false;
    if (any_hull) *any_hull = false;
    if (max_hull) *max_hull = 0;
    if (!shape) return nullptr;
    for (size_t i = 0; i < count; ++i) {
        if (shape[i] == AVN_SHAPE_CONVEX_HULL && hull_count) {
            const double h = scalar_bits == 64 ? static_cast<const double*>(dims)[3 * i] : double(static_cast<const float*>(dims)[3 * i]);
            if (*hull_count == 0) { *at = i; return "a convex hull collider, and no hull table is set (avn_set_convex_hulls)"; }
            if (!(h >= 0 && h < double(*hull_count)) || h != double(uint32_t(h))) {
                *at = i;
                return "a convex hull's index must be integral, not negative and below the hull table's count";
            }
            if (any_hull) *any_hull = true;
            if (max_hull && uint32_t(h) > *max_hull) *max_hull = uint32_t(h);
            continue;
        }
        if (shape[i] > AVN_SHAPE_CAPSULE) {
            *at = i;
            return hull_count ? "unknown shape (AVN_SHAPE_CUBOID, AVN_SHAPE_SPHERE, AVN_SHAPE_CAPSULE and AVN_SHAPE_CONVEX_HULL are known)"
                              : "unknown shape (AVN_SHAPE_CUBOID, AVN_SHAPE_SPHERE and AVN_SHAPE_CAPSULE are known)";
        }
        if (shape[i] != AVN_SHAPE_CAPSULE) continue;
        if (any_capsule) *any_capsule = true;
        const double r = scalar_bits == 64 ? static_cast<const double*>(dims)[3 * i] : double(static_cast<const float*>(dims)[3 * i]);
        const double h = scalar_bits == 64 ? static_cast<const double*>(dims)[3 * i + 1] : double(static_cast<const float*>(dims)[3 * i + 1]);
        if (r < 0 || h < 0) { *at = i; return "a capsule's radius and half length must not be negative"; }
    }
    return nullptr;
}

}  // namespace avn
