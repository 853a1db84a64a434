// The device view of the convex hull table (avn_set_convex_hulls, DESIGN.md §7k), without the geometry: what the context, the AABB updater and
// the kernels' arguments need.  csrc/hull_math.hpp derives the table and holds the contact geometry that reads it.
#pragma once
#include <cstdint>

namespace hm {

// A read-only view of the table (host vectors or device buffers).  Per hull h: vertices [voff[h], voff[h+1]) of vert, faces
// [foff[h], foff[h+1]) of plane / loff, edges [eoff[h], eoff[h+1]) of edge.  Face f's loop is loop[loff[f] .. loff[f+1]) (hull-local vertex
// indices, counter-clockwise from outside), its plane {n, d} with n unit and outward: dot(n, x) <= d inside.  An edge is {v0, v1, f0, f1}
// (hull-local vertex and face indices): f0 holds the directed edge v0 -> v1, f1 the reverse.  centre: the vertex mean; radius: max |v|.
struct Table {
    uint32_t count;
    const double* vert; const double* plane; const double* centre; const double* radius;
    const uint32_t* voff; const uint32_t* foff; const uint32_t* loff; const uint32_t* loop; const uint32_t* eoff; const uint32_t* edge;
};

}  // namespace hm
