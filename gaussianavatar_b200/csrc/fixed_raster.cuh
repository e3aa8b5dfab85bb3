// Exact integer triangle coverage shared by the UV-space position-map rasterizer (posmap.cu) and the screen-space mesh renderer
// (mesh_render.cu): window coordinates snapped to 1/256 of a pixel, int64 edge functions, and one tie rule for centres on an edge.
#pragma once
#include <cuda_runtime.h>

namespace ga {

// A window coordinate already scaled by 256 (formed exactly in fp64) -> 1/256-pixel fixed point, round half to even.
__device__ __forceinline__ long long snap_fixed(double x) { return __double2ll_rn(x); }

// edge function of (a -> b) at p: > 0 when p is to the left (y up)
__device__ __forceinline__ long long edge_fn(long long ax, long long ay, long long bx, long long by, long long px, long long py)
{
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}

// Whether a point with edge value e belongs to the face, for an edge (dx, dy) of a counter-clockwise face (y up): inside, or on an
// edge that goes down (dy < 0) or, when horizontal, to the left (dy == 0, dx < 0).  Two faces that share an edge traverse it in
// opposite directions, so each point on it belongs to exactly one of them; a face of zero area owns nothing.
__device__ __forceinline__ bool edge_owns(long long e, long long dx, long long dy)
{
    return e > 0 || (e == 0 && (dy < 0 || (dy == 0 && dx < 0)));
}

}  // namespace ga
