// The inverse of ReorderInvocations(20) (FirstHit/compute.glsl:236-262), shared by the device and a host test.
//
// The reference dispatches gx x gy groups of 8x8 invocations over the image and lets dispatch group (bx, by) shade the pixels
// of a swizzled group (sx, sy): the grid is cut into columns of 20 groups (the last one gx % 20 groups wide when 20 does not
// divide gx), and the dispatch groups, in row-major order, fill column after column, row by row within each column. A pixel's
// random numbers are seeded from its un-swizzled invocation id, so a kernel that starts from the pixel needs the map back.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define IDK_HD __host__ __device__ __forceinline__
#else
#define IDK_HD inline
#endif

#define IDK_REORDER_COLUMN 20u

// swizzled group (sx, sy) of a gx x gy dispatch -> the dispatch group (bx, by) that shades it
IDK_HD void reorder_invocations_inverse(uint32_t gx, uint32_t gy, uint32_t sx, uint32_t sy, uint32_t& bx, uint32_t& by) {
    const uint32_t columnIdx = sx / IDK_REORDER_COLUMN;
    const uint32_t columnWidth = columnIdx == gx / IDK_REORDER_COLUMN ? gx % IDK_REORDER_COLUMN : IDK_REORDER_COLUMN;
    const uint32_t idx = columnIdx * (gy * IDK_REORDER_COLUMN) + sy * columnWidth + sx % IDK_REORDER_COLUMN;
    bx = idx % gx;
    by = idx / gx;
}
