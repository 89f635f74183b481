// reorder_invocations_inverse (idkengine_b200/csrc/idk_reorder.h) against the forward map of ReorderInvocations(20),
// FirstHit/compute.glsl:236-262, for every group of the dispatch over each image size given as "WxH" arguments.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "idk_reorder.h"

// dispatch group (bx, by) of a gx x gy dispatch -> the swizzled group whose pixels it shades
static void reorder_invocations(uint32_t gx, uint32_t gy, uint32_t bx, uint32_t by, uint32_t& sx, uint32_t& sy) {
    const uint32_t n = 20;
    const uint32_t idx = by * gx + bx;
    const uint32_t columnSize = gy * n;
    const uint32_t fullColumnCount = gx / n;
    const uint32_t lastColumnWidth = gx % n;
    const uint32_t columnIdx = idx / columnSize;
    const uint32_t idxInColumn = idx % columnSize;
    uint32_t columnWidth = n;
    if (columnIdx == fullColumnCount) columnWidth = lastColumnWidth;
    sy = idxInColumn / columnWidth;
    sx = idxInColumn % columnWidth + columnIdx * n;
}

int main(int argc, char** argv) {
    for (int i = 1; i < argc; i++) {
        unsigned w = 0, h = 0;
        if (std::sscanf(argv[i], "%ux%u", &w, &h) != 2 || !w || !h) { std::printf("bad size %s\n", argv[i]); return 2; }
        const uint32_t gx = (w + 7) / 8, gy = (h + 7) / 8;
        std::vector<char> seen((size_t)gx * gy, 0);
        for (uint32_t by = 0; by < gy; by++)
            for (uint32_t bx = 0; bx < gx; bx++) {
                uint32_t sx, sy, ix, iy;
                reorder_invocations(gx, gy, bx, by, sx, sy);
                if (sx >= gx || sy >= gy || seen[(size_t)sy * gx + sx]) {
                    std::printf("%s: group (%u, %u) -> (%u, %u) is not a permutation\n", argv[i], bx, by, sx, sy);
                    return 1;
                }
                seen[(size_t)sy * gx + sx] = 1;
                reorder_invocations_inverse(gx, gy, sx, sy, ix, iy);
                if (ix != bx || iy != by) {
                    std::printf("%s: group (%u, %u) -> (%u, %u) -> (%u, %u)\n", argv[i], bx, by, sx, sy, ix, iy);
                    return 1;
                }
            }
        std::printf("%s: %u x %u groups OK\n", argv[i], gx, gy);
    }
    std::printf("OK\n");
    return 0;
}
