// Compile + link check of idk::PathTracer::BuildBlases (include/idkpt.hpp). Without a CUDA device the constructor throws
// idk::Error(IDKPT_ERR_NO_DEVICE); with one, a batch of two one-triangle BLASes is built and its descs are checked.
#include <cstdio>

#include "idkpt.hpp"

int main() {
    try {
        idk::PathTracer pt(16, 16);
        const PackedVec3 pos[4] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
        GpuBlasTriangle tris[2] = {};
        tris[0].X = 0; tris[0].Y = 1; tris[0].Z = 2;
        tris[1].X = 0; tris[1].Y = 1; tris[1].Z = 3;
        GpuBlasDesc descs[2] = {};
        descs[0].TriangleOffset = 0; descs[0].TriangleCount = 1;
        descs[1].TriangleOffset = 1; descs[1].TriangleCount = 1; descs[1].IsRefittable = 1;
        const idk::PathTracer::BlasBatchResult r = pt.BuildBlases(pos, 4, tris, 2, descs, 2);
        if (r.descs.size() != 2 || r.descs[1].NodeOffset != r.descs[0].NodeCount || r.descs[1].IsRefittable != 1) return 1;
        if (r.nodes.size() != (size_t)(r.descs[0].NodeCount + r.descs[1].NodeCount) || r.sahs.size() != 2) return 1;
        std::puts("OK device");
        return 0;
    } catch (const idk::Error& e) {
        if (e.status() == IDKPT_ERR_NO_DEVICE) { std::printf("OK no-device: %s\n", e.what()); return 0; }
        std::printf("FAIL: %d %s\n", e.status(), e.what());
        return 1;
    }
}
