// Compile + link check of idk::PathTracer::AddModels (include/idkpt.hpp). Without a CUDA device the constructor throws
// idk::Error(IDKPT_ERR_NO_DEVICE); with one, a one-triangle model is added to a one-triangle scene and the descs are checked.
#include <cstdio>

#include "idkpt.hpp"

int main() {
    try {
        idk::PathTracer pt(16, 16);
        const PackedVec3 pos[3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}};
        GpuVertex vtx[3] = {};
        GpuBlasTriangle tri = {};
        tri.X = 0; tri.Y = 1; tri.Z = 2;
        GpuBlasDesc desc = {};
        desc.TriangleCount = 1;
        GpuBlasInstance inst = {};
        GpuMeshTransform xf = {};
        xf.ModelMatrix[0][0] = xf.ModelMatrix[1][1] = xf.ModelMatrix[2][2] = 1.0f;
        xf.InvModelMatrix[0][0] = xf.InvModelMatrix[1][1] = xf.InvModelMatrix[2][2] = 1.0f;
        GpuMesh mesh = {};
        GpuMaterial mat = {};
        mat.BaseColorFactor = 0xFFFFFFFFu;
        const idk::PathTracer::BlasBuildResult b = pt.BuildBlas(pos, 3, &tri, 1);
        desc.NodeCount = (int32_t)b.nodes.size();
        desc.TriangleCount = (int32_t)b.triangles.size();
        desc.RequiredStackSize = b.requiredStackSize;
        IdkPtSceneDesc s = {};
        s.BlasNodes = b.nodes.data(); s.BlasNodeCount = b.nodes.size();
        s.BlasTriangles = b.triangles.data(); s.BlasTriangleCount = b.triangles.size();
        s.BlasDescs = &desc; s.BlasDescCount = 1;
        s.BlasInstances = &inst; s.BlasInstanceCount = 1;
        s.MeshTransforms = &xf; s.MeshTransformCount = 1;
        s.Meshes = &mesh; s.MeshCount = 1;
        s.Materials = &mat; s.MaterialCount = 1;
        s.Vertices = vtx; s.VertexCount = 3;
        s.VertexPositions = pos; s.VertexPositionCount = 3;
        s.BlasStackSize = b.requiredStackSize;
        pt.SetScene(s);
        GpuBlasDesc add = {};
        add.TriangleCount = 1;
        add.IsRefittable = 1;
        IdkPtAddModelsDesc m = {};
        m.Triangles = &tri; m.TriangleCount = 1;
        m.BlasDescs = &add; m.BlasDescCount = 1;
        m.BlasInstances = &inst; m.BlasInstanceCount = 1;
        m.MeshTransforms = &xf; m.MeshTransformCount = 1;
        m.Meshes = &mesh; m.MeshCount = 1;
        m.Materials = &mat; m.MaterialCount = 1;
        m.Vertices = vtx; m.VertexPositions = pos; m.VertexCount = 3;
        pt.AddModels(m);
        GpuBlasDesc descs[2] = {};
        pt.ReadRange(IDKPT_ARRAY_BLAS_DESCS, 0, 2, descs);
        if (descs[1].NodeOffset != descs[0].NodeCount || descs[1].TriangleOffset != descs[0].TriangleCount || descs[1].IsRefittable != 1) return 1;
        std::puts("OK device");
        return 0;
    } catch (const idk::Error& e) {
        if (e.status() == IDKPT_ERR_NO_DEVICE) { std::printf("OK no-device: %s\n", e.what()); return 0; }
        std::printf("FAIL: %d %s\n", e.status(), e.what());
        return 1;
    }
}
