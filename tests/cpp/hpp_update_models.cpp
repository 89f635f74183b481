// Compile + link check of idk::PathTracer's animation calls (include/idkpt.hpp). Without a CUDA device the constructor
// throws idk::Error(IDKPT_ERR_NO_DEVICE); with one, a one-triangle scene whose transform one animated node owns is moved
// by UpdateModels and the transform and node global are read back.
#include <cmath>
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
        GpuBlasInstance inst = {};
        GpuMeshTransform xf = {};
        xf.ModelMatrix[0][0] = xf.ModelMatrix[1][1] = xf.ModelMatrix[2][2] = 1.0f;
        xf.InvModelMatrix[0][0] = xf.InvModelMatrix[1][1] = xf.InvModelMatrix[2][2] = 1.0f;
        xf.PrevModelMatrix[0][0] = xf.PrevModelMatrix[1][1] = xf.PrevModelMatrix[2][2] = 1.0f;
        GpuMesh mesh = {};
        GpuMaterial mat = {};
        const idk::PathTracer::BlasBuildResult b = pt.BuildBlas(pos, 3, &tri, 1);
        desc.NodeCount = (int32_t)b.nodes.size();
        desc.TriangleCount = (int32_t)b.triangles.size();
        desc.RequiredStackSize = b.requiredStackSize;
        GpuTlasNode tlas = {};
        tlas.IsLeafAndChildOrInstanceId = 0x80000000u;
        IdkPtSceneDesc s = {};
        s.BlasNodes = b.nodes.data(); s.BlasNodeCount = b.nodes.size();
        s.BlasTriangles = b.triangles.data(); s.BlasTriangleCount = b.triangles.size();
        s.BlasDescs = &desc; s.BlasDescCount = 1;
        s.BlasInstances = &inst; s.BlasInstanceCount = 1;
        s.TlasNodes = &tlas; s.TlasNodeCount = 1; s.UseTlas = 1;
        s.MeshTransforms = &xf; s.MeshTransformCount = 1;
        s.Meshes = &mesh; s.MeshCount = 1;
        s.Materials = &mat; s.MaterialCount = 1;
        s.Vertices = vtx; s.VertexCount = 3;
        s.VertexPositions = pos; s.VertexPositionCount = 3;
        s.BlasStackSize = b.requiredStackSize;
        pt.SetScene(s);
        IdkPtNode node = {};
        node.Parent = -1; node.MeshTransformsCount = 1;
        node.Rotation[3] = 1.0f;
        node.Scale[0] = node.Scale[1] = node.Scale[2] = 1.0f;
        node.GlobalTransform[0] = node.GlobalTransform[5] = node.GlobalTransform[10] = node.GlobalTransform[15] = 1.0f;
        const float times[2] = {0.0f, 1.0f};
        const float data[6] = {0, 0, 0, 2, 0, 0};
        IdkPtNodeAnimation ch = {};
        ch.Type = IDKPT_ANIM_TRANSLATION; ch.Mode = IDKPT_ANIM_LINEAR; ch.KeyFrameCount = 2;
        IdkPtModelAnimation anim = {0.0f, 1.0f, 0, 1, 1};
        IdkPtAnimationDesc d = {};
        d.Nodes = &node; d.NodeCount = 1;
        d.Channels = &ch; d.ChannelCount = 1;
        d.Animations = &anim; d.AnimationCount = 1;
        d.KeyFrameTimes = times; d.KeyFrameTimeCount = 2;
        d.KeyFrameData = data; d.KeyFrameDataCount = 6;
        pt.SetAnimations(d);
        const uint8_t on = 1;
        pt.EnableAnimations(0, 1, &on);
        pt.SetNodeTransforms(0, 1, &node);
        if (pt.UpdateModels(0.5f) != 3u) return 1;
        GpuMeshTransform got = {};
        pt.ReadRange(IDKPT_ARRAY_MESH_TRANSFORMS, 0, 1, &got);
        float global[16] = {};
        pt.ReadRange(IDKPT_ARRAY_NODE_GLOBAL_TRANSFORMS, 0, 1, global);
        if (got.ModelMatrix[0][3] != 1.0f || got.InvModelMatrix[0][3] != -1.0f || got.PrevModelMatrix[0][3] != 0.0f || global[12] != 1.0f) return 2;
        std::puts("OK device");
        return 0;
    } catch (const idk::Error& e) {
        if (e.status() == IDKPT_ERR_NO_DEVICE) { std::printf("OK no-device: %s\n", e.what()); return 0; }
        std::printf("FAIL: %d %s\n", e.status(), e.what());
        return 1;
    }
}
