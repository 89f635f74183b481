// idkpt_add_models (ModelManager.Add, ModelManager.cs:128-216, on the device scene in place): the call's records that carry
// ids, staged on the device as the host handed them over, are written into the grown scene arrays with every id rebased
// behind the scene's old counts (BVH.Add, BVH.cs:255-272; ModelManager.cs:150-190). One thread per record of the four
// arrays, laid end to end: source triangles, meshes, materials, instances.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/idk_gpu_types.h"

struct SceneAddArgs {
    GpuBlasTriangle* tris;                 // the BLAS build's source triangles, rebased in place
    const GpuMesh* meshesIn;
    GpuMesh* meshesOut;
    const GpuMaterial* materialsIn;
    GpuMaterial* materialsOut;
    const GpuBlasInstance* instancesIn;
    GpuBlasInstance* instancesOut;
    uint64_t triCount, meshCount, materialCount, instanceCount;
    int32_t vertexOffset, meshOffset, materialOffset;
    uint32_t blasOffset, transformOffset;
    uint64_t textureOffset;                // handle k > 0 becomes k + textureOffset; 0 (the white fallback) stays 0
};

__device__ __forceinline__ uint64_t scene_add_handle(uint64_t h, uint64_t offset) { return h ? h + offset : 0; }

__global__ void k_scene_add_rebase(SceneAddArgs a) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.triCount) {
        GpuBlasTriangle t = a.tris[i];
        t.X += a.vertexOffset; t.Y += a.vertexOffset; t.Z += a.vertexOffset;
        t.MeshId += a.meshOffset;
        a.tris[i] = t;
        return;
    }
    i -= a.triCount;
    if (i < a.meshCount) {
        GpuMesh m = a.meshesIn[i];
        m.MaterialId += a.materialOffset;
        a.meshesOut[i] = m;
        return;
    }
    i -= a.meshCount;
    if (i < a.materialCount) {
        GpuMaterial m = a.materialsIn[i];
        m.BaseColorTexture = scene_add_handle(m.BaseColorTexture, a.textureOffset);
        m.MetallicRoughnessTexture = scene_add_handle(m.MetallicRoughnessTexture, a.textureOffset);
        m.NormalTexture = scene_add_handle(m.NormalTexture, a.textureOffset);
        m.EmissiveTexture = scene_add_handle(m.EmissiveTexture, a.textureOffset);
        m.TransmissionTexture = scene_add_handle(m.TransmissionTexture, a.textureOffset);
        a.materialsOut[i] = m;
        return;
    }
    i -= a.materialCount;
    if (i < a.instanceCount) {
        GpuBlasInstance b = a.instancesIn[i];
        b.BlasId += a.blasOffset;
        b.MeshTransformId += a.transformOffset;
        a.instancesOut[i] = b;
    }
}
