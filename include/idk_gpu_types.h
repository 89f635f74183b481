/*
 * idk_gpu_types.h -- the data contract between the IDKEngine C# host and libidkpt.
 *
 * Every struct below is byte-identical to a blittable struct the reference
 * already uploads into an SSBO/UBO; the host hands over the same arrays it
 * builds today, unchanged. File:line citations are relative to the reference
 * tree (IDKEngine/Source = SRC, IDKEngine/Resource/Shaders = SH).
 *
 * Plain C, no CUDA / torch types. Included by the C-ABI header (idkpt.h), by
 * the CUDA sources and by the host-side C++ mirror.
 */
#ifndef IDK_GPU_TYPES_H
#define IDK_GPU_TYPES_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
#define IDK_STATIC_ASSERT(c, m) static_assert(c, m)
#else
#define IDK_STATIC_ASSERT(c, m) _Static_assert(c, m)
#endif

/* SRC/GpuTypes/GpuBlasNode.cs:7-37, SH/include/GpuTypes.glsl:186-192.
 * TriCount > 0  => leaf, TriStartOrChild = first triangle (BLAS-local).
 * TriCount == 0 => interior, TriStartOrChild = left child; right = left + 1.
 * Node 0 is a 32-byte pad, node 1 the root, nodes 2/3 the root's children
 * (SRC/Bvh/BLAS.cs:16-22). */
typedef struct GpuBlasNode {
    float   Min[3];
    int32_t TriStartOrChild;
    float   Max[3];
    int32_t TriCount;
} GpuBlasNode;
IDK_STATIC_ASSERT(sizeof(GpuBlasNode) == 32, "GpuBlasNode must be 32 bytes");

/* SRC/GpuTypes/GpuBlasTriangle.cs:3-9, GpuTypes.glsl:160-164.
 * Global vertex ids (already vertex-offset rebased, SRC/Bvh/BVH.cs:265-268). */
typedef struct GpuBlasTriangle {
    int32_t X, Y, Z;
    int32_t MeshId;
} GpuBlasTriangle;
IDK_STATIC_ASSERT(sizeof(GpuBlasTriangle) == 16, "GpuBlasTriangle must be 16 bytes");

/* SRC/GpuTypes/GpuBlasDesc.cs:3-20, GpuTypes.glsl:166-178. */
typedef struct GpuBlasDesc {
    int32_t NodeOffset;
    int32_t NodeCount;
    int32_t TriangleOffset;
    int32_t TriangleCount;
    int32_t LeafIndicesOffset;
    int32_t LeafIndicesCount;
    int32_t ParentIndicesOffset;
    int32_t ParentIndicesCount;
    int32_t RequiredStackSize;
    int32_t IsRefittable; /* C# bool marshalled as 4 bytes */
} GpuBlasDesc;
IDK_STATIC_ASSERT(sizeof(GpuBlasDesc) == 40, "GpuBlasDesc must be 40 bytes");

/* SRC/GpuTypes/GpuBlasInstance.cs:3-7, GpuTypes.glsl:180-184. */
typedef struct GpuBlasInstance {
    uint32_t BlasId;
    uint32_t MeshTransformId;
} GpuBlasInstance;
IDK_STATIC_ASSERT(sizeof(GpuBlasInstance) == 8, "GpuBlasInstance must be 8 bytes");

/* SRC/GpuTypes/GpuTlasNode.cs:7-46, GpuTypes.glsl:194-200. Root at 0. */
typedef struct GpuTlasNode {
    float    Min[3];
    uint32_t IsLeafAndChildOrInstanceId; /* bit31 = leaf, low 31 = child or instance */
    float    Max[3];
    float    _pad0;
} GpuTlasNode;
IDK_STATIC_ASSERT(sizeof(GpuTlasNode) == 32, "GpuTlasNode must be 32 bytes");

/* SRC/GpuTypes/GpuMeshTransform.cs:6-54, GpuTypes.glsl:153-158 (SSBO 4 is
 * row_major, SH/include/StaticStorageBuffers.glsl:24): three 3x4 matrices,
 * each stored as 3 rows of 4 floats acting on COLUMN vectors:
 *   out[r] = Row[r].x*v.x + Row[r].y*v.y + Row[r].z*v.z + Row[r].w*v.w     */
typedef struct GpuMeshTransform {
    float ModelMatrix[3][4];
    float InvModelMatrix[3][4];
    float PrevModelMatrix[3][4];
} GpuMeshTransform;
IDK_STATIC_ASSERT(sizeof(GpuMeshTransform) == 144, "GpuMeshTransform must be 144 bytes");

/* SRC/GpuTypes/GpuMesh.cs:5-33, GpuTypes.glsl:122-145. */
typedef struct GpuMesh {
    float    LocalBoundsMin[3];
    int32_t  MaterialId;
    float    LocalBoundsMax[3];
    float    NormalMapStrength;
    float    AbsorbanceBias[3];
    int32_t  MeshletsOffset;
    int32_t  MeshletCount;
    float    EmissiveBias;
    float    SpecularBias;
    float    RoughnessBias;
    float    TransmissionBias;
    float    IORBias;
    int32_t  InstanceCount;
    int32_t  VertexCount;
    float    _pad0[3];
    int32_t  TintOnTransmissive; /* bool + 3 pad bytes */
} GpuMesh;
IDK_STATIC_ASSERT(sizeof(GpuMesh) == 96, "GpuMesh must be 96 bytes");

/* SRC/GpuTypes/GpuMaterial.cs:8-67, GpuTypes.glsl:226-248.
 * The five 64-bit slots hold GL bindless sampler handles in the reference;
 * libidkpt reads them as CUDA texture object handles, 0 = "1x1 white"
 * (the reference's own fallback, SRC/Utils/ModelLoader.cs:877-885). */
typedef struct GpuMaterial {
    float    EmissiveFactor[3];
    uint32_t BaseColorFactor;   /* unorm8 x4, R in the low byte */
    float    Absorbance[3];
    float    IOR;
    float    TransmissionFactor;
    float    RoughnessFactor;
    float    MetallicFactor;
    float    AlphaCutoff;       /* 0 = opaque, 2.0 = blend sentinel */
    uint64_t BaseColorTexture;
    uint64_t MetallicRoughnessTexture;
    uint64_t NormalTexture;
    uint64_t EmissiveTexture;
    uint64_t TransmissionTexture;
    int32_t  IsVolumetric;
    int32_t  IsDoubleSided;
} GpuMaterial;
IDK_STATIC_ASSERT(sizeof(GpuMaterial) == 96, "GpuMaterial must be 96 bytes");

/* SRC/GpuTypes/GpuVertex.cs:5-10, GpuTypes.glsl:250-255. Tangent/Normal are
 * snorm R11G11B10 (SRC/Utils/Compression.cs:21-40). */
typedef struct GpuVertex {
    float    TexCoord[2];
    uint32_t Tangent;
    uint32_t Normal;
} GpuVertex;
IDK_STATIC_ASSERT(sizeof(GpuVertex) == 16, "GpuVertex must be 16 bytes");

/* SRC/GpuTypes/GpuUnskinnedVertex.cs:5-12, GpuTypes.glsl:283-291 (scalar-packed, 52 bytes). */
typedef struct GpuUnskinnedVertex {
    uint32_t JointIndices[4];
    float    JointWeights[4];
    float    Position[3];
    uint32_t Tangent;
    uint32_t Normal;
} GpuUnskinnedVertex;
IDK_STATIC_ASSERT(sizeof(GpuUnskinnedVertex) == 52, "GpuUnskinnedVertex must be 52 bytes");

/* PackedVec3 Positions[] (SSBO 8, StaticStorageBuffers.glsl:44-47): 12 bytes. */
typedef struct PackedVec3 {
    float x, y, z;
} PackedVec3;
IDK_STATIC_ASSERT(sizeof(PackedVec3) == 12, "PackedVec3 must be 12 bytes");

/* SRC/GpuTypes/GpuLight.cs:5-45, GpuTypes.glsl:92-102 (std140, 48 bytes). */
typedef struct GpuLight {
    float   Position[3];
    float   Radius;
    float   Color[3];
    int32_t PointShadowIndex;
    float   PrevPosition[3];
    float   _pad0;
} GpuLight;
IDK_STATIC_ASSERT(sizeof(GpuLight) == 48, "GpuLight must be 48 bytes");
#define IDK_GPU_MAX_UBO_LIGHT_COUNT 256 /* StaticUniformBuffers.glsl:6 */

/* SRC/GpuTypes/GpuPointShadow.cs:7-41, GpuTypes.glsl:104-120 (std140, 432 bytes): what CpuPointShadow.GetGpuPointShadow()
 * returns. libidkpt reads Position, NearPlane, FarPlane and LightIndex; the bindless handles and the six face matrices
 * (+X,-X,+Y,-Y,+Z,-Z, OpenTK row-vector view * projection) are carried so the engine can pass the struct as it is. */
typedef struct GpuPointShadow {
    uint64_t Texture;
    uint64_t ShadowTexture;
    float    ProjViewMatrices[6][16];
    float    Position[3];
    float    NearPlane;
    uint64_t RayTracedShadowTexture;
    float    FarPlane;
    int32_t  LightIndex;
} GpuPointShadow;
IDK_STATIC_ASSERT(sizeof(GpuPointShadow) == 432, "GpuPointShadow must be 432 bytes");
IDK_STATIC_ASSERT(offsetof(GpuPointShadow, Position) == 400, "GpuPointShadow.Position offset");
IDK_STATIC_ASSERT(offsetof(GpuPointShadow, FarPlane) == 424, "GpuPointShadow.FarPlane offset");

/* SRC/GpuTypes/GpuPerFrameData.cs:5-21, GpuTypes.glsl:74-90 (UBO 1).
 * Matrices are OpenTK row-vector matrices uploaded raw, i.e. GLSL sees
 * column c = the 4 floats at [c*4 .. c*4+3]:  (M*v)[i] = sum_c M[c*4+i]*v[c]. */
typedef struct GpuPerFrameData {
    float    ProjView[16];
    float    View[16];
    float    InvView[16];
    float    PrevView[16];
    float    ViewPos[3];
    uint32_t Frame;
    float    Projection[16];
    float    InvProjection[16];
    float    InvProjView[16];
    float    PrevProjView[16];
    float    NearPlane;
    float    FarPlane;
    float    DeltaRenderTime;
    float    Time;
} GpuPerFrameData;
IDK_STATIC_ASSERT(sizeof(GpuPerFrameData) == 544, "GpuPerFrameData must be 544 bytes");
IDK_STATIC_ASSERT(offsetof(GpuPerFrameData, InvView) == 128, "InvView offset");
IDK_STATIC_ASSERT(offsetof(GpuPerFrameData, ViewPos) == 256, "ViewPos offset");
IDK_STATIC_ASSERT(offsetof(GpuPerFrameData, InvProjection) == 336, "InvProjection offset");

/* SRC/GpuTypes/GpuWavefrontRay.cs:5-15, GpuTypes.glsl:202-212. The reference's
 * internal per-pixel ray record. libidkpt keeps its wavefront state in its own
 * slot-compacted layout (DESIGN.md) but can export this layout for inspection. */
typedef struct GpuWavefrontRay {
    float Origin[3];
    float PreviousIOROrTraverseCost;
    float Throughput[3];
    float PackedDirectionX;
    float Radiance[3];
    float PackedDirectionY;
} GpuWavefrontRay;
IDK_STATIC_ASSERT(sizeof(GpuWavefrontRay) == 48, "GpuWavefrontRay must be 48 bytes");

/* SRC/GpuTypes/GpuAovRay.cs:5-11, GpuTypes.glsl:214-220. */
typedef struct GpuAovRay {
    float Albedo[3];
    float NewWeight;
    float Normal[3];
    float _pad0;
} GpuAovRay;
IDK_STATIC_ASSERT(sizeof(GpuAovRay) == 32, "GpuAovRay must be 32 bytes");

/* PathTracer.GpuSettings, SRC/Render/PathTracer.cs:127-138 (UBO 0, std140). */
typedef struct IdkPtGpuSettings {
    float   FocalLength;
    float   LenseRadius;
    int32_t DoDebugBVHTraversal;
    int32_t DoTraceLights;
    int32_t DoRussianRoulette;
} IdkPtGpuSettings;
IDK_STATIC_ASSERT(sizeof(IdkPtGpuSettings) == 20, "GpuSettings must be 20 bytes");

#endif /* IDK_GPU_TYPES_H */
