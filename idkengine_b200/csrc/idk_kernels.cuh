// Wavefront path-tracing kernels for sm_90a (H100). See DESIGN.md for the HBM layout and the
// algorithmic-byte accounting of each kernel.
//
//   k_prepare_triangles/vertices/surfaces  scene upload: 48-byte triangle records, decoded vertex frames, per-mesh surfaces
//   k_init_sample        per sample: zero alive counts and work tickets
//   k_raygen             FirstHit/compute.glsl:44-81   ray generation (camera, jitter, thin lens)
//   k_traverse           BVHIntersect.glsl:27-105,183-291  closest hit, one ray per lane (primary rays, TLAS walk)
//   k_traverse2          same per-ray operation sequence, warp-level SETUP/BOX/LEAF phase scheduling with lane refill
//   k_shade              FirstHit/compute.glsl:100-234, NHit/compute.glsl:91-215 (barrier-free, state in place)
//   k_compact            the ordered (canonical) outcome of the alive-list atomics, decoupled look-back scan
//   k_accumulate         FinalDraw/compute.glsl:24-62; k_accumulate_scatter: fused with the NVLink peer gather
//   k_trace_rays         stand-alone closest-hit batch (BVH.Intersect analogue)
#pragma once
#include "idk_device.cuh"
#include "../../include/idk_gpu_types.h"

#define IDK_BLOCK 256
#define IDK_WARPS (IDK_BLOCK / 32)
#ifndef IDK_T2_BLOCK
#define IDK_T2_BLOCK 256     // threads per block of k_traverse2 (smaller blocks hand their registers / shared memory back sooner in the tail of a launch)
#endif

struct DeviceScene {
    const float4* nodes;          // 2 x float4 per GpuBlasNode
    const float4* triRec;         // IDK_TRI_STRIDE x float4 per triangle: (p0.xyz,e1.x) (e1.yz,e2.xy) (e2.z,n.xyz) [pad]
    const int4* blasTris;         // GpuBlasTriangle
    const GpuBlasDesc* descs;
    const GpuBlasInstance* instances;
    const float4* xforms;         // 9 x float4 per GpuMeshTransform
    const GpuMesh* meshes;
    const GpuMaterial* materials;
    const uint4* vertices;        // GpuVertex
    const GpuLight* lights;
    uint32_t instanceCount;
    uint32_t lightCount;
    float skyR, skyG, skyB;
    int stackSize;
    const float4* skyFaces;       // 6 faces x skyFaceSize^2 rgba32f texels (+X,-X,+Y,-Y,+Z,-Z), null = constant colour
    int skyFaceSize;
    const float4* tlasNodes;      // 2 x float4 per GpuTlasNode, root at 0 (USE_TLAS path, BVHIntersect.glsl:205-272)
    int useTlas;
    int treeletNodes;             // node indices < treeletNodes (BFS-first re-layout, single-BLAS scenes) are staged in shared memory
    const float4* vtxFrame;       // device-private, 2 x float4 per vertex: decoded (normal.xyz, tangent.x) (tangent.yz, 0, 0)
    const float4* surfRec;        // device-private, 5 x float4 per mesh: GetSurface + SurfaceApplyModificatons, see k_prepare_surfaces
    const struct TexRec* textures; // material texture table (handle k > 0 = textures[k - 1]; 0 = the reference's 1x1 white fallback)
    uint32_t textureCount;
    const float* srgbLut;         // 256-entry sRGB -> linear decode table
};


#define IDK_TLAS_STACK_SIZE 24   // BVHIntersect.glsl:4

// 64-byte per-slot path state (slot = position in the alive list of the current bounce).
struct __align__(16) PathState {
    float ox, oy, oz, prevIor;     // Origin, PreviousIOROrTraverseCost
    float pdx, pdy;                // PackedDirectionX/Y (octahedral)
    uint32_t pix;                  // tile-local ray index (y_local * W + x)
    uint32_t reseed;               // FirstHit only: gl_GlobalInvocationID.y*4096 + .x (un-swizzled)
    float tx, ty, tz;              // Throughput
    uint32_t rng;                  // FirstHit only: RNG state after ray generation
    float rx, ry, rz;              // Radiance
    uint32_t pad;
};
static_assert(sizeof(PathState) == 64, "PathState must be 64 bytes");

struct HitRec { float bx, by, t; uint32_t tri; };   // 16 bytes, + uint32 transform id in a second array

struct TraceCounters { unsigned long long steps, tris, instances, hits; unsigned int maxSteps[64];
                       unsigned long long phaseRounds[4], phaseLanes[4], boxIdle[4]; };   // IDK_PHASE_STATS builds: warp rounds / active lanes per phase (SETUP, BOX, LEAF, TLAS)
#ifndef IDK_PHASE_STATS
#define IDK_PHASE_STATS 0
#endif

// ------------------------------------------------------------------------------------------------
// Per sample: zero the alive counts and the work tickets, counts[0] = number of primary rays.
__global__ void k_init_sample(uint32_t* counts, int nCounts, uint32_t* tickets, int nTickets, uint32_t primaryRays) {
    for (int i = threadIdx.x; i < nCounts; i += blockDim.x) counts[i] = i == 0 ? primaryRays : 0u;
    for (int i = threadIdx.x; i < nTickets; i += blockDim.x) tickets[i] = 0u;
}

__global__ void k_prepare_triangles(const int4* __restrict__ tris, const float* __restrict__ positions,
                                    float4* __restrict__ triRec, uint32_t count) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    int4 t = tris[i];
    f3 p0 = mk3(positions[3 * t.x], positions[3 * t.x + 1], positions[3 * t.x + 2]);
    f3 p1 = mk3(positions[3 * t.y], positions[3 * t.y + 1], positions[3 * t.y + 2]);
    f3 p2 = mk3(positions[3 * t.z], positions[3 * t.z + 1], positions[3 * t.z + 2]);
    f3 e1 = p1 - p0, e2 = p2 - p0;
    f3 n = cross3(e1, e2);
    triRec[IDK_TRI_STRIDE * (size_t)i + 0] = make_float4(p0.x, p0.y, p0.z, e1.x);
    triRec[IDK_TRI_STRIDE * (size_t)i + 1] = make_float4(e1.y, e1.z, e2.x, e2.y);
    triRec[IDK_TRI_STRIDE * (size_t)i + 2] = make_float4(e2.z, n.x, n.y, n.z);
#if IDK_TRI_STRIDE == 4
    triRec[IDK_TRI_STRIDE * (size_t)i + 3] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#endif
}

// Scene upload: DecompressSR11G11B10 of every vertex normal / tangent (Compression.glsl:11-32), hoisted out of the
// per-hit path (same fp32 operations, same bits).
__global__ void k_prepare_vertices(const uint4* __restrict__ vertices, float4* __restrict__ vtxFrame, uint32_t count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint4 v = vertices[i];
    const f3 n = decompress_sr11g11b10(v.w), t = decompress_sr11g11b10(v.z);
    vtxFrame[2 * (size_t)i] = make_float4(n.x, n.y, n.z, t.x);
    vtxFrame[2 * (size_t)i + 1] = make_float4(t.y, t.z, 0.0f, 0.0f);
}

// Scene upload / mesh-material edits: with constant (1x1 white) textures the Surface of a hit depends only on its mesh:
// GetSurface(material) (Surface.glsl:49-77) followed by SurfaceApplyModificatons(mesh) (Surface.glsl:85-96).
//   [0] Albedo.xyz, Alpha   [1] Emissive.xyz, Metallic   [2] Absorbance.xyz, Roughness
//   [3] Transmission, IOR, AlphaCutoff, NormalMapStrength   [4] flags (bit0 IsVolumetric, bit1 TintOnTransmissive,
//   bit2 material has textures: the record is then only valid for the flags; surface_textured() evaluates the hit)
__global__ void k_prepare_surfaces(const GpuMesh* __restrict__ meshes, const GpuMaterial* __restrict__ materials,
                                   float4* __restrict__ surfRec, uint32_t meshCount) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= meshCount) return;
    const GpuMesh& mesh = meshes[i];
    const GpuMaterial& mat = materials[mesh.MaterialId];
    const uint32_t c = mat.BaseColorFactor;
    const f3 albedo = mk3((float)(c & 255u) / 255.0f, (float)((c >> 8) & 255u) / 255.0f, (float)((c >> 16) & 255u) / 255.0f);
    const float alpha = (float)((c >> 24) & 255u) / 255.0f;
    f3 emissive = mk3(mat.EmissiveFactor[0], mat.EmissiveFactor[1], mat.EmissiveFactor[2]);
    emissive = emissive * 1.0f + mesh.EmissiveBias * albedo;
    const f3 ab = mk3(mat.Absorbance[0], mat.Absorbance[1], mat.Absorbance[2]) + mk3(mesh.AbsorbanceBias[0], mesh.AbsorbanceBias[1], mesh.AbsorbanceBias[2]);
    const f3 absorbance = mk3(fmaxf(ab.x, 0.0f), fmaxf(ab.y, 0.0f), fmaxf(ab.z, 0.0f));
    const float metallic = clamp1(mat.MetallicFactor + mesh.SpecularBias, 0.0f, 1.0f);
    const float roughness = clamp1(mat.RoughnessFactor + mesh.RoughnessBias, 0.0f, 1.0f);
    const float transmission = clamp1(mat.TransmissionFactor + mesh.TransmissionBias, 0.0f, 1.0f);
    const float ior = fmaxf(mat.IOR + mesh.IORBias, 1.0f);
    const bool textured = (mat.BaseColorTexture | mat.MetallicRoughnessTexture | mat.NormalTexture | mat.EmissiveTexture | mat.TransmissionTexture) != 0;
    const uint32_t flags = (mat.IsVolumetric != 0 ? 1u : 0u) | (mesh.TintOnTransmissive != 0 ? 2u : 0u) | (textured ? 4u : 0u);
    float4* o = surfRec + 5 * (size_t)i;
    o[0] = make_float4(albedo.x, albedo.y, albedo.z, alpha);
    o[1] = make_float4(emissive.x, emissive.y, emissive.z, metallic);
    o[2] = make_float4(absorbance.x, absorbance.y, absorbance.z, roughness);
    o[3] = make_float4(transmission, ior, mat.AlphaCutoff, mesh.NormalMapStrength);
    o[4] = make_float4(__uint_as_float(flags), 0.0f, 0.0f, 0.0f);
}

// ------------------------------------------------------------------------------------------------
// IntersectBlas (BVHIntersect.glsl:27-105) for one local-space ray. `stack` points at this thread's column of the
// shared stack (stride IDK_BLOCK), exactly the reference's `shared uint BlasTraversalStack[SIZE][LOCAL_SIZE]`.
template <bool STATS>
__device__ __forceinline__ bool intersect_blas(const DeviceScene& sc, const float4* nodes, uint32_t triOffset, f3 lo, f3 ld, f3 inv,
                                               bool rootTest, uint32_t* stack, HitRec& hit, uint32_t& S, uint32_t& T, float& cost) {
    float tMinLeft, tMinRight;
    if (rootTest) {   // #if !USE_TLAS
        const float4 a = ldg4(nodes + 2), b = ldg4(nodes + 3);   // root = node 1
        if (!(ray_box(lo, inv, a, b, tMinLeft) && tMinLeft < hit.t)) return false;
    }
    bool blasHit = false;
    uint32_t sp = 0;
    uint32_t top = 2;
    while (true) {
        if (STATS) { S++; cost += 1.0f; }
        const NodePair pr = ldg_pair(nodes + 2 * (size_t)top);
        const float4 lA = pr.lA, lB = pr.lB, rA = pr.rA, rB = pr.rB;
        const int lChild = __float_as_int(lA.w), lCount = __float_as_int(lB.w);
        const int rChild = __float_as_int(rA.w), rCount = __float_as_int(rB.w);

        const bool hitLeft = ray_box(lo, inv, lA, lB, tMinLeft) && tMinLeft <= hit.t;
        const bool hitRight = ray_box(lo, inv, rA, rB, tMinRight) && tMinRight <= hit.t;

        const bool intersectLeft = hitLeft && lCount > 0;
        const bool intersectRight = hitRight && rCount > 0;
        if (intersectLeft || intersectRight) {
            uint32_t first = intersectLeft ? (uint32_t)lChild : (uint32_t)rChild;
            uint32_t end = !intersectRight ? (uint32_t)(lChild + lCount) : (uint32_t)(rChild + rCount);
            first += triOffset;
            end += triOffset;
            if (STATS) { T += end - first; cost += (float)(end - first) * 1.1f; }
            for (uint32_t i = first; i < end; i++) {
                float4 a, b, c;
                ldg_tri(sc.triRec, i, a, b, c);
                float bx, by, t;
                if (ray_triangle(lo, ld, mk3(a.x, a.y, a.z), mk3(a.w, b.x, b.y), mk3(b.z, b.w, c.x), mk3(c.y, c.z, c.w), bx, by, t) && t < hit.t) {
                    blasHit = true;
                    hit.tri = i;
                    hit.bx = bx;
                    hit.by = by;
                    hit.t = t;
                }
            }
        }

        const bool traverseLeft = hitLeft && lCount == 0;
        const bool traverseRight = hitRight && rCount == 0;
        if (traverseLeft || traverseRight) {
            if (traverseLeft && traverseRight) {
                const bool leftCloser = tMinLeft < tMinRight;
                top = leftCloser ? (uint32_t)lChild : (uint32_t)rChild;
                stack[(sp++) * IDK_BLOCK] = leftCloser ? (uint32_t)rChild : (uint32_t)lChild;
            } else {
                top = traverseLeft ? (uint32_t)lChild : (uint32_t)rChild;
            }
        } else {
            if (sp == 0) break;
            top = stack[(--sp) * IDK_BLOCK];
        }
    }
    return blasHit;
}

// One BLAS instance: local ray (Ray.glsl:7-12) + IntersectBlas.
template <bool STATS>
__device__ __forceinline__ void trace_instance(const DeviceScene& sc, uint32_t inst, f3 o, f3 d, bool rootTest, uint32_t* stack,
                                               HitRec& hit, uint32_t& hitXform, uint32_t& S, uint32_t& T, uint32_t& I, float& cost) {
    const GpuBlasInstance bi = sc.instances[inst];
    const int nodeOffset = sc.descs[bi.BlasId].NodeOffset;
    const uint32_t triOffset = (uint32_t)sc.descs[bi.BlasId].TriangleOffset;
    const float4* xf = sc.xforms + 9 * (size_t)bi.MeshTransformId + 3;   // InvModelMatrix rows
    const float4 r0 = ldg4(xf), r1 = ldg4(xf + 1), r2 = ldg4(xf + 2);
    const f3 lo = xform_point(r0, r1, r2, o);
    const f3 ld = xform_vector(r0, r1, r2, d);
    const f3 inv = mk3(1.0f / ld.x, 1.0f / ld.y, 1.0f / ld.z);
    if (STATS) I++;
    if (intersect_blas<STATS>(sc, sc.nodes + 2 * (size_t)nodeOffset, triOffset, lo, ld, inv, rootTest, stack, hit, S, T, cost)) hitXform = bi.MeshTransformId;
}

// TraceRay (BVHIntersect.glsl:183-291): lights, then the instance loop (default) or the TLAS walk.
template <bool STATS>
__device__ __forceinline__ void trace_closest(const DeviceScene& sc, f3 o, f3 d, float tMax, bool traceLights,
                                              uint32_t* stack, HitRec& hit, uint32_t& hitXform,
                                              uint32_t& S, uint32_t& T, uint32_t& I, float& cost) {
    hit.t = tMax;
    hit.tri = ~0u;
    hit.bx = 0.0f;
    hit.by = 0.0f;
    hitXform = 0;

    if (traceLights) {
        for (uint32_t i = 0; i < sc.lightCount; i++) {
            const GpuLight& L = sc.lights[i];
            float tMin, tMx;
            if (ray_sphere(o, d, mk3(L.Position[0], L.Position[1], L.Position[2]), L.Radius, tMin, tMx) && tMin < hit.t) {
                hit.t = tMin < 0.0f ? tMx : tMin;
                hitXform = i;
                hit.tri = ~0u;
            }
        }
    }

    if (sc.useTlas) {
        const f3 inv = mk3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
        uint32_t tstack[IDK_TLAS_STACK_SIZE];
        uint32_t sp = 0, top = 0;
        while (true) {
            const float4 pA = ldg4(sc.tlasNodes + 2 * (size_t)top);
            const uint32_t word = __float_as_uint(pA.w);
            const uint32_t id = word & 0x7FFFFFFFu;
            if (word >> 31) {
                trace_instance<STATS>(sc, id, o, d, false, stack, hit, hitXform, S, T, I, cost);
                if (sp == 0) break;
                top = tstack[--sp];
                continue;
            }
            const NodePair pr = ldg_pair(sc.tlasNodes + 2 * (size_t)id);
            const float4 lA = pr.lA, lB = pr.lB, rA = pr.rA, rB = pr.rB;
            float tMinLeft, tMinRight;
            const bool traverseLeft = ray_box(o, inv, lA, lB, tMinLeft) && tMinLeft < hit.t;
            const bool traverseRight = ray_box(o, inv, rA, rB, tMinRight) && tMinRight < hit.t;
            if (traverseLeft || traverseRight) {
                if (traverseLeft && traverseRight) {
                    const bool leftCloser = tMinLeft < tMinRight;
                    top = leftCloser ? id : id + 1;
                    tstack[sp++] = leftCloser ? id + 1 : id;
                } else {
                    top = traverseLeft ? id : id + 1;
                }
            } else {
                if (sp == 0) break;
                top = tstack[--sp];
            }
        }
    } else {
        for (uint32_t inst = 0; inst < sc.instanceCount; inst++) trace_instance<STATS>(sc, inst, o, d, true, stack, hit, hitXform, S, T, I, cost);
    }
}

struct TraverseArgs {
    DeviceScene sc;
    const PathState* state;        // indexed by perm[gid] (or gid)
    const uint32_t* perm;          // may be null
    const uint32_t* count;         // alive count of this bounce (device)
    uint32_t* ticket;              // dynamic fetch counter (zeroed per launch)
    HitRec* hits;                  // by gid
    uint32_t* hitXform;            // by gid
    float* debugCost;              // by gid, STATS only
    TraceCounters* counters;       // STATS only
    int traceLights;
    int bounce;
};

// Persistent warps: every warp repeatedly claims 32 consecutive slots of the alive list.
template <bool STATS>
__global__ void __launch_bounds__(IDK_BLOCK) k_traverse(TraverseArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t count = *a.count;
    uint32_t S = 0, T = 0, I = 0, H = 0;
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(a.ticket, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= count) break;
        const uint32_t gid = base + lane;
        if (gid < count) {
            const uint32_t src = a.perm ? a.perm[gid] : gid;
            const float4* sp = reinterpret_cast<const float4*>(a.state + src);
            const float4 s0 = sp[0], s1 = sp[1];
            const f3 o = mk3(s0.x, s0.y, s0.z);
            const f3 d = decode_unit_vec(s1.x, s1.y);
            HitRec hit;
            uint32_t xf;
            float cost = 0.0f;
            const uint32_t stepsBefore = S;
            trace_closest<STATS>(a.sc, o, d, IDK_FLOAT_MAX, a.traceLights != 0, stack, hit, xf, S, T, I, cost);
            if (STATS) atomicMax(&a.counters->maxSteps[a.bounce & 63], S - stepsBefore);
            reinterpret_cast<float4*>(a.hits)[gid] = make_float4(hit.bx, hit.by, hit.t, __uint_as_float(hit.tri));
            a.hitXform[gid] = xf;
            if (STATS) {
                a.debugCost[gid] = cost;
                if (hit.tri != ~0u) H++;
            }
        }
    }
    if (STATS) {
        for (int off = 16; off > 0; off >>= 1) {
            S += __shfl_down_sync(0xffffffffu, S, off);
            T += __shfl_down_sync(0xffffffffu, T, off);
            I += __shfl_down_sync(0xffffffffu, I, off);
            H += __shfl_down_sync(0xffffffffu, H, off);
        }
        if (lane == 0) {
            atomicAdd(&a.counters->steps, (unsigned long long)S);
            atomicAdd(&a.counters->tris, (unsigned long long)T);
            atomicAdd(&a.counters->instances, (unsigned long long)I);
            atomicAdd(&a.counters->hits, (unsigned long long)H);
        }
    }
}


// ------------------------------------------------------------------------------------------------
// k_traverse2: the production traversal kernel. Same per-ray operation sequence as trace_closest (hence the same
// bits and the same S/T/I counters), but the warp is scheduled as a small state machine so that divergent work is
// batched instead of serialised:
//   SETUP  lanes whose ray is finished write their hit, claim a new slot (one atomicAdd per warp for all needy
//          lanes -- persistent threads with lane refill) and set up the next BLAS instance (local ray, root test);
//   BOX    lanes test one sibling pair, decide descend / pop (independent of the leaf results, exactly as in the
//          reference where hitLeft/hitRight are evaluated before the triangle loop) and park a pending leaf range;
//   LEAF   lanes with a pending range test ONE triangle.
// Each iteration the warp votes (ballots) which phase to run: a phase runs when enough lanes wait for it or nothing
// else can run. Traversal stacks live in shared memory, one column per thread (the reference's layout).
struct TraverseTuning { int setupThreshold; int leafThreshold; int packRays; int setupThresholdStaged; int packCta; };   // packRays: 32 rays per warp whatever the count (throughput mode: several samples share the SMs)

// TMA (bulk async copy) staging of the hot top of the BVH into shared memory: one elected thread arms an mbarrier with
// the byte count and issues cp.async.bulk global -> shared; every thread then waits on the barrier phase.
__device__ __forceinline__ void tma_stage_treelet(void* smemDst, const void* gmemSrc, uint32_t bytes, uint64_t* mbar) {
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(mbar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(smemDst);
        const uint32_t chunk = 16384u;
        for (uint32_t off = 0; off < bytes; off += chunk) {
            const uint32_t n = min(chunk, bytes - off);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst + off), "l"((const char*)gmemSrc + off), "r"(n), "r"(bar) : "memory");
        }
    }
    uint32_t done = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(0u) : "memory");
    }
}

// Staged ray fetch (IDK_STAGED_FETCH): in the bulk regime every warp owns a double-buffered shared-memory staging area of
// 2 x 32 ray records. A batch = one ticket of 32 consecutive alive-list slots; its alive-list indices are loaded coalesced
// and the 32-byte head of every ray's PathState is copied global -> shared with cp.async (LDGSTS) one batch AHEAD of its use,
// and the ticket of the batch after that is already in a register. A SETUP round then hands rays out of shared memory
// instead of walking the dependent chain atomicAdd -> alive[] -> PathState (three L2/HBM round trips) for a dozen lanes at
// a time; that makes SETUP rounds cheap enough to run them for few waiting lanes (lower setupThreshold, fewer idle lanes
// in the BOX rounds). Which lane traces which ray changes; what is traced does not.
#ifndef IDK_STAGE_CG
#define IDK_STAGE_CG 0
#endif
#ifndef IDK_STAGE_GSS
#define IDK_STAGE_GSS 1
#endif
#define IDK_STAGE_BYTES ((IDK_T2_BLOCK / 32) * 2 * 32 * 32)
__device__ __forceinline__ void cp_async16(void* smemDst, const void* gmemSrc) {
#if IDK_STAGE_CG
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smemDst)), "l"(gmemSrc) : "memory");
#else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smemDst)), "l"(gmemSrc) : "memory");
#endif
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <bool STATS, bool TREELET, bool TLAS>
__global__ void __launch_bounds__(IDK_T2_BLOCK) k_traverse2(TraverseArgs a, TraverseTuning tune) {
    // dynamic shared memory: [treelet: treeletNodes x 32 B][traversal stacks: stackSize x IDK_T2_BLOCK x 4 B][ray staging: IDK_STAGE_BYTES]
    extern __shared__ __align__(128) unsigned char s_dyn[];
    __shared__ __align__(8) uint64_t s_mbar;
    const DeviceScene& sc = a.sc;
    const uint32_t treeletNodes = TREELET ? (uint32_t)sc.treeletNodes : 0u;
    const float4* s_treelet = reinterpret_cast<const float4*>(s_dyn);
    uint32_t* s_stack = reinterpret_cast<uint32_t*>(s_dyn + (size_t)treeletNodes * 32);
    if (TREELET && treeletNodes) tma_stage_treelet(s_dyn, sc.nodes, treeletNodes * 32u, &s_mbar);
    uint32_t* stack = s_stack + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t laneLt = (1u << lane) - 1u;
    const uint32_t count = *a.count;
    enum { ST_SETUP = 0, ST_BOX = 1, ST_LEAF = 2, ST_EXIT = 3, ST_TLAS = 4 };
    // Latency regime (few rays, e.g. late bounces or a 1/8 screen tile): spread the rays over ALL resident warps instead
    // of packing 32 per warp -- a warp that carries few rays has short BOX/LEAF/SETUP rounds and little L1 wavefront
    // serialisation, so the longest ray (which bounds the launch) finishes sooner. quota = rays per warp, 32 in the bulk.
    // Pipelined launches (packRays): a launch with few rays needs few CTAs. Only the first ceil(count / (block * packRays)) CTAs take
    // part, the others retire at once and leave their registers / shared memory to the other samples' kernels (a CTA that keeps one
    // busy warp holds a quarter of an SM). packCta = rays per thread a participating CTA is expected to take (1 = tightest packing, 0 = every CTA takes part).
    if (tune.packCta > 0 && (uint64_t)blockIdx.x * (IDK_T2_BLOCK * (uint32_t)tune.packCta) >= (uint64_t)count && blockIdx.x > 0) return;
    const uint32_t totalWarps = gridDim.x * (IDK_T2_BLOCK / 32);
    const uint32_t quota = tune.packRays ? 32u : min(32u, max(1u, (count + totalWarps - 1) / totalWarps));
#if IDK_STAGED_FETCH
    const bool bulk = quota == 32u;     // staged fetch in the throughput regime only; the latency regime keeps one ticket per SETUP round
    const int setupThreshold = max(1, min(bulk ? tune.setupThresholdStaged : tune.setupThreshold, (int)(quota * 3 / 8)));
#else
    const int setupThreshold = max(1, min(tune.setupThreshold, (int)(quota * 3 / 8)));
#endif
    const int leafThreshold = max(1, min(tune.leafThreshold, (int)(quota / 8)));
#if IDK_FAST_VOTE
    const int fastBox = 33 - min(setupThreshold, leafThreshold);   // > 32 (never) when a threshold is 1
#endif

    int state = ST_SETUP;
    bool haveRay = false, finished = false, blasHit = false;
    uint32_t gid = 0, inst = 0, curXf = 0, hitXf = 0;
    f3 wo = mk3(0, 0, 0), wd = mk3(0, 0, 1);
    f3 lo = wo, ld = wd, inv = wd;
    HitRec hit;
    hit.bx = hit.by = 0.0f; hit.t = 0.0f; hit.tri = ~0u;
    const float4* nodes = sc.nodes;
    uint32_t triOffset = 0, top = 2, sp = 0, first = 0, end = 0;
    uint32_t S = 0, T = 0, I = 0, H = 0, rayS0 = 0;
    float cost = 0.0f;
    // Traversal stack: the top IDK_REG_STACK entries live in registers (rs[0] = top, `rc` of them valid), everything below
    // them in this thread's shared-memory column (`sp` entries). Registers spill one entry when full and refill one when
    // empty, so a ray that oscillates around one depth never touches shared memory and a pop's next node index is
    // available without a load in the dependent chain. The sequence of popped values is that of the reference's array stack.
#if IDK_REG_STACK > 0
    uint32_t rs[IDK_REG_STACK];
#pragma unroll
    for (int k = 0; k < IDK_REG_STACK; k++) rs[k] = 0;
    uint32_t rc = 0;
#endif
    // TLAS walk (BVHIntersect.glsl:205-272): per-lane stack of IDK_TLAS_STACK_SIZE entries (local memory: touched once per
    // TLAS node, i.e. rarely next to the BLAS steps), `ttop` = the TLAS node to visit next.
    uint32_t tstack[TLAS ? IDK_TLAS_STACK_SIZE : 1];
    uint32_t tsp = 0, ttop = 0;
    f3 winv = wd;

#if IDK_REG_STACK > 0
#define IDK_STACK_RESET() do { sp = 0; rc = 0; } while (0)
#define IDK_STACK_EMPTY() (rc == 0u && sp == 0u)
#define IDK_STACK_PUSH(x) do {                                                         \
        if (rc == IDK_REG_STACK) { stack[(sp++) * IDK_T2_BLOCK] = rs[IDK_REG_STACK - 1]; rc = IDK_REG_STACK - 1; } \
        _Pragma("unroll") for (int k_ = IDK_REG_STACK - 1; k_ > 0; k_--) rs[k_] = rs[k_ - 1]; \
        rs[0] = (x); rc++;                                                             \
    } while (0)
#define IDK_STACK_POP(dst) do {                                                        \
        if (rc == 0u) { rs[0] = stack[(--sp) * IDK_T2_BLOCK]; rc = 1; }                   \
        (dst) = rs[0];                                                                 \
        _Pragma("unroll") for (int k_ = 0; k_ < IDK_REG_STACK - 1; k_++) rs[k_] = rs[k_ + 1]; \
        rc--;                                                                          \
    } while (0)
#else
#define IDK_STACK_RESET() do { sp = 0; } while (0)
#define IDK_STACK_EMPTY() (sp == 0u)
#define IDK_STACK_PUSH(x) do { stack[(sp++) * IDK_T2_BLOCK] = (x); } while (0)
#define IDK_STACK_POP(dst) do { (dst) = stack[(--sp) * IDK_T2_BLOCK]; } while (0)
#endif
    // a BLAS has been exhausted: commit its hit, then the instance loop advances (SETUP) or the TLAS walk pops / ends
#define IDK_BLAS_DONE() do {                                                           \
        if (blasHit) hitXf = curXf;                                                    \
        if (TLAS) {                                                                    \
            if (tsp == 0u) { inst = 0xFFFFFFFFu; state = ST_SETUP; }                   \
            else { ttop = tstack[--tsp]; state = ST_TLAS; }                            \
        } else { inst++; state = ST_SETUP; }                                           \
    } while (0)

#if IDK_STAGED_FETCH
    float4* const stage = reinterpret_cast<float4*>(s_dyn + (size_t)treeletNodes * 32 + (size_t)sc.stackSize * IDK_T2_BLOCK * 4) + (size_t)(threadIdx.x >> 5) * (2 * 32 * 2);
    uint32_t curBase = 0, curCount = 0, curNext = 0, nxtBase = 0, pendBase = 0, bufCur = 0, nxtCnt = 32, pendCnt = 32, lastBase = 0;
    // Guided self-scheduling: a ticket covers 32 slots while plenty of rays remain and shrinks to 4 as the list drains (judged
    // from the newest ticket this warp has seen), so that the batches a warp holds in advance do not unbalance the tail.
#define IDK_GRAB(dst, cnt) do {                                                          \
        const uint32_t rem_ = count > lastBase ? count - lastBase : 0u;                  \
        (cnt) = IDK_STAGE_GSS ? min(32u, max(4u, rem_ / (2u * totalWarps))) : 32u;       \
        uint32_t b_ = 0; if (lane == 0) b_ = atomicAdd(a.ticket, (cnt));                 \
        (dst) = __shfl_sync(0xffffffffu, b_, 0); lastBase = (dst);                       \
    } while (0)
#define IDK_ISSUE(buf, base, cnt) do {                                                   \
        const uint32_t g_ = (base) + lane;                                               \
        if (lane < (cnt) && g_ < count) {                                                \
            const uint32_t src_ = a.perm ? a.perm[g_] : g_;                              \
            const float4* sp_ = reinterpret_cast<const float4*>(a.state + src_);         \
            float4* d_ = stage + ((buf) * 32 + lane) * 2;                                \
            cp_async16(d_, sp_); cp_async16(d_ + 1, sp_ + 1);                            \
        }                                                                                \
        cp_async_commit();                                                               \
    } while (0)
    if (bulk) {
        uint32_t b1, c0;
        IDK_GRAB(curBase, c0); IDK_ISSUE(0u, curBase, c0);
        IDK_GRAB(b1, nxtCnt); IDK_ISSUE(1u, b1, nxtCnt);
        IDK_GRAB(pendBase, pendCnt);
        nxtBase = b1;
        curCount = curBase < count ? min(c0, count - curBase) : 0u;
        cp_async_wait<1>();
        __syncwarp();
    }
#endif
#if IDK_PHASE_STATS
    uint32_t pr0 = 0, pr1 = 0, pr2 = 0, pl0 = 0, pl1 = 0, pl2 = 0, pw0 = 0, pw2 = 0, pwx = 0;   // pw*: lanes idle during BOX rounds (waiting for SETUP / LEAF, exited)
#endif
    for (;;) {
        const uint32_t mBox = __ballot_sync(0xffffffffu, state == ST_BOX);
#if IDK_FAST_VOTE
        // Fast path: with this many lanes in BOX neither the SETUP nor the LEAF (nor the TLAS) threshold can be met by the
        // remaining lanes, so the full vote would pick BOX anyway -- skip its three other ballots (same schedule, fewer instructions).
        const bool boxOnly = __popc(mBox) >= fastBox;
        const uint32_t mSetup = boxOnly ? 0u : __ballot_sync(0xffffffffu, state == ST_SETUP);
        const uint32_t mLeaf = boxOnly ? 0u : __ballot_sync(0xffffffffu, state == ST_LEAF);
        const uint32_t mTlas = (TLAS && !boxOnly) ? __ballot_sync(0xffffffffu, state == ST_TLAS) : 0u;
#else
        const uint32_t mSetup = __ballot_sync(0xffffffffu, state == ST_SETUP);
        const uint32_t mLeaf = __ballot_sync(0xffffffffu, state == ST_LEAF);
        const uint32_t mTlas = TLAS ? __ballot_sync(0xffffffffu, state == ST_TLAS) : 0u;
#endif
        if ((mSetup | mBox | mLeaf | mTlas) == 0u) break;
#if IDK_PHASE_STATS
        if (mSetup && (__popc(mSetup) >= setupThreshold || (mBox | mLeaf | mTlas) == 0u)) { pr0++; pl0 += __popc(mSetup); }
        else if (mLeaf && (__popc(mLeaf) >= leafThreshold || mBox == 0u)) { pr2++; pl2 += __popc(mLeaf); }
        else { pr1++; pl1 += __popc(mBox); pw0 += __popc(mSetup); pw2 += __popc(mLeaf); pwx += 32 - __popc(mSetup | mBox | mLeaf | mTlas); }
#endif

        if (mSetup && (__popc(mSetup) >= setupThreshold || (mBox | mLeaf | mTlas) == 0u)) {
            // ------------------------------------------------------------------ SETUP
            const bool mine = state == ST_SETUP;
            if (mine && haveRay && inst >= sc.instanceCount) {
                reinterpret_cast<float4*>(a.hits)[gid] = make_float4(hit.bx, hit.by, hit.t, __uint_as_float(hit.tri));
                a.hitXform[gid] = hitXf;
                if (STATS) {
                    a.debugCost[gid] = cost;
                    if (hit.tri != ~0u) H++;
                    atomicMax(&a.counters->maxSteps[a.bounce & 63], S - rayS0);
                }
                haveRay = false;
            }
            const bool needFetch = mine && !haveRay && lane < quota;
            if (mine && !haveRay && lane >= quota) state = ST_EXIT;
            const uint32_t fm = __ballot_sync(0xffffffffu, needFetch);
            if (fm) {
                bool got = false, exhausted = true;     // exhausted: a lane that got no ray will never get one (end of the alive list)
                float4 s0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), s1 = s0;
#if IDK_STAGED_FETCH
                if (bulk) {
                    const uint32_t need = (uint32_t)__popc(fm), rank = (uint32_t)__popc(fm & laneLt);
                    if (needFetch && curNext + rank < curCount) {
                        const float4* r_ = stage + (bufCur * 32 + curNext + rank) * 2;
                        s0 = r_[0]; s1 = r_[1];
                        gid = curBase + curNext + rank;
                        got = true;
                    }
                    if (curNext + need >= curCount) {
                        // current batch used up: the prefetched one becomes current, the vacated buffer receives the batch whose
                        // ticket is already here, and the ticket after that is requested (its value is needed one swap later)
                        const uint32_t served = curCount - curNext;
                        cp_async_wait<0>();
                        __syncwarp();
                        bufCur ^= 1u;
                        curBase = nxtBase;
                        curCount = curBase < count ? min(nxtCnt, count - curBase) : 0u;
                        IDK_ISSUE(bufCur ^ 1u, pendBase, pendCnt);
                        nxtBase = pendBase; nxtCnt = pendCnt;
                        IDK_GRAB(pendBase, pendCnt);
                        if (needFetch && !got && rank - served < curCount) {
                            const float4* r_ = stage + (bufCur * 32 + (rank - served)) * 2;
                            s0 = r_[0]; s1 = r_[1];
                            gid = curBase + (rank - served);
                            got = true;
                        }
                        curNext = min(curCount, need - served);
                    } else {
                        curNext += need;
                    }
                    exhausted = curBase >= count;    // otherwise an unserved lane (small guided batches) asks again next SETUP round
                } else
#endif
                {
                    const int leader = __ffs(fm) - 1;
                    uint32_t base = 0;
                    if ((int)lane == leader) base = atomicAdd(a.ticket, (uint32_t)__popc(fm));
                    base = __shfl_sync(0xffffffffu, base, leader);
                    if (needFetch) {
                        gid = base + __popc(fm & laneLt);
                        if (gid < count) {
                            const uint32_t src = a.perm ? a.perm[gid] : gid;
                            const float4* spp = reinterpret_cast<const float4*>(a.state + src);
                            s0 = spp[0]; s1 = spp[1];
                            got = true;
                        }
                    }
                }
                if (needFetch) {
                    if (got) {
                        wo = mk3(s0.x, s0.y, s0.z);
                        wd = decode_unit_vec(s1.x, s1.y);
                        hit.t = IDK_FLOAT_MAX; hit.tri = ~0u; hit.bx = 0.0f; hit.by = 0.0f;
                        hitXf = 0;
                        cost = 0.0f;
                        if (a.traceLights) {
                            for (uint32_t i = 0; i < sc.lightCount; i++) {
                                const GpuLight& L = sc.lights[i];
                                float tMin, tMx;
                                if (ray_sphere(wo, wd, mk3(L.Position[0], L.Position[1], L.Position[2]), L.Radius, tMin, tMx) && tMin < hit.t) {
                                    hit.t = tMin < 0.0f ? tMx : tMin;
                                    hitXf = i;
                                    hit.tri = ~0u;
                                }
                            }
                        }
                        inst = 0;
                        haveRay = true;
                        rayS0 = S;
                        if (TLAS) {   // the walk starts at the TLAS root (node 0) with the world-space ray
                            winv = mk3(1.0f / wd.x, 1.0f / wd.y, 1.0f / wd.z);
                            ttop = 0; tsp = 0;
                            state = ST_TLAS;
                        }
                    } else if (exhausted) {
                        state = ST_EXIT;
                    }
                }
            }
            if (!TLAS && mine && haveRay && inst < sc.instanceCount) {
                const GpuBlasInstance bi = sc.instances[inst];
                const int nodeOffset = sc.descs[bi.BlasId].NodeOffset;
                triOffset = (uint32_t)sc.descs[bi.BlasId].TriangleOffset;
                const float4* xf = sc.xforms + 9 * (size_t)bi.MeshTransformId + 3;
                const float4 r0 = ldg4(xf), r1 = ldg4(xf + 1), r2 = ldg4(xf + 2);
                lo = xform_point(r0, r1, r2, wo);
                ld = xform_vector(r0, r1, r2, wd);
                inv = mk3(1.0f / ld.x, 1.0f / ld.y, 1.0f / ld.z);
                nodes = sc.nodes + 2 * (size_t)nodeOffset;
                curXf = bi.MeshTransformId;
                if (STATS) I++;
                const float4 ra = ldg4(nodes + 2), rb = ldg4(nodes + 3);
                float tRoot;
                if (ray_box(lo, inv, ra, rb, tRoot) && tRoot < hit.t) {
                    state = ST_BOX;
                    top = 2; IDK_STACK_RESET(); blasHit = false; finished = false;
                } else {
                    inst++;
                }
            }
        } else if (TLAS && mTlas && (__popc(mTlas) >= setupThreshold || (mBox | mLeaf) == 0u)) {
            // ------------------------------------------------------------------ TLAS (one node of the top-level walk)
            if (state == ST_TLAS) {
                const float4 pA = ldg4(sc.tlasNodes + 2 * (size_t)ttop);
                const uint32_t word = __float_as_uint(pA.w);
                const uint32_t id = word & 0x7FFFFFFFu;
                if (word >> 31) {
                    // leaf: IntersectBlas of instance `id` without the root test (BVHIntersect.glsl:226-243)
                    const GpuBlasInstance bi = sc.instances[id];
                    const int nodeOffset = sc.descs[bi.BlasId].NodeOffset;
                    triOffset = (uint32_t)sc.descs[bi.BlasId].TriangleOffset;
                    const float4* xf = sc.xforms + 9 * (size_t)bi.MeshTransformId + 3;
                    const float4 r0 = ldg4(xf), r1 = ldg4(xf + 1), r2 = ldg4(xf + 2);
                    lo = xform_point(r0, r1, r2, wo);
                    ld = xform_vector(r0, r1, r2, wd);
                    inv = mk3(1.0f / ld.x, 1.0f / ld.y, 1.0f / ld.z);
                    nodes = sc.nodes + 2 * (size_t)nodeOffset;
                    curXf = bi.MeshTransformId;
                    if (STATS) I++;
                    state = ST_BOX;
                    top = 2; IDK_STACK_RESET(); blasHit = false; finished = false;
                } else {
                    const NodePair pr = ldg_pair(sc.tlasNodes + 2 * (size_t)id);
                    float tMinLeft, tMinRight;
                    const bool traverseLeft = ray_box(wo, winv, pr.lA, pr.lB, tMinLeft) && tMinLeft < hit.t;
                    const bool traverseRight = ray_box(wo, winv, pr.rA, pr.rB, tMinRight) && tMinRight < hit.t;
                    if (traverseLeft || traverseRight) {
                        if (traverseLeft && traverseRight) {
                            const bool leftCloser = tMinLeft < tMinRight;
                            ttop = leftCloser ? id : id + 1;
                            tstack[tsp++] = leftCloser ? id + 1 : id;
                        } else {
                            ttop = traverseLeft ? id : id + 1;
                        }
                    } else if (tsp == 0u) {
                        inst = 0xFFFFFFFFu;        // walk finished: SETUP writes the hit and fetches the next ray
                        state = ST_SETUP;
                    } else {
                        ttop = tstack[--tsp];
                    }
                }
            }
        } else if (mLeaf && (__popc(mLeaf) >= leafThreshold || mBox == 0u)) {
            // ------------------------------------------------------------------ LEAF (one triangle)
            if (state == ST_LEAF) {
#if IDK_LEAF_LOOP
                do {      // the lane's whole pending range in one round (leaves hold 1-2 triangles with the reference's build settings)
#endif
                float4 ta, tb, tc;
                ldg_tri(sc.triRec, first, ta, tb, tc);
                float bx, by, t;
                if (ray_triangle(lo, ld, mk3(ta.x, ta.y, ta.z), mk3(ta.w, tb.x, tb.y), mk3(tb.z, tb.w, tc.x), mk3(tc.y, tc.z, tc.w), bx, by, t) && t < hit.t) {
                    blasHit = true;
                    hit.tri = first; hit.bx = bx; hit.by = by; hit.t = t;
                }
                first++;
#if IDK_LEAF_LOOP
                } while (first != end);
#endif
                if (first == end) {
                    if (finished) IDK_BLAS_DONE();
                    else state = ST_BOX;
                }
            }
        } else {
            // ------------------------------------------------------------------ BOX (one sibling pair)
#if IDK_BOX_LOOP
            // While (nearly) every lane stays in BOX no other phase can reach its threshold, so the full four-ballot vote would pick
            // BOX again: stay in this loop with one ballot per round instead (same schedule, fewer instructions).
            const int boxStay = 33 - min(setupThreshold, leafThreshold);
            do {
#endif
            if (state == ST_BOX) {
                if (STATS) { S++; cost += 1.0f; }
                float4 lA, lB, rA, rB;
                if (TREELET && top < treeletNodes) {       // hot top of the tree: shared memory (single-BLAS scenes, nodes == sc.nodes)
                    const float4* np = s_treelet + 2 * (size_t)top;
                    lA = np[0]; lB = np[1]; rA = np[2]; rB = np[3];
                } else {
                    const NodePair pr = ldg_pair(nodes + 2 * (size_t)top);
                    lA = pr.lA; lB = pr.lB; rA = pr.rA; rB = pr.rB;
                }
                const int lChild = __float_as_int(lA.w), lCount = __float_as_int(lB.w);
                const int rChild = __float_as_int(rA.w), rCount = __float_as_int(rB.w);
                float tMinLeft, tMinRight;
                const bool hitLeft = ray_box(lo, inv, lA, lB, tMinLeft) && tMinLeft <= hit.t;
                const bool hitRight = ray_box(lo, inv, rA, rB, tMinRight) && tMinRight <= hit.t;
                const bool intersectLeft = hitLeft && lCount > 0;
                const bool intersectRight = hitRight && rCount > 0;
                bool pending = false;
                if (intersectLeft || intersectRight) {
                    first = (intersectLeft ? (uint32_t)lChild : (uint32_t)rChild) + triOffset;
                    end = (!intersectRight ? (uint32_t)(lChild + lCount) : (uint32_t)(rChild + rCount)) + triOffset;
                    if (STATS) { T += end - first; cost += (float)(end - first) * 1.1f; }
                    pending = first < end;
                }
                const bool traverseLeft = hitLeft && lCount == 0;
                const bool traverseRight = hitRight && rCount == 0;
                if (traverseLeft || traverseRight) {
                    if (traverseLeft && traverseRight) {
                        const bool leftCloser = tMinLeft < tMinRight;
                        top = leftCloser ? (uint32_t)lChild : (uint32_t)rChild;
                        IDK_STACK_PUSH(leftCloser ? (uint32_t)rChild : (uint32_t)lChild);
                    } else {
                        top = traverseLeft ? (uint32_t)lChild : (uint32_t)rChild;
                    }
                } else if (IDK_STACK_EMPTY()) {
                    finished = true;
                } else {
                    IDK_STACK_POP(top);
                }
                if (pending) {
                    state = ST_LEAF;
                } else if (finished) {
                    IDK_BLAS_DONE();
                }
            }
#if IDK_BOX_LOOP
            } while (__popc(__ballot_sync(0xffffffffu, state == ST_BOX)) >= boxStay);
#endif
        }
    }
#undef IDK_STACK_RESET
#undef IDK_STACK_EMPTY
#undef IDK_STACK_PUSH
#undef IDK_STACK_POP
#undef IDK_BLAS_DONE
#if IDK_STAGED_FETCH
#undef IDK_GRAB
#undef IDK_ISSUE
    cp_async_wait<0>();     // a prefetched batch beyond the end of the list may still be in flight
#endif
#if IDK_PHASE_STATS
    if (lane == 0) {
        atomicAdd(&a.counters->phaseRounds[0], (unsigned long long)pr0); atomicAdd(&a.counters->phaseLanes[0], (unsigned long long)pl0);
        atomicAdd(&a.counters->phaseRounds[1], (unsigned long long)pr1); atomicAdd(&a.counters->phaseLanes[1], (unsigned long long)pl1);
        atomicAdd(&a.counters->phaseRounds[2], (unsigned long long)pr2); atomicAdd(&a.counters->phaseLanes[2], (unsigned long long)pl2);
        atomicAdd(&a.counters->boxIdle[0], (unsigned long long)pw0); atomicAdd(&a.counters->boxIdle[1], (unsigned long long)pw2); atomicAdd(&a.counters->boxIdle[2], (unsigned long long)pwx);
    }
#endif
    if (STATS) {
        for (int off = 16; off > 0; off >>= 1) {
            S += __shfl_down_sync(0xffffffffu, S, off);
            T += __shfl_down_sync(0xffffffffu, T, off);
            I += __shfl_down_sync(0xffffffffu, I, off);
            H += __shfl_down_sync(0xffffffffu, H, off);
        }
        if (lane == 0) {
            atomicAdd(&a.counters->steps, (unsigned long long)S);
            atomicAdd(&a.counters->tris, (unsigned long long)T);
            atomicAdd(&a.counters->instances, (unsigned long long)I);
            atomicAdd(&a.counters->hits, (unsigned long long)H);
        }
    }
}

// Stand-alone batch: rays in, hits out (IdkPtRay / IdkPtHit of idkpt.h), per-ray S/T always reported.
struct TraceRaysArgs {
    DeviceScene sc;
    const float4* rays;   // 2 x float4 per ray
    uint4* hits;          // 2 x uint4 per hit
    uint32_t count;
    uint32_t* ticket;
    int traceLights;
};

__global__ void __launch_bounds__(IDK_BLOCK) k_trace_rays(TraceRaysArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(a.ticket, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= a.count) break;
        const uint32_t gid = base + lane;
        if (gid < a.count) {
            const float4 r0 = a.rays[2 * (size_t)gid], r1 = a.rays[2 * (size_t)gid + 1];
            HitRec hit;
            uint32_t xf, S = 0, T = 0, I = 0;
            float cost = 0.0f;
            trace_closest<true>(a.sc, mk3(r0.x, r0.y, r0.z), mk3(r1.x, r1.y, r1.z), r0.w, a.traceLights != 0, stack, hit, xf, S, T, I, cost);
            a.hits[2 * (size_t)gid] = make_uint4(__float_as_uint(hit.bx), __float_as_uint(hit.by), __float_as_uint(hit.t), hit.tri);
            a.hits[2 * (size_t)gid + 1] = make_uint4(xf, S, T, 0u);
        }
    }
}

// ------------------------------------------------------------------------------------------------
struct FrameParams {
    float invProj[16];
    float invView[16];
    float viewPos[3];
    float focalLength, lenseRadius;
    int width, height;             // full image
    int stripeH, tileIndex, tileCount;
    uint32_t accumulatedSamples;
    int doDebugTraversal, doTraceLights, doRussianRoulette;
};

__device__ __forceinline__ bool tile_owns_row(const FrameParams& f, int y, int& localRow) {
    const int stripe = y / f.stripeH;
    if (f.tileCount > 1 && (stripe % f.tileCount) != f.tileIndex) return false;
    localRow = (f.tileCount > 1 ? (stripe / f.tileCount) : stripe) * f.stripeH + (y % f.stripeH);
    return true;
}

// One thread per (un-swizzled) invocation of the reference's 8x8 FirstHit dispatch.
__global__ void __launch_bounds__(64) k_raygen(FrameParams f, PathState* __restrict__ state) {
    // ReorderInvocations(20), FirstHit/compute.glsl:236-262
    const uint32_t n = 20;
    const uint32_t idx = blockIdx.y * gridDim.x + blockIdx.x;
    const uint32_t columnSize = gridDim.y * n;
    const uint32_t fullColumnCount = gridDim.x / n;
    const uint32_t lastColumnWidth = gridDim.x % n;
    const uint32_t columnIdx = idx / columnSize;
    const uint32_t idxInColumn = idx % columnSize;
    uint32_t columnWidth = n;
    if (columnIdx == fullColumnCount) columnWidth = lastColumnWidth;
    const uint32_t swy = idxInColumn / columnWidth;
    const uint32_t swx = idxInColumn % columnWidth + columnIdx * n;
    const int x = (int)(swx * 8 + threadIdx.x), y = (int)(swy * 8 + threadIdx.y);
    if (x >= f.width || y >= f.height) return;
    int localRow;
    if (!tile_owns_row(f, y, localRow)) return;

    const uint32_t gidX = blockIdx.x * 8 + threadIdx.x, gidY = blockIdx.y * 8 + threadIdx.y;
    uint32_t seed = (uint32_t)(y * 4096 + x) * (f.accumulatedSamples + 1u);
    const float sx = rnd01(seed), sy = rnd01(seed);
    const float ndcx = ((float)x + sx) / (float)f.width * 2.0f - 1.0f;
    const float ndcy = ((float)y + sy) / (float)f.height * 2.0f - 1.0f;
    const float rvx = f.invProj[0] * ndcx + f.invProj[4] * ndcy;
    const float rvy = f.invProj[1] * ndcx + f.invProj[5] * ndcy;
    f3 camDir = normalize3(mat4_mul_xyz(f.invView, rvx, rvy, -1.0f, 0.0f));
    const f3 focalPoint = mk3(f.viewPos[0], f.viewPos[1], f.viewPos[2]) + camDir * f.focalLength;
    float dx, dy;
    sample_disk(seed, dx, dy);
    const f3 pointOnLense = mat4_mul_xyz(f.invView, f.lenseRadius * dx, f.lenseRadius * dy, 0.0f, 1.0f);
    camDir = normalize3(focalPoint - pointOnLense);

    float pdx, pdy;
    encode_unit_vec(camDir, pdx, pdy);
    const uint32_t li = (uint32_t)localRow * (uint32_t)f.width + (uint32_t)x;
    float4* out = reinterpret_cast<float4*>(state + li);
    out[0] = make_float4(pointOnLense.x, pointOnLense.y, pointOnLense.z, 1.0f);
    out[1] = make_float4(pdx, pdy, __uint_as_float(li), __uint_as_float(gidY * 4096u + gidX));
    out[2] = make_float4(1.0f, 1.0f, 1.0f, __uint_as_float(seed));
    out[3] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// ------------------------------------------------------------------------------------------------
struct Surface {
    f3 Albedo; float Alpha;
    f3 Normal, Emissive, Absorbance;
    float Metallic, Roughness, Transmission, IOR, AlphaCutoff;
    bool IsVolumetric, TintOnTransmissive;
};


__device__ __forceinline__ float4 tex_sample(const DeviceScene& sc, unsigned long long handle, float u, float v) {
    return tex_sample_raw(sc.textures, sc.srgbLut, handle, u, v);
}
// Interpolate(vec2, vec2, vec2, bary) of the hit triangle's TexCoords (Math.glsl:54-57)
__device__ __forceinline__ void interp_texcoord(const DeviceScene& sc, int4 tri, float b0, float b1, float b2, float& u, float& v) {
    const uint4 v0 = __ldg(sc.vertices + tri.x), v1 = __ldg(sc.vertices + tri.y), v2 = __ldg(sc.vertices + tri.z);
    u = (__uint_as_float(v0.x) * b0 + __uint_as_float(v1.x) * b1) + __uint_as_float(v2.x) * b2;
    v = (__uint_as_float(v0.y) * b0 + __uint_as_float(v1.y) * b1) + __uint_as_float(v2.y) * b2;
}
// GetSurface(material, uv) + SurfaceApplyModificatons(mesh) (Surface.glsl:49-96) with real textures.
__device__ __forceinline__ void surface_textured(const DeviceScene& sc, int meshId, float u, float v, Surface& s) {
    const GpuMesh& mesh = sc.meshes[meshId];
    const GpuMaterial& m = sc.materials[mesh.MaterialId];
    const uint32_t c = m.BaseColorFactor;
    const float4 base = tex_sample(sc, m.BaseColorTexture, u, v);
    s.Albedo = mk3(base.x * ((float)(c & 255u) / 255.0f), base.y * ((float)((c >> 8) & 255u) / 255.0f), base.z * ((float)((c >> 16) & 255u) / 255.0f));
    s.Alpha = base.w * ((float)((c >> 24) & 255u) / 255.0f);
    const float4 nt = tex_sample(sc, m.NormalTexture, u, v);
    s.Normal = mk3(nt.x * 2.0f - 1.0f, nt.y * 2.0f - 1.0f, sqrtf(fmaxf(1.0f - (nt.x * nt.x + nt.y * nt.y), 0.0f)));   // ReconstructPackedNormal
    const float4 et = tex_sample(sc, m.EmissiveTexture, u, v);
    s.Emissive = mk3(et.x * m.EmissiveFactor[0], et.y * m.EmissiveFactor[1], et.z * m.EmissiveFactor[2]);
    s.Absorbance = mk3(m.Absorbance[0], m.Absorbance[1], m.Absorbance[2]);
    const float4 mr = tex_sample(sc, m.MetallicRoughnessTexture, u, v);
    s.Metallic = mr.x * m.MetallicFactor;
    s.Roughness = mr.y * m.RoughnessFactor;
    s.Transmission = tex_sample(sc, m.TransmissionTexture, u, v).x * m.TransmissionFactor;
    s.IOR = m.IOR;
    s.AlphaCutoff = m.AlphaCutoff;
    s.IsVolumetric = m.IsVolumetric != 0;
    // SurfaceApplyModificatons
    s.Emissive = s.Emissive * 1.0f + mesh.EmissiveBias * s.Albedo;
    const f3 ab = s.Absorbance + mk3(mesh.AbsorbanceBias[0], mesh.AbsorbanceBias[1], mesh.AbsorbanceBias[2]);
    s.Absorbance = mk3(fmaxf(ab.x, 0.0f), fmaxf(ab.y, 0.0f), fmaxf(ab.z, 0.0f));
    s.Metallic = clamp1(s.Metallic + mesh.SpecularBias, 0.0f, 1.0f);
    s.Roughness = clamp1(s.Roughness + mesh.RoughnessBias, 0.0f, 1.0f);
    s.Transmission = clamp1(s.Transmission + mesh.TransmissionBias, 0.0f, 1.0f);
    s.IOR = fmaxf(s.IOR + mesh.IORBias, 1.0f);
    s.TintOnTransmissive = mesh.TintOnTransmissive != 0;
}

// GL_TEXTURE_CUBE_MAP_SEAMLESS (the engine enables it: SkyBoxManager.cs:74): a bilinear footprint that leaves the face takes
// the texel from the face across that edge (OpenGL 4.6 spec 8.17, "seamless cube map filtering"); at a cube corner, where no
// face holds the fourth texel, the three defined texels are averaged. Coordinates are kept as odd integers c = 2*texel+1-size
// (texel centres in units of 1/size on the cube [-size, size]^3), so folding over an edge is exact integer arithmetic.
__device__ __forceinline__ void sky_face_to_cube(int face, int sc, int tc, int size, int& X, int& Y, int& Z) {
    switch (face) {   // spec table 8.19 inverted: +X (ma, -tc, -sc), -X (-ma, -tc, sc), +Y (sc, ma, tc), -Y (sc, -ma, -tc), +Z (sc, -tc, ma), -Z (-sc, -tc, -ma)
        case 0: X = size; Y = -tc; Z = -sc; break;
        case 1: X = -size; Y = -tc; Z = sc; break;
        case 2: X = sc; Y = size; Z = tc; break;
        case 3: X = sc; Y = -size; Z = -tc; break;
        case 4: X = sc; Y = -tc; Z = size; break;
        default: X = -sc; Y = -tc; Z = -size; break;
    }
}
__device__ __forceinline__ f3 sky_texel_in(const DeviceScene& sc, int face, int x, int y) {
    const float4 t = __ldg(sc.skyFaces + ((size_t)face * sc.skyFaceSize + y) * sc.skyFaceSize + x);
    return mk3(t.x, t.y, t.z);
}
// texel (x, y) of `face` where x or y (not both) may lie one texel outside the face
__device__ __forceinline__ f3 sky_texel_edge(const DeviceScene& sc, int face, int x, int y) {
    const int size = sc.skyFaceSize;
    if (x >= 0 && x < size && y >= 0 && y < size) return sky_texel_in(sc, face, x, y);
    int s2 = 2 * x + 1 - size, t2 = 2 * y + 1 - size;     // |.| == size + 1 for the coordinate that left the face
    int X, Y, Z;
    sky_face_to_cube(face, s2, t2, size, X, Y, Z);
    // fold the overhang (1 unit) over the edge: the in-plane coordinate stops at the cube surface, the old major axis retreats by it
    if (X > size || X < -size) { X = X > 0 ? size : -size; if (Y == size || Y == -size) Y += Y > 0 ? -1 : 1; else Z += Z > 0 ? -1 : 1; }
    else if (Y > size || Y < -size) { Y = Y > 0 ? size : -size; if (X == size || X == -size) X += X > 0 ? -1 : 1; else Z += Z > 0 ? -1 : 1; }
    else { Z = Z > 0 ? size : -size; if (X == size || X == -size) X += X > 0 ? -1 : 1; else Y += Y > 0 ? -1 : 1; }
    int nf, ns, nt;
    if (X == size) { nf = 0; ns = -Z; nt = -Y; } else if (X == -size) { nf = 1; ns = Z; nt = -Y; }
    else if (Y == size) { nf = 2; ns = X; nt = Z; } else if (Y == -size) { nf = 3; ns = X; nt = -Z; }
    else if (Z == size) { nf = 4; ns = X; nt = -Y; } else { nf = 5; ns = -X; nt = -Y; }
    return sky_texel_in(sc, nf, (ns + size - 1) / 2, (nt + size - 1) / 2);
}

// texture(skyBoxUBO.Albedo, dir).rgb: GL cube-map face selection (spec table 8.19), bilinear filtering, seamless across edges.
__device__ __forceinline__ f3 sample_sky(const DeviceScene& sc, f3 d) {
    if (sc.skyFaceSize == 0) return mk3(sc.skyR, sc.skyG, sc.skyB);
    const int size = sc.skyFaceSize;
    const float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
    int face;
    float scc, tc, ma;
    if (ax >= ay && ax >= az) { face = d.x >= 0.0f ? 0 : 1; scc = d.x >= 0.0f ? -d.z : d.z; tc = -d.y; ma = ax; }
    else if (ay >= az) { face = d.y >= 0.0f ? 2 : 3; scc = d.x; tc = d.y >= 0.0f ? d.z : -d.z; ma = ay; }
    else { face = d.z >= 0.0f ? 4 : 5; scc = d.z >= 0.0f ? d.x : -d.x; tc = -d.y; ma = az; }
    const float s = 0.5f * (scc / ma + 1.0f), t = 0.5f * (tc / ma + 1.0f);
    const float px = s * (float)size - 0.5f, py = t * (float)size - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    const int x0 = (int)fx0, x1 = (int)fx0 + 1, y0 = (int)fy0, y1 = (int)fy0 + 1;      // each in [-1, size]
    const bool ox0 = x0 < 0, ox1 = x1 >= size, oy0 = y0 < 0, oy1 = y1 >= size;
    f3 t00, t10, t01, t11;
    if ((ox0 || ox1) && (oy0 || oy1)) {
        // cube corner: exactly one of the four texels lies outside in both directions; it is the mean of the other three
        const bool c00 = ox0 && oy0, c10 = ox1 && oy0, c01 = ox0 && oy1;
        t00 = c00 ? mk3(0, 0, 0) : sky_texel_edge(sc, face, x0, y0);
        t10 = c10 ? mk3(0, 0, 0) : sky_texel_edge(sc, face, x1, y0);
        t01 = c01 ? mk3(0, 0, 0) : sky_texel_edge(sc, face, x0, y1);
        t11 = (c00 || c10 || c01) ? sky_texel_edge(sc, face, x1, y1) : mk3(0, 0, 0);
        const f3 mean = ((t00 + t10) + (t01 + t11)) / 3.0f;
        if (c00) t00 = mean; else if (c10) t10 = mean; else if (c01) t01 = mean; else t11 = mean;
    } else {
        t00 = sky_texel_edge(sc, face, x0, y0); t10 = sky_texel_edge(sc, face, x1, y0);
        t01 = sky_texel_edge(sc, face, x0, y1); t11 = sky_texel_edge(sc, face, x1, y1);
    }
    const f3 a = mix3(t00, t10, fx);
    const f3 b = mix3(t01, t11, fx);
    return mix3(a, b, fy);
}

struct ShadeArgs {
    DeviceScene sc;
    FrameParams f;
    PathState* state;              // pixel-indexed, updated in place (the reference's Rays[rayIndex], SSBO 30)
    float4* aov;                   // 2 x float4 per pixel, in place (SSBO 31), AOVs only
    const uint32_t* alive;         // alive list of this bounce: slot -> tile pixel; null = identity (first hit)
    const HitRec* hits;            // by slot
    const uint32_t* hitXform;
    const float* debugCost;        // by slot (debug traversal only)
    const uint32_t* count;         // alive count in
    uint32_t* survivors;           // by slot: tile pixel of a surviving ray, ~0u otherwise (input of k_compact)
    uint32_t* keysTmp;             // by slot: sort key of a surviving ray (ray sorting only), may be null
    float4* radiance;              // per tile pixel: final radiance (w = traversal cost)
    float4* aovAlbedoFinal;        // per tile pixel (AOVs only)
    float4* aovNormalFinal;
    const uint32_t* slotDelta;     // multi-GPU global slots (k_slot_exchange): per local stripe, global slot - local slot; null = local slots
    uint32_t stripePixels;         // pixels per stripe (stripe height x width)
    int exportState;               // debug export: terminated paths also write their final state back
    int firstHit;
    int lastBounce;                // survivors are final: no compaction
    int outputAovs;
};

// status word: [63:34] epoch (30 bits), [33:32] flag (1 = aggregate, 2 = inclusive prefix), [31:0] value.
// The host hands out epochs in [1, IDK_EPOCH_MASK] per lane and clears the status words when the counter wraps, so a
// stale word can never look like the current epoch (pack and compare go through the same 30-bit helpers).
#define IDK_EPOCH_MASK 0x3FFFFFFFu
__device__ __forceinline__ unsigned long long pack_status(uint32_t epoch, uint32_t flag, uint32_t value) {
    return ((unsigned long long)(epoch & IDK_EPOCH_MASK) << 34) | ((unsigned long long)flag << 32) | value;
}
__device__ __forceinline__ uint32_t status_epoch(unsigned long long sv) { return (uint32_t)(sv >> 34) & IDK_EPOCH_MASK; }

// One thread per alive ray, no block-level cooperation: every warp runs at its own pace (the ordered compaction of
// the reference's atomic alive list is a separate, uniform-cost pass over 4-byte entries: k_compact).
// TEX = the scene has material textures (idkpt_set_scene); the untextured instantiation is the north-star path.
#ifndef IDK_SHADE_MIN_BLOCKS
#define IDK_SHADE_MIN_BLOCKS 3
#endif
template <bool TEX>
__global__ void __launch_bounds__(IDK_BLOCK, IDK_SHADE_MIN_BLOCKS) k_shade(ShadeArgs a) {
    const uint32_t count = *a.count;
    const DeviceScene& sc = a.sc;
    const FrameParams& f = a.f;

    for (uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x; gid < count; gid += gridDim.x * blockDim.x) {
        bool survive = false;
        PathState st;
        float4 aov0 = make_float4(0.0f, 0.0f, 0.0f, 1.0f), aov1 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        uint32_t sortingKey = 0;
        const uint32_t src = a.alive ? a.alive[gid] : gid;
        {
            {
                const float4* sp = reinterpret_cast<const float4*>(a.state + src);
                float4 v0 = sp[0], v1 = sp[1], v2 = sp[2], v3 = sp[3];
                st.ox = v0.x; st.oy = v0.y; st.oz = v0.z; st.prevIor = v0.w;
                st.pdx = v1.x; st.pdy = v1.y; st.pix = __float_as_uint(v1.z); st.reseed = __float_as_uint(v1.w);
                st.tx = v2.x; st.ty = v2.y; st.tz = v2.z; st.rng = __float_as_uint(v2.w);
                st.rx = v3.x; st.ry = v3.y; st.rz = v3.z; st.pad = 0;
            }
            if (a.outputAovs && !a.firstHit) { aov0 = a.aov[2 * (size_t)src]; aov1 = a.aov[2 * (size_t)src + 1]; }
            // NHit's gl_GlobalInvocationID.x is the ray's slot in the alive list of the WHOLE image; a stripe tile adds the number of
            // alive rays in the other ranks' stripes above it (k_slot_exchange), so that N GPUs draw the 1-GPU random numbers
            const uint32_t slot = (a.slotDelta && !a.firstHit) ? gid + a.slotDelta[src / a.stripePixels] : gid;
            uint32_t rng = a.firstHit ? st.rng : (slot * 4096u + f.accumulatedSamples);
            const uint32_t reseed = a.firstHit ? st.reseed : slot;   // gl_GlobalInvocationID.y*4096 + .x

            const float4 hv = reinterpret_cast<const float4*>(a.hits)[gid];
            const float hitT = hv.z;
            const uint32_t hitTri = __float_as_uint(hv.w);
            const uint32_t hitXf = a.hitXform[gid];
            const bool hitScene = hitT != IDK_FLOAT_MAX;
            const f3 rayDir = decode_unit_vec(st.pdx, st.pdy);
            f3 origin = mk3(st.ox, st.oy, st.oz);
            f3 thr = mk3(st.tx, st.ty, st.tz);
            f3 rad = mk3(st.rx, st.ry, st.rz);

            if (a.firstHit && f.doDebugTraversal) {
                st.prevIor = a.debugCost[gid];
                survive = false;
            } else if (hitScene) {
                origin = origin + rayDir * hitT;
                Surface s;
                s.Albedo = mk3(1.0f, 1.0f, 1.0f); s.Alpha = 1.0f;
                s.Normal = mk3(0.0f, 0.0f, 0.0f); s.Emissive = mk3(0.0f, 0.0f, 0.0f); s.Absorbance = mk3(0.0f, 0.0f, 0.0f);
                s.Metallic = 0.0f; s.Roughness = 0.0f; s.Transmission = 0.0f; s.IOR = 1.5f; s.AlphaCutoff = 0.5f;
                s.IsVolumetric = false; s.TintOnTransmissive = true;
                f3 geometricNormal = mk3(0.0f, 0.0f, 0.0f);
                bool passThrough = false;
                const bool hitLight = hitTri == ~0u;
                if (!hitLight) {
                    sortingKey = hitTri;
                    const int4 tri = __ldg(sc.blasTris + hitTri);
                    // independent gathers issued together: vertex frames, transform, per-mesh surface record, triangle normal
                    const float4* vf = sc.vtxFrame;
                    const float4 a0 = ldg4(vf + 2 * (size_t)tri.x), a1 = ldg4(vf + 2 * (size_t)tri.x + 1);
                    const float4 c0 = ldg4(vf + 2 * (size_t)tri.y), c1 = ldg4(vf + 2 * (size_t)tri.y + 1);
                    const float4 e0 = ldg4(vf + 2 * (size_t)tri.z), e1 = ldg4(vf + 2 * (size_t)tri.z + 1);
                    const float4* xf = sc.xforms + 9 * (size_t)hitXf + 3;
                    const float4 r0 = ldg4(xf), r1 = ldg4(xf + 1), r2 = ldg4(xf + 2);
                    const float4* sr = sc.surfRec + 5 * (size_t)tri.w;
                    const float4 s0 = ldg4(sr), s1 = ldg4(sr + 1), s2 = ldg4(sr + 2), s3 = ldg4(sr + 3), s4 = ldg4(sr + 4);
                    const float b0 = hv.x, b1 = hv.y, b2 = 1.0f - hv.x - hv.y;
                    const f3 interpNormal = normalize3((mk3(a0.x, a0.y, a0.z) * b0 + mk3(c0.x, c0.y, c0.z) * b1) + mk3(e0.x, e0.y, e0.z) * b2);
                    const f3 interpTangent = normalize3((mk3(a0.w, a1.x, a1.y) * b0 + mk3(c0.w, c1.x, c1.y) * b1) + mk3(e0.w, e1.x, e1.y) * b2);
                    const float normalMapStrength = s3.w;

                    // GetSurface (1x1 white textures, Surface.glsl:49-77) + SurfaceApplyModificatons (Surface.glsl:85-96),
                    // precomputed per mesh at upload (k_prepare_surfaces)
                    s.Albedo = mk3(s0.x, s0.y, s0.z);
                    s.Alpha = s0.w;
                    s.Normal = mk3(1.0f, 1.0f, 0.0f);
                    s.Emissive = mk3(s1.x, s1.y, s1.z);
                    s.Metallic = s1.w;
                    s.Absorbance = mk3(s2.x, s2.y, s2.z);
                    s.Roughness = s2.w;
                    s.Transmission = s3.x;
                    s.IOR = s3.y;
                    s.AlphaCutoff = s3.z;
                    s.IsVolumetric = (__float_as_uint(s4.x) & 1u) != 0;
                    s.TintOnTransmissive = (__float_as_uint(s4.x) & 2u) != 0;
                    if (TEX && (__float_as_uint(s4.x) & 4u)) {
                        float tu, tv;
                        interp_texcoord(sc, tri, b0, b1, b2, tu, tv);
                        surface_textured(sc, tri.w, tu, tv, s);
                    }

                    const float alphaCutoff = (s.AlphaCutoff == 2.0f) ? rnd01(rng) : s.AlphaCutoff;
                    if (s.Alpha < alphaCutoff) {
                        origin = origin + rayDir * 0.001f;
                        passThrough = true;
                    } else {
                        const f3 worldNormal = normalize3(xform_normal(r0, r1, r2, interpNormal));
                        const f3 worldTangent = normalize3(xform_normal(r0, r1, r2, interpTangent));
                        const f3 N = normalize3(worldNormal);
                        const f3 T = normalize3(worldTangent);
                        const f3 B = normalize3(cross3(N, T));
                        const f3 tbnN = (T * s.Normal.x + B * s.Normal.y) + N * s.Normal.z;
                        s.Normal = normalize3(mix3(worldNormal, tbnN, normalMapStrength));
                        const float4 tr = ldg4(sc.triRec + IDK_TRI_STRIDE * (size_t)hitTri + 2);
                        geometricNormal = normalize3(mk3(tr.y, tr.z, tr.w));   // GetTriangleNormal
                        geometricNormal = normalize3(xform_normal(r0, r1, r2, geometricNormal));
                    }
                } else if (f.doTraceLights) {
                    sortingKey = hitXf;
                    const GpuLight& L = sc.lights[hitXf];
                    s.Emissive = mk3(L.Color[0], L.Color[1], L.Color[2]);
                    s.Albedo = s.Emissive;
                    s.Normal = (origin - mk3(L.Position[0], L.Position[1], L.Position[2])) / L.Radius;
                    geometricNormal = s.Normal;
                }

                if (passThrough) {
                    survive = true;
                } else {
                    float prevIor = a.firstHit ? 1.0f : st.prevIor;
                    const bool fromInside = dot3(-rayDir, geometricNormal) < 0.0f;
                    if (fromInside) {
                        if (a.firstHit) prevIor = s.IOR;
                        geometricNormal = geometricNormal * -1.0f;
                        if (s.IsVolumetric) {
                            const f3 e = -s.Absorbance * hitT;
                            thr = thr * mk3(det_exp(e.x), det_exp(e.y), det_exp(e.z));
                        }
                    }
                    float cosTheta = dot3(-rayDir, s.Normal);
                    if (cosTheta < 0.0f) s.Normal = s.Normal * -1.0f;

                    rad = rad + s.Emissive * thr;

                    // ---- SampleMaterial (Shading.glsl:52-150)
                    Surface m = s;
                    m.Roughness *= m.Roughness;
                    cosTheta = dot3(-rayDir, m.Normal);
                    {
                        const float diffuseChance = 1.0f - m.Metallic - m.Transmission;
                        const float r0f = (prevIor - m.IOR) / (prevIor + m.IOR);
                        const float f0 = r0f * r0f;
                        const float fres = f0 + (1.0f - f0) * pow5f(1.0f - cosTheta);
                        m.Metallic = mix1(m.Metallic, 1.0f, fres);
                        m.Transmission = fmaxf(1.0f - diffuseChance - m.Metallic, 0.0f);
                    }
                    uint32_t bsdfType;
                    {
                        const float rnd = rnd01(rng);
                        if (m.Metallic > rnd) bsdfType = 1u;
                        else if (m.Metallic + m.Transmission > rnd) bsdfType = 2u;
                        else bsdfType = 0u;
                    }
                    f3 diffuseRayDir;
                    {
                        uint32_t tmp = reseed;
                        const float g = 1.32471795724474602596f;
                        const float a1 = 1.0f / g, a2 = 1.0f / (g * g);
                        const float r2u = fract1((float)f.accumulatedSamples * a1), r2v = fract1((float)f.accumulatedSamples * a2);
                        const float po0 = rnd01(tmp), po1 = rnd01(tmp);
                        const float u = fract1(r2u + po0), v = fract1(r2v + po1);
                        diffuseRayDir = normalize3(m.Normal + sample_sphere(u, v));
                    }
                    f3 newDir, bsdf;
                    float newIor;
                    if (bsdfType == 0u) {
                        newDir = diffuseRayDir; newIor = prevIor; bsdf = m.Albedo;
                    } else if (bsdfType == 1u) {
                        newDir = normalize3(mix3(reflect3(rayDir, m.Normal), diffuseRayDir, m.Roughness));
                        bsdf = m.Albedo; newIor = prevIor;
                    } else {
                        newIor = fromInside ? 1.0f : m.IOR;
                        f3 refr;
                        bool tir;
                        if (!m.IsVolumetric) {
                            refr = rayDir; tir = false; newIor = 1.0f;
                        } else {
                            refr = refract3(rayDir, m.Normal, prevIor / newIor);
                            tir = refr.x == 0.0f && refr.y == 0.0f && refr.z == 0.0f;
                            if (tir) { refr = reflect3(rayDir, m.Normal); newIor = prevIor; }
                        }
                        newDir = normalize3(mix3(refr, !tir ? -diffuseRayDir : diffuseRayDir, m.Roughness));
                        const bool gltfWantsTint = m.IsVolumetric || !fromInside;
                        bsdf = (gltfWantsTint && m.TintOnTransmissive) ? m.Albedo : mk3(1.0f, 1.0f, 1.0f);
                    }
                    // result.Pdf = max(1.0, 0.0001) = 1.0 in every branch; bsdf / 1.0f == bsdf exactly
                    thr = thr * bsdf;

                    if (a.outputAovs) {
                        // GetSurfaceVariance uses the un-remapped surface (FirstHit:197-203)
                        const float dc = 1.0f - s.Metallic - s.Transmission;
                        const float weight = dc + s.Metallic * s.Roughness + s.Transmission * s.Roughness;
                        if (a.firstHit) {
                            const f3 al = s.Albedo * weight, no = s.Normal * weight;
                            aov0 = make_float4(al.x, al.y, al.z, 1.0f - weight);
                            aov1 = make_float4(no.x, no.y, no.z, 0.0f);
                        } else {
                            const f3 al = mk3(aov0.x, aov0.y, aov0.z) + aov0.w * s.Albedo * weight;
                            const f3 no = mk3(aov1.x, aov1.y, aov1.z) + aov0.w * s.Normal * weight;
                            aov0 = make_float4(al.x, al.y, al.z, aov0.w * (1.0f - weight));
                            aov1 = make_float4(no.x, no.y, no.z, 0.0f);
                        }
                    }

                    bool terminate = false;
                    if (!a.firstHit && f.doRussianRoulette) {
                        const float p = fmaxf(thr.x, fmaxf(thr.y, thr.z));
                        if (rnd01(rng) > p) terminate = true;
                        else thr = thr / p;
                    }
                    if (!terminate) {
                        if (bsdfType == 2u) geometricNormal = geometricNormal * -1.0f;
                        origin = origin + geometricNormal * 0.001f;
                        st.prevIor = newIor;
                        encode_unit_vec(newDir, st.pdx, st.pdy);
                        survive = true;
                    }
                }
            } else {
                const f3 albedo = sample_sky(sc, rayDir);
                if (a.outputAovs) {
                    const f3 fn = cubemap_face_normal(rayDir);
                    if (a.firstHit) {
                        aov0 = make_float4(albedo.x, albedo.y, albedo.z, 0.0f);
                        aov1 = make_float4(fn.x, fn.y, fn.z, 0.0f);
                    } else {
                        const f3 al = mk3(aov0.x, aov0.y, aov0.z) + aov0.w * albedo;
                        const f3 no = mk3(aov1.x, aov1.y, aov1.z) + aov0.w * fn;
                        aov0 = make_float4(al.x, al.y, al.z, 0.0f);
                        aov1 = make_float4(no.x, no.y, no.z, 0.0f);
                    }
                }
                rad = rad + albedo * thr;
                survive = false;
            }
            st.ox = origin.x; st.oy = origin.y; st.oz = origin.z;
            st.tx = thr.x; st.ty = thr.y; st.tz = thr.z;
            st.rx = rad.x; st.ry = rad.y; st.rz = rad.z;

            if (!survive || a.lastBounce) {
                // path is final for this sample: hand its radiance (and AOVs) to the accumulate kernel
                a.radiance[src] = make_float4(st.rx, st.ry, st.rz, st.prevIor);
                if (a.outputAovs) { a.aovAlbedoFinal[src] = aov0; a.aovNormalFinal[src] = aov1; }
            }
            if ((survive && !a.lastBounce) || a.exportState) {
                // wavefrontRaySSBO.Rays[rayIndex] = wavefrontRay (FirstHit:84, NHit:63), in place
                float4* op = reinterpret_cast<float4*>(a.state + src);
                op[0] = make_float4(st.ox, st.oy, st.oz, st.prevIor);
                op[1] = make_float4(st.pdx, st.pdy, __uint_as_float(src), 0.0f);
                op[2] = make_float4(st.tx, st.ty, st.tz, 0.0f);
                op[3] = make_float4(st.rx, st.ry, st.rz, 0.0f);
                if (a.outputAovs) { a.aov[2 * (size_t)src] = aov0; a.aov[2 * (size_t)src + 1] = aov1; }
            }
            if (!a.lastBounce) {
                a.survivors[gid] = survive ? src : ~0u;
                if (a.keysTmp) a.keysTmp[gid] = sortingKey & 0x1FFFFFu;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Ordered stream compaction of the survivor list: the canonical (ascending slot) outcome of the reference's
// `index = atomicAdd(Counts[1 - pingPong], 1); AliveRayIndices[index] = rayIndex` (FirstHit:89-97, NHit:69-77).
// Single pass, decoupled look-back over tiles of IDK_BLOCK x IDK_COMPACT_ITEMS entries; every tile costs the same,
// so the look-back never waits long (unlike doing it inside the shading kernel).
#define IDK_COMPACT_ITEMS 8
struct CompactArgs {
    const uint32_t* survivors;     // by slot: pixel or ~0u
    const uint32_t* keysTmp;       // by slot, may be null
    const uint32_t* count;
    uint32_t* aliveOut;
    uint32_t* keysOut;             // may be null
    uint32_t* countOut;
    uint32_t* ticket;
    unsigned long long* tileStatus;
    uint32_t epoch;
};

__global__ void __launch_bounds__(IDK_BLOCK) k_compact(CompactArgs a) {
    __shared__ uint32_t s_tile;
    __shared__ uint32_t s_warpCount[IDK_WARPS];
    __shared__ uint32_t s_base;
    const uint32_t count = *a.count;
    const uint32_t tileSize = IDK_BLOCK * IDK_COMPACT_ITEMS;
    const uint32_t numTiles = (count + tileSize - 1) / tileSize;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) s_tile = atomicAdd(a.ticket, 1u);
        __syncthreads();
        const uint32_t tile = s_tile;
        if (tile >= numTiles) break;
        // each thread owns IDK_COMPACT_ITEMS consecutive slots (keeps the order trivially stable)
        const uint32_t first = tile * tileSize + threadIdx.x * IDK_COMPACT_ITEMS;
        uint32_t v[IDK_COMPACT_ITEMS];
        uint32_t mine = 0;
#pragma unroll
        for (int i = 0; i < IDK_COMPACT_ITEMS; i++) {
            const uint32_t s = first + i;
            v[i] = s < count ? a.survivors[s] : ~0u;
            mine += v[i] != ~0u ? 1u : 0u;
        }
        // warp exclusive scan of per-thread counts
        uint32_t incl = mine;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t n = __shfl_up_sync(0xffffffffu, incl, off);
            if ((int)lane >= off) incl += n;
        }
        if (lane == 31) s_warpCount[warp] = incl;
        __syncthreads();
        uint32_t warpOffset = 0, blockTotal = 0;
#pragma unroll
        for (int w = 0; w < IDK_WARPS; w++) {
            const uint32_t c = s_warpCount[w];
            if (w < (int)warp) warpOffset += c;
            blockTotal += c;
        }
        if (threadIdx.x == 0) {
            uint32_t exclusive = 0;
            if (tile > 0) {
                atomicExch(&a.tileStatus[tile], pack_status(a.epoch, 1u, blockTotal));
                int look = (int)tile - 1;
                while (look >= 0) {
                    const unsigned long long sv = *((volatile unsigned long long*)&a.tileStatus[look]);
                    if (status_epoch(sv) != (a.epoch & IDK_EPOCH_MASK)) continue;   // not published yet
                    const uint32_t flag = (uint32_t)(sv >> 32) & 3u;
                    exclusive += (uint32_t)sv;
                    if (flag == 2u) break;
                    look--;
                }
            }
            __threadfence();
            atomicExch(&a.tileStatus[tile], pack_status(a.epoch, 2u, exclusive + blockTotal));
            if (tile == numTiles - 1) *a.countOut = exclusive + blockTotal;
            s_base = exclusive;
        }
        __syncthreads();
        uint32_t dst = s_base + warpOffset + (incl - mine);
#pragma unroll
        for (int i = 0; i < IDK_COMPACT_ITEMS; i++) {
            if (v[i] != ~0u) {
                a.aliveOut[dst] = v[i];
                if (a.keysOut) a.keysOut[dst] = a.keysTmp[first + i];
                dst++;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// FinalDraw/compute.glsl:24-62 over this tile's compact rows.
__device__ __forceinline__ f3 turbo_colormap(float x) {
    x = clamp1(x, 0.0f, 1.0f);
    const float v0 = 1.0f, v1 = x, v2 = x * x, v3 = x * x * x;
    const float w0 = v2 * v2, w1 = v3 * v2;
    return mk3((((v0 * 0.13572138f + v1 * 4.61539260f) + v2 * -42.66032258f) + v3 * 132.13108234f) + (w0 * -152.94239396f + w1 * 59.28637943f),
               (((v0 * 0.09140261f + v1 * 2.19418839f) + v2 * 4.84296658f) + v3 * -14.18503333f) + (w0 * 4.27729857f + w1 * 2.82956604f),
               (((v0 * 0.10667330f + v1 * 12.64194608f) + v2 * -60.58204836f) + v3 * 110.36276771f) + (w0 * -89.90310912f + w1 * 27.34824973f));
}

// ------------------------------------------------------------------------------------------------
// Multi-GPU: FinalDraw fused with the tile all-gather over NVLink peer memory. Every rank owns a full-size image
// (double-buffered) that all ranks can write (CUDA IPC mappings). The accumulate kernel of the last sample stores each
// finished pixel into its own Result tile AND into every rank's full image at the pixel's final (de-interleaved)
// position; the last CTA to finish then raises this rank's flag on every peer (release), and a one-warp kernel waits
// until all peers' flags for this frame have arrived (acquire). No NCCL call, no separate de-interleave pass.
#define IDK_MAX_PEERS 16
struct GatherArgs {
    float4* peerImage[IDK_MAX_PEERS];      // this frame's full image on every rank (own rank included)
    uint32_t* peerFlags[IDK_MAX_PEERS];    // flags[world] on every rank; entry [rank] is written by `rank`
    const int* tileRows;                   // owned image rows, ascending (device)
    uint32_t* doneCounter;                 // CTA completion counter (zeroed per frame)
    int world, rank, width;
    uint32_t epoch;
};

__global__ void __launch_bounds__(IDK_BLOCK) k_accumulate_scatter(const float4* __restrict__ radiance, float4* __restrict__ result,
                                                                  uint32_t count, uint32_t accumulatedSamples, int debugTraversal,
                                                                  GatherArgs g);

// Multi-GPU "global slots" (SURVEY 8e option ii): NHit seeds its random numbers with the ray's slot in the alive list
// (NHit/compute.glsl: gl_GlobalInvocationID.x), and in the canonical (ascending pixel) order that slot counts the alive rays of
// the WHOLE image below it. A stripe tile knows only its own rays, so once per bounce the ranks exchange their per-stripe
// alive counts over NVLink peer memory -- one 8-byte word per stripe, written straight into every peer's table, tagged with
// the exchange epoch -- and every rank prefix-sums the full table: global slot = local slot + delta[local stripe]. With this
// the N-GPU image is bit-identical to the 1-GPU image. One CTA; the alive list is ascending, so the stripe boundaries are
// binary searches. Double-buffered by epoch parity: a rank can be at most one exchange ahead of the slowest peer, because
// finishing exchange e needs every peer's word e, which a peer publishes only after it has finished reading e - 1.
#define IDK_MAX_STRIPES 4096
struct SlotExchangeArgs {
    const uint32_t* alive;                          // this bounce's alive list (ascending tile pixel)
    const uint32_t* count;
    unsigned long long* peerTable[IDK_MAX_PEERS];   // this lane's table of epoch parity `epoch & 1` on every rank: [nStripes] words
    uint32_t* delta;                                // out: [nLocalStripes]
    uint32_t* timedOut;
    long long timeoutCycles;
    uint32_t epoch;
    int world, rank;
    uint32_t stripePixels, nLocalStripes, nStripes;
};

__global__ void __launch_bounds__(256) k_slot_exchange(SlotExchangeArgs a) {
    __shared__ uint32_t s_val[IDK_MAX_STRIPES + 1];   // local stripe starts, then the global per-stripe counts / bases
    __shared__ uint32_t s_start[IDK_MAX_STRIPES / 2 + 2];
    __shared__ uint32_t s_part[256];
    const uint32_t count = *a.count;
    const uint32_t tid = threadIdx.x;
    // first alive-list index whose pixel lies in local stripe t or above
    for (uint32_t t = tid; t <= a.nLocalStripes; t += blockDim.x) {
        uint32_t lo = 0, hi = count;
        if (t == a.nLocalStripes) lo = count;
        else {
            const uint32_t firstPixel = t * a.stripePixels;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (a.alive[mid] < firstPixel) lo = mid + 1; else hi = mid;
            }
        }
        s_start[t] = lo;
    }
    __syncthreads();
    // publish: local stripe t is global stripe t * world + rank
    for (uint32_t t = tid; t < a.nLocalStripes; t += blockDim.x) {
        const unsigned long long word = ((unsigned long long)a.epoch << 32) | (unsigned long long)(s_start[t + 1] - s_start[t]);
        for (int p = 0; p < a.world; p++) *((volatile unsigned long long*)&a.peerTable[p][t * (uint32_t)a.world + (uint32_t)a.rank]) = word;
    }
    __threadfence_system();
    // collect every stripe's count of this epoch
    const unsigned long long* mine = a.peerTable[a.rank];
    const long long t0 = clock64();
    for (uint32_t s = tid; s < a.nStripes; s += blockDim.x) {
        unsigned long long w;
        for (;;) {
            w = *((volatile const unsigned long long*)&mine[s]);
            if ((uint32_t)(w >> 32) == a.epoch) break;
            if (clock64() - t0 > a.timeoutCycles) { *a.timedOut = 2u; w = 0; break; }   // a peer died: fail (idkpt_sync reports it) instead of hanging
        }
        s_val[s] = (uint32_t)w;
    }
    __syncthreads();
    // exclusive prefix sum over the stripes in image order: each thread owns a contiguous chunk
    const uint32_t chunk = (a.nStripes + blockDim.x - 1) / blockDim.x;
    const uint32_t c0 = min(tid * chunk, a.nStripes), c1 = min(c0 + chunk, a.nStripes);
    uint32_t sum = 0;
    for (uint32_t s = c0; s < c1; s++) sum += s_val[s];
    s_part[tid] = sum;
    __syncthreads();
    if (tid == 0) {
        uint32_t run = 0;
        for (uint32_t i = 0; i < blockDim.x; i++) { const uint32_t v = s_part[i]; s_part[i] = run; run += v; }
    }
    __syncthreads();
    uint32_t run = s_part[tid];
    for (uint32_t s = c0; s < c1; s++) { const uint32_t v = s_val[s]; s_val[s] = run; run += v; }
    __syncthreads();
    for (uint32_t t = tid; t < a.nLocalStripes; t += blockDim.x) a.delta[t] = s_val[t * (uint32_t)a.world + (uint32_t)a.rank] - s_start[t];
}

// timeoutCycles: SM clocks (idkpt.cu: IDKPT_GATHER_TIMEOUT_MS, default 30 s). Peers only have to have called
// idkpt_gather_import before their first gathered Compute; a rank that is still uploading its scene just makes the others
// wait here. After a timeout the frame is lost and the ranks' gather epochs may disagree: re-run export/import.
__global__ void __launch_bounds__(32) k_gather_wait(const uint32_t* flags, int world, uint32_t epoch, uint32_t* timedOut, long long timeoutCycles) {
    const int p = threadIdx.x;
    if (p < world) {
        const long long t0 = clock64();
        while (*((volatile const uint32_t*)&flags[p]) != epoch) {
            if (clock64() - t0 > timeoutCycles) { *timedOut = 1u; break; }   // a peer died; fail instead of hanging the GPU
        }
    }
    __threadfence_system();
}

__global__ void __launch_bounds__(IDK_BLOCK) k_accumulate(const float4* __restrict__ radiance, const float4* __restrict__ aovAlbedo,
                                                          const float4* __restrict__ aovNormal, float4* __restrict__ result,
                                                          float4* __restrict__ albedo, float4* __restrict__ normal,
                                                          uint32_t count, uint32_t accumulatedSamples, int debugTraversal, int outputAovs) {
    const float w = 1.0f / ((float)accumulatedSamples + 1.0f);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const float4 r = radiance[i];
        f3 nr = mk3(r.x, r.y, r.z);
        if (debugTraversal) nr = turbo_colormap(r.w / 150.0f);
        const float4 last = result[i];
        const f3 o = mix3(mk3(last.x, last.y, last.z), nr, w);
        result[i] = make_float4(o.x, o.y, o.z, 1.0f);
        if (outputAovs) {
            const float4 la = albedo[i], ln = normal[i], a = aovAlbedo[i], n = aovNormal[i];
            const f3 oa = mix3(mk3(la.x, la.y, la.z), mk3(a.x, a.y, a.z), w);
            const f3 on = mix3(mk3(ln.x, ln.y, ln.z), mk3(n.x, n.y, n.z), w);
            albedo[i] = make_float4(oa.x, oa.y, oa.z, 1.0f);
            normal[i] = make_float4(on.x, on.y, on.z, 1.0f);
        }
    }
}


__global__ void __launch_bounds__(IDK_BLOCK) k_accumulate_scatter(const float4* __restrict__ radiance, float4* __restrict__ result,
                                                                  uint32_t count, uint32_t accumulatedSamples, int debugTraversal,
                                                                  GatherArgs g) {
    __shared__ bool s_last;
    const float w = 1.0f / ((float)accumulatedSamples + 1.0f);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const float4 r = radiance[i];
        f3 nr = mk3(r.x, r.y, r.z);
        if (debugTraversal) nr = turbo_colormap(r.w / 150.0f);
        const float4 last = result[i];
        const f3 o = mix3(mk3(last.x, last.y, last.z), nr, w);
        const float4 v = make_float4(o.x, o.y, o.z, 1.0f);
        result[i] = v;
        const uint32_t row = i / (uint32_t)g.width, x = i - row * (uint32_t)g.width;
        const size_t dst = (size_t)g.tileRows[row] * (size_t)g.width + x;
        for (int p = 0; p < g.world; p++) g.peerImage[p][dst] = v;      // 16-byte stores over NVLink (P2P)
    }
    // release: all of this CTA's peer stores, then count it; the last CTA publishes the flag on every rank
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(g.doneCounter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (s_last) {
        __threadfence_system();
        if ((int)threadIdx.x < g.world) {
            *((volatile uint32_t*)&g.peerFlags[threadIdx.x][g.rank]) = g.epoch;
            __threadfence_system();
        }
    }
}

__global__ void __launch_bounds__(IDK_BLOCK) k_accumulate_aov(const float4* __restrict__ aovAlbedo, const float4* __restrict__ aovNormal,
                                                              float4* __restrict__ albedo, float4* __restrict__ normal,
                                                              uint32_t count, uint32_t accumulatedSamples) {
    const float w = 1.0f / ((float)accumulatedSamples + 1.0f);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const float4 la = albedo[i], ln = normal[i], a = aovAlbedo[i], n = aovNormal[i];
        const f3 oa = mix3(mk3(la.x, la.y, la.z), mk3(a.x, a.y, a.z), w);
        const f3 on = mix3(mk3(ln.x, ln.y, ln.z), mk3(n.x, n.y, n.z), w);
        albedo[i] = make_float4(oa.x, oa.y, oa.z, 1.0f);
        normal[i] = make_float4(on.x, on.y, on.z, 1.0f);
    }
}
