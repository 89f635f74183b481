// ModelManager.Update's host half on the device (idkpt_update_models): keyframe sampling, the dirty node hierarchy, the
// mesh-transform step and the joint matrices. Arithmetic in idk_anim_math.h, shared with the host mirror
// (host_mirror/animation.cpp), so every array equals the mirror's byte for byte.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "idk_anim_math.h"

#define IDK_ANIM_FLAG_NODE_MOVED 1u
#define IDK_ANIM_FLAG_INSTANCE_MOVED 2u
#define IDK_ANIM_FLAG_SINGULAR 4u
// k_anim_nodes is one block: 256 threads leave each thread the registers the double-precision inverse needs without spilling
#define IDK_ANIM_NODES_BLOCK 256

struct AnimArgs {
    const IdkPtNodeAnimation* channels;
    const IdkPtModelAnimation* animations;
    const uint32_t* enabled;            // per animation
    const idkanim::Group* groups;
    const uint32_t* pairs;
    const float* times;
    const float* data;
    const IdkPtNode* nodes;             // Parent and the transform ranges
    const uint32_t* levelNodes;
    const uint32_t* levelStart;
    const IdkPtSkin* skins;
    const uint32_t* jointNodes;
    const float* inverseJoints;
    const uint32_t* jointSlotSkin;
    const uint32_t* jointSlotJoint;
    const int32_t* owner;
    IdkPtNodeLocal* locals;             // scratch: this call's locals (start: a copy of the committed ones)
    const idkanim::M4* globals;         // committed globals ("before")
    idkanim::M4* newGlobals;            // scratch
    idkanim::M4* diffs;                 // per node with mesh transforms in the dirty set
    idkanim::M4* invSkin;               // per skin
    uint8_t* dirty;                     // scratch: pending dirty flags, then the sampled ones
    uint8_t* inSet;
    uint8_t* movedBits;                 // per owned mesh transform
    GpuMeshTransform* xforms;
    float* joints;                      // 12 floats per joint matrix
    uint32_t* flags;
    float time;
    uint32_t groupCount, levelCount, skinCount, transformCount, jointMatrixCount;
};

// One thread per (node, property) group: its channels in application order (UpdateNodeAnimations, ModelManager.cs:514-592).
__global__ void k_anim_sample(AnimArgs a) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.groupCount) return;
    const idkanim::Group gr = a.groups[g];
    IdkPtNodeLocal l = a.locals[gr.node];
    bool dirty = false;
    for (uint32_t k = gr.first; k < gr.first + gr.count; k++) {
        const uint32_t an = a.pairs[2 * k + 1];
        if (!a.enabled[an]) continue;
        if (idkanim::sampleChannel(a.channels[a.pairs[2 * k]], a.animations[an], a.time, a.times, a.data, l)) dirty = true;
    }
    if (!dirty) return;
    // groups of one node write disjoint properties
    IdkPtNodeLocal& dst = a.locals[gr.node];
    const int type = a.channels[a.pairs[2 * gr.first]].Type;
    if (type == IDKPT_ANIM_ROTATION) for (int i = 0; i < 4; i++) dst.Rotation[i] = l.Rotation[i];
    else if (type == IDKPT_ANIM_SCALE) for (int i = 0; i < 3; i++) dst.Scale[i] = l.Scale[i];
    else for (int i = 0; i < 3; i++) dst.Translation[i] = l.Translation[i];
    a.dirty[gr.node] = 1;
}

// UpdateNodeHierarchy + Node.TraverseUpdate (ModelManager.cs:482-512): one block walks the hierarchy level by level, so
// every parent's new global is in place before its children read it; then the skinned nodes' inverses.
__global__ void __launch_bounds__(IDK_ANIM_NODES_BLOCK) k_anim_nodes(AnimArgs a) {
    __shared__ uint32_t anyMoved, singular;
    if (threadIdx.x == 0) { anyMoved = 0; singular = 0; }
    __syncthreads();
    for (uint32_t lv = 0; lv < a.levelCount; lv++) {
        for (uint32_t k = a.levelStart[lv] + threadIdx.x; k < a.levelStart[lv + 1]; k += blockDim.x) {
            const uint32_t i = a.levelNodes[k];
            const int32_t par = a.nodes[i].Parent;
            const uint8_t in = a.dirty[i] || (par >= 0 && a.inSet[par]);
            a.inSet[i] = in;
            if (!in) { a.newGlobals[i] = a.globals[i]; continue; }
            anyMoved = 1;
            const idkanim::M4 before = a.globals[i];
            const idkanim::M4 local = idkanim::getMatrix(a.locals[i]);
            const idkanim::M4 g = par < 0 ? local : idkanim::mul(local, a.newGlobals[par]);
            a.newGlobals[i] = g;
            if (a.nodes[i].MeshTransformsCount) {
                idkanim::M4 inv;
                if (!idkanim::invert4(before, inv)) singular = 1;
                a.diffs[i] = idkanim::mul(g, inv);
            }
        }
        __syncthreads();
    }
    if (anyMoved)
        for (uint32_t s = threadIdx.x; s < a.skinCount; s += blockDim.x)
            if (!idkanim::invert4(a.newGlobals[a.skins[s].SkinnedNode], a.invSkin[s])) singular = 1;
    __syncthreads();
    if (threadIdx.x == 0) *a.flags = (anyMoved ? IDK_ANIM_FLAG_NODE_MOVED : 0u) | (singular ? IDK_ANIM_FLAG_SINGULAR : 0u);
}

// UpdateMeshTransformBufferBatched as the device sees it: one thread per mesh transform; skipped after a singular matrix.
// The 144-byte records are 16-byte aligned (cudaMalloc base, 9 x 16 B each), so they move as float4s; one atomic per warp
// raises the "instance moved" flag.
__global__ void k_anim_transforms(AnimArgs a) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    bool moved = false;
    if (t < a.transformCount && !(*a.flags & IDK_ANIM_FLAG_SINGULAR)) {
        const int32_t o = a.owner[t];
        const bool touched = o >= 0 && a.inSet[o];
        if (touched || a.movedBits[t]) {
            float4* rec = reinterpret_cast<float4*>(a.xforms + t);
            union { float4 v[9]; GpuMeshTransform x; } u;
#pragma unroll
            for (int i = 0; i < 9; i++) u.v[i] = rec[i];
            moved = idkanim::transformStep(u.x, touched ? &a.diffs[o] : nullptr);
            if (touched) {
#pragma unroll
                for (int i = 0; i < 9; i++) rec[i] = u.v[i];
            } else {
#pragma unroll
                for (int i = 6; i < 9; i++) rec[i] = u.v[i];   // untouched: only PrevModelMatrix (the last 48 B) changes
            }
            a.movedBits[t] = moved;
        }
    }
    if (__any_sync(0xffffffffu, moved) && (threadIdx.x & 31) == 0) atomicOr(a.flags, IDK_ANIM_FLAG_INSTANCE_MOVED);
}

// ComputeSkinnedPositions' joint matrices (ModelManager.cs:263-279): one thread per joint matrix, when a node moved.
__global__ void k_anim_joints(AnimArgs a) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t f = *a.flags;
    if (j >= a.jointMatrixCount || (f & IDK_ANIM_FLAG_SINGULAR) || !(f & IDK_ANIM_FLAG_NODE_MOVED)) return;
    const uint32_t s = a.jointSlotSkin[j];
    if (s == ~0u) return;
    const uint32_t jj = a.skins[s].FirstJoint + a.jointSlotJoint[j];
    idkanim::M4 ij;
    for (int i = 0; i < 16; i++) ij.m[i / 4][i % 4] = a.inverseJoints[16 * (size_t)jj + i];
    const idkanim::X34 m = idkanim::jointMatrix(ij, a.newGlobals[a.jointNodes[jj]], a.invSkin[s]);
    for (int i = 0; i < 12; i++) a.joints[12 * (size_t)j + i] = m.m[i / 4][i % 4];
}

// idkpt_set_node_transforms: the LocalTransform setter for nodes [first, first + count)
__global__ void k_anim_set_locals(const IdkPtNode* src, IdkPtNodeLocal* locals, uint8_t* pendingDirty, uint32_t first, uint32_t count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const IdkPtNodeLocal l = idkanim::nodeLocal(src[i]);
    if (idkanim::localEq(locals[first + i], l)) return;
    locals[first + i] = l;
    pendingDirty[first + i] = 1;
}
