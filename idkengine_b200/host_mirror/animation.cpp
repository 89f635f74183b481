// Host mirror of idkpt_update_models (ModelManager.Update's host half, ModelManager.cs:236-592): the same plan, state and
// arithmetic (idk_anim_math.h) as the device, run serially. The device's node locals and globals, mesh transforms and
// joint matrices equal this byte for byte; skinning, refit and the TLAS are the existing paths, which the caller runs on
// the flags this returns.
#include <string.h>

#include <string>
#include <vector>

#include "idk_anim_math.h"

#define IDKHOST_API extern "C" __attribute__((visibility("default")))

using namespace idkanim;

struct IdkHostAnim {
    Plan plan;
    std::vector<IdkPtNodeLocal> locals;
    std::vector<M4> globals;
    std::vector<uint8_t> pendingDirty;       // dirtied by idkhost_anim_set_node_transforms, consumed by the next update
    std::vector<uint8_t> movedBits;          // per mesh transform: moved in the previous update
    std::vector<X34> joints;
    float prevTime = -FLT_MAX;               // float.MinValue
    bool runSkinning = false;
};

IDKHOST_API IdkHostAnim* idkhost_anim_create(const IdkPtAnimationDesc* d, uint64_t transformCount, uint64_t blasCount, char* err, uint32_t errBytes) {
    IdkHostAnim* h = new IdkHostAnim();
    const std::string e = buildPlan(d, transformCount, blasCount, h->plan);
    if (!e.empty()) {
        if (err && errBytes) { strncpy(err, e.c_str(), errBytes - 1); err[errBytes - 1] = 0; }
        delete h;
        return nullptr;
    }
    const size_t n = h->plan.nodes.size();
    h->locals.resize(n);
    h->globals.resize(n);
    for (size_t i = 0; i < n; i++) {
        h->locals[i] = nodeLocal(h->plan.nodes[i]);
        memcpy(h->globals[i].m, h->plan.nodes[i].GlobalTransform, 64);
    }
    h->pendingDirty.assign(n, 0);
    h->movedBits.assign(transformCount, 0);
    h->joints.assign(h->plan.jointMatrixCount, X34{});
    return h;
}

IDKHOST_API void idkhost_anim_free(IdkHostAnim* h) { delete h; }

IDKHOST_API int idkhost_anim_enable(IdkHostAnim* h, uint32_t first, uint32_t count, const uint8_t* enabled) {
    if ((uint64_t)first + count > h->plan.animations.size()) return -1;
    for (uint32_t i = 0; i < count; i++) h->plan.animations[first + i].Enabled = enabled[i] ? 1u : 0u;
    return 0;
}

IDKHOST_API int idkhost_anim_set_node_transforms(IdkHostAnim* h, uint32_t first, uint32_t count, const IdkPtNode* nodes) {
    if ((uint64_t)first + count > h->locals.size()) return -1;
    for (uint32_t i = 0; i < count; i++)
        if (!localEq(h->locals[first + i], nodeLocal(nodes[i]))) { h->locals[first + i] = nodeLocal(nodes[i]); h->pendingDirty[first + i] = 1; }
    return 0;
}

// One update over `transforms` (the scene's mesh transforms, at least as many as at create). Returns 0, or -1 for a singular
// matrix (nothing changed). *moved: bit 0 anyNodeMoved, bit 1 anyMeshInstanceMoved; *skin: 1 when skinning runs this call.
IDKHOST_API int idkhost_anim_update(IdkHostAnim* h, float time, GpuMeshTransform* transforms, uint32_t* moved, int32_t* skin) {
    const Plan& p = h->plan;
    const size_t N = p.nodes.size();
    std::vector<IdkPtNodeLocal> locals = h->locals;
    std::vector<uint8_t> dirty = h->pendingDirty;
    const bool sample = !(time == h->prevTime);
    if (sample)
        for (const Group& g : p.groups)
            for (uint32_t k = g.first; k < g.first + g.count; k++) {
                const IdkPtNodeAnimation& ch = p.channels[p.pairs[2 * k]];
                const IdkPtModelAnimation& an = p.animations[p.pairs[2 * k + 1]];
                if (an.Enabled && sampleChannel(ch, an, time, p.times.data(), p.data.data(), locals[g.node])) dirty[g.node] = 1;
            }
    std::vector<M4> globals = h->globals, diffs(N);
    std::vector<uint8_t> inSet(N, 0);
    bool anyNode = false, singular = false;
    for (uint32_t i = 0; i < N; i++) {     // pre-order: every parent before its children
        const int32_t par = p.nodes[i].Parent;
        inSet[i] = dirty[i] || (par >= 0 && inSet[par]);
        if (!inSet[i]) continue;
        anyNode = true;
        const M4 before = h->globals[i];
        const M4 local = getMatrix(locals[i]);
        globals[i] = par < 0 ? local : mul(local, globals[par]);
        if (p.nodes[i].MeshTransformsCount) {
            M4 inv;
            if (!invert4(before, inv)) singular = true;
            diffs[i] = mul(globals[i], inv);
        }
    }
    std::vector<M4> invSkin(p.skins.size());
    if (anyNode)
        for (size_t s = 0; s < p.skins.size(); s++)
            if (!invert4(globals[p.skins[s].SkinnedNode], invSkin[s])) singular = true;
    if (singular) return -1;

    bool anyInstance = false;
    for (size_t t = 0; t < p.owner.size(); t++) {
        const int32_t o = p.owner[t];
        const bool touched = o >= 0 && inSet[o];
        if (!touched && !h->movedBits[t]) continue;
        const bool m = transformStep(transforms[t], touched ? &diffs[o] : nullptr);
        h->movedBits[t] = m;
        anyInstance = anyInstance || m;
    }
    if (anyNode)
        for (uint32_t j = 0; j < p.jointMatrixCount; j++) {
            const uint32_t s = p.jointSlotSkin[j];
            if (s == ~0u) continue;
            const uint32_t jj = p.skins[s].FirstJoint + p.jointSlotJoint[j];
            M4 ij;
            memcpy(ij.m, &p.inverseJoints[16 * (size_t)jj], 64);
            h->joints[j] = jointMatrix(ij, globals[p.jointNodes[jj]], invSkin[s]);
        }
    h->locals = locals;
    h->globals = globals;
    h->pendingDirty.assign(N, 0);
    if (sample) h->prevTime = time;
    const bool runSkin = anyNode || h->runSkinning;
    h->runSkinning = anyNode;
    if (moved) *moved = (anyNode ? 1u : 0u) | (anyInstance ? 2u : 0u);
    if (skin) *skin = runSkin ? 1 : 0;
    return 0;
}

// which: 0 node locals (IdkPtNodeLocal), 1 node globals (float[16]), 2 joint matrices (float[12]); returns the element count
IDKHOST_API uint64_t idkhost_anim_read(const IdkHostAnim* h, int32_t which, void* out) {
    const void* src = which == 0 ? (const void*)h->locals.data() : which == 1 ? (const void*)h->globals.data() : (const void*)h->joints.data();
    const uint64_t n = which == 0 ? h->locals.size() : which == 1 ? h->globals.size() : h->joints.size();
    const size_t elem = which == 0 ? sizeof(IdkPtNodeLocal) : which == 1 ? sizeof(M4) : sizeof(X34);
    if (out && n) memcpy(out, src, n * elem);
    return n;
}

// sin / acos / SortedLowerBound of idk_anim_math.h, for the tests
IDKHOST_API void idkhost_anim_sin(const float* x, float* y, uint64_t n) { for (uint64_t i = 0; i < n; i++) y[i] = sinF(x[i]); }
IDKHOST_API void idkhost_anim_acos(const float* x, float* y, uint64_t n) { for (uint64_t i = 0; i < n; i++) y[i] = acosF(x[i]); }
IDKHOST_API int32_t idkhost_anim_lower_bound(const float* keys, int32_t n, float v) { return sortedLowerBound(keys, n, v); }
IDKHOST_API void idkhost_anim_slerp(const float* q1, const float* q2, float blend, float* out) { slerp(q1, q2, blend, out); }
