// Arithmetic of ModelManager.Update (ModelManager.cs:236-592), shared by the device (idk_animation.cuh) and the host mirror
// (host_mirror/animation.cpp): keyframe sampling, Transformation.GetMatrix, the node hierarchy, the mesh-transform step and
// the joint matrices, plus the set-time checks and the plan (sampling groups, hierarchy levels, transform owners) both sides
// run from. The device equals the mirror byte for byte because both run this code.
//
// Float semantics: float products and sums are written out in OpenTK's order (each matrix element a sum of four products,
// left to right) and compiled without contraction (nvcc -fmad=false, g++ -ffp-contract=off). The inverses are cofactor
// expansions in double, rounded to float once. acos and sin (Quaternion.Slerp) are series evaluated in double with plain
// IEEE operations and rounded once, because acosf / sinf differ between glibc and CUDA in the last bit.
#ifndef IDK_ANIM_MATH_H
#define IDK_ANIM_MATH_H

#include <float.h>
#include <math.h>
#include <stdint.h>

#include "../../include/idkpt.h"

#if defined(__CUDACC__)
#define IDK_ANIM_HD __host__ __device__ __forceinline__
#else
#define IDK_ANIM_HD static inline
#endif

namespace idkanim {

struct M4 { float m[4][4]; };
struct X34 { float m[3][4]; };

// float.Equals: +0 == -0, NaN == NaN (the record structs' field-wise Equals)
IDK_ANIM_HD bool eqf(float a, float b) { return a == b || (a != a && b != b); }

IDK_ANIM_HD M4 mul(const M4& a, const M4& b) {   // OpenTK Matrix4.Mult
    M4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j] + a.m[i][3] * b.m[3][j];
    return r;
}

// Matrix4.CreateFromQuaternion (OpenTK 4)
IDK_ANIM_HD M4 fromQuat(const float q[4]) {
    const float sqx = q[0] * q[0], sqy = q[1] * q[1], sqz = q[2] * q[2], sqw = q[3] * q[3];
    const float xy = q[0] * q[1], xz = q[0] * q[2], xw = q[0] * q[3], yz = q[1] * q[2], yw = q[1] * q[3], zw = q[2] * q[3];
    const float s2 = 2.0f / (sqx + sqy + sqz + sqw);
    M4 r = {{{1.0f - s2 * (sqy + sqz), s2 * (xy + zw), s2 * (xz - yw), 0.0f},
             {s2 * (xy - zw), 1.0f - s2 * (sqx + sqz), s2 * (yz + xw), 0.0f},
             {s2 * (xz + yw), s2 * (yz - xw), 1.0f - s2 * (sqx + sqy), 0.0f},
             {0.0f, 0.0f, 0.0f, 1.0f}}};
    return r;
}

// Transformation.GetMatrix (Transformation.cs:57-64): CreateScale(S) * CreateFromQuaternion(R), Row3.xyz = T
IDK_ANIM_HD M4 getMatrix(const IdkPtNodeLocal& l) {
    M4 s = {{{l.Scale[0], 0.0f, 0.0f, 0.0f}, {0.0f, l.Scale[1], 0.0f, 0.0f}, {0.0f, 0.0f, l.Scale[2], 0.0f}, {0.0f, 0.0f, 0.0f, 1.0f}}};
    M4 r = mul(s, fromQuat(l.Rotation));
    r.m[3][0] = l.Translation[0]; r.m[3][1] = l.Translation[1]; r.m[3][2] = l.Translation[2];
    return r;
}

// Matrix4.Invert by cofactors in double; false when the determinant is 0 (OpenTK throws there)
IDK_ANIM_HD bool invert4(const M4& a, M4& out) {
    double m[16], inv[16];
    for (int i = 0; i < 16; i++) m[i] = (double)a.m[i / 4][i % 4];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    if (!(det != 0.0)) return false;   // 0 or NaN
    for (int i = 0; i < 16; i++) out.m[i / 4][i % 4] = (float)(inv[i] / det);
    return true;
}

// GpuMeshTransform's 3x4 (rows act on column vectors, MyMath.Matrix4x4ToTranposed3x4) and back
IDK_ANIM_HD M4 to4x4(const X34& x) {
    M4 r;
    for (int c = 0; c < 4; c++) { for (int k = 0; k < 3; k++) r.m[c][k] = x.m[k][c]; r.m[c][3] = c == 3 ? 1.0f : 0.0f; }
    return r;
}
IDK_ANIM_HD X34 to3x4(const M4& a) {
    X34 r;
    for (int k = 0; k < 3; k++) for (int c = 0; c < 4; c++) r.m[k][c] = a.m[c][k];
    return r;
}
// Matrix3x4.Invert of an affine map x -> A x + t: (A^-1, -A^-1 t), by cofactors in double, rounded once
IDK_ANIM_HD X34 invert3x4(const X34& x) {
    double a[3][3], t[3], c[3][3];
    for (int r = 0; r < 3; r++) { for (int k = 0; k < 3; k++) a[r][k] = x.m[r][k]; t[r] = x.m[r][3]; }
    c[0][0] = a[1][1] * a[2][2] - a[1][2] * a[2][1];
    c[0][1] = a[0][2] * a[2][1] - a[0][1] * a[2][2];
    c[0][2] = a[0][1] * a[1][2] - a[0][2] * a[1][1];
    c[1][0] = a[1][2] * a[2][0] - a[1][0] * a[2][2];
    c[1][1] = a[0][0] * a[2][2] - a[0][2] * a[2][0];
    c[1][2] = a[0][2] * a[1][0] - a[0][0] * a[1][2];
    c[2][0] = a[1][0] * a[2][1] - a[1][1] * a[2][0];
    c[2][1] = a[0][1] * a[2][0] - a[0][0] * a[2][1];
    c[2][2] = a[0][0] * a[1][1] - a[0][1] * a[1][0];
    const double det = a[0][0] * c[0][0] + a[0][1] * c[1][0] + a[0][2] * c[2][0];
    X34 r;
    for (int i = 0; i < 3; i++) {
        double inv[3];
        for (int k = 0; k < 3; k++) { inv[k] = c[i][k] / det; r.m[i][k] = (float)inv[k]; }
        r.m[i][3] = (float)(-(inv[0] * t[0] + inv[1] * t[1] + inv[2] * t[2]));
    }
    return r;
}

IDK_ANIM_HD bool eq34(const X34& a, const X34& b) {
    bool e = true;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) e = e && eqf(a.m[r][c], b.m[r][c]);
    return e;
}

// sin(x) for |x| <= 4 and acos(x) for x in [-1, 1]: Taylor series in double, rounded to float once. The terms fall below
// 2^-60 of the sum before the loops end, so the double result is within a few double ulps and the float rounding is
// correct except within that distance of a float midpoint.
IDK_ANIM_HD float sinF(float xf) {
    const double x = xf, x2 = x * x;
    double term = x, sum = x;
    for (int k = 1; k < 16; k++) { term = -term * x2 / (double)((2 * k) * (2 * k + 1)); sum = sum + term; }
    return (float)sum;
}
IDK_ANIM_HD double asinSeries(double x) {   // |x| <= sqrt(1/2)
    const double x2 = x * x;
    double term = x, sum = x;
    for (int k = 1; k < 60; k++) {
        term = term * x2 * (double)((2 * k - 1) * (2 * k - 1)) / (double)((2 * k) * (2 * k + 1));
        sum = sum + term;
    }
    return sum;
}
IDK_ANIM_HD float acosF(float xf) {
    const double x = xf, halfPi = 1.5707963267948966;
    if (!(x >= -1.0 && x <= 1.0)) return NAN;
    if (x >= 0.5) return (float)(2.0 * asinSeries(sqrt((1.0 - x) * 0.5)));
    if (x <= -0.5) return (float)(2.0 * halfPi - 2.0 * asinSeries(sqrt((1.0 + x) * 0.5)));
    return (float)(halfPi - asinSeries(x));
}

// OpenTK Quaternion.Slerp
IDK_ANIM_HD void slerp(const float* q1, const float* q2in, float blend, float out[4]) {
    float q2[4] = {q2in[0], q2in[1], q2in[2], q2in[3]};
    const float l1 = q1[0] * q1[0] + q1[1] * q1[1] + q1[2] * q1[2] + q1[3] * q1[3];
    const float l2 = q2[0] * q2[0] + q2[1] * q2[1] + q2[2] * q2[2] + q2[3] * q2[3];
    if (l1 == 0.0f) {
        if (l2 == 0.0f) { out[0] = 0.0f; out[1] = 0.0f; out[2] = 0.0f; out[3] = 1.0f; return; }
        for (int i = 0; i < 4; i++) out[i] = q2[i];
        return;
    }
    if (l2 == 0.0f) { for (int i = 0; i < 4; i++) out[i] = q1[i]; return; }
    float cosHalf = q1[3] * q2[3] + (q1[0] * q2[0] + q1[1] * q2[1] + q1[2] * q2[2]);
    if (cosHalf >= 1.0f || cosHalf <= -1.0f) { for (int i = 0; i < 4; i++) out[i] = q1[i]; return; }
    if (cosHalf < 0.0f) { for (int i = 0; i < 4; i++) q2[i] = -q2[i]; cosHalf = -cosHalf; }
    float blendA, blendB;
    if (cosHalf < 0.99f) {
        const float halfAngle = acosF(cosHalf);
        const float sinHalf = sinF(halfAngle);
        const float oneOverSin = 1.0f / sinHalf;
        blendA = sinF(halfAngle * (1.0f - blend)) * oneOverSin;
        blendB = sinF(halfAngle * blend) * oneOverSin;
    } else {
        blendA = 1.0f - blend;
        blendB = blend;
    }
    float r[4];
    for (int i = 0; i < 4; i++) r[i] = blendA * q1[i] + blendB * q2[i];
    const float lr = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
    if (lr > 0.0f) {
        const float scale = 1.0f / sqrtf(lr);
        for (int i = 0; i < 4; i++) out[i] = r[i] * scale;
    } else {
        out[0] = 0.0f; out[1] = 0.0f; out[2] = 0.0f; out[3] = 1.0f;
    }
}

// Algorithms.SortedLowerBound (Algorithms.cs:123-146), the engine's variant: hi = mid - 1, then one fix-up step
IDK_ANIM_HD int sortedLowerBound(const float* arr, int n, float value) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if (arr[mid] < value) lo = mid + 1;
        else hi = mid - 1;
    }
    if (arr[lo] < value) lo++;
    return lo;
}

// One NodeAnimation of UpdateNodeAnimations (ModelManager.cs:535-589) applied to `l` through the LocalTransform setter.
// Returns true when the setter marked the node dirty.
IDK_ANIM_HD bool sampleChannel(const IdkPtNodeAnimation& ch, const IdkPtModelAnimation& anim, float time, const float* times,
                               const float* data, IdkPtNodeLocal& l) {
    const float t = fmodf(time, anim.TMax - anim.TMin);
    const float* keys = times + ch.KeyFrameOffset;
    const int n = (int)ch.KeyFrameCount;
    if (!(t >= keys[0] && t <= keys[n - 1])) return false;
    int index = sortedLowerBound(keys, n, t);
    if (index < 1) index = 1;
    const float prevT = keys[index - 1], nextT = keys[index];
    const float alpha = ch.Mode == IDKPT_ANIM_STEP ? 0.0f : (t - prevT) / (nextT - prevT) * (1.0f - 0.0f) + 0.0f;   // MyMath.MapToZeroOne
    float v[4];
    float* dst;
    int w;
    if (ch.Type == IDKPT_ANIM_ROTATION) {
        const float* q = data + ch.DataOffset;
        slerp(q + 4 * (index - 1), q + 4 * index, alpha, v);
        dst = l.Rotation; w = 4;
    } else {
        const float* p = data + ch.DataOffset + 3 * (index - 1);
        for (int i = 0; i < 3; i++) v[i] = alpha * (p[3 + i] - p[i]) + p[i];   // Vector3.Lerp
        dst = ch.Type == IDKPT_ANIM_SCALE ? l.Scale : l.Translation; w = 3;
    }
    bool same = true;
    for (int i = 0; i < w; i++) same = same && eqf(dst[i], v[i]);
    if (same) return false;
    for (int i = 0; i < w; i++) dst[i] = v[i];
    return true;
}

IDK_ANIM_HD IdkPtNodeLocal nodeLocal(const IdkPtNode& n) {
    IdkPtNodeLocal l;
    for (int i = 0; i < 3; i++) { l.Translation[i] = n.Translation[i]; l.Scale[i] = n.Scale[i]; }
    for (int i = 0; i < 4; i++) l.Rotation[i] = n.Rotation[i];
    return l;
}

IDK_ANIM_HD bool localEq(const IdkPtNodeLocal& a, const IdkPtNodeLocal& b) {
    const float* x = a.Translation; const float* y = b.Translation;
    bool e = true;
    for (int i = 0; i < 10; i++) e = e && eqf(x[i], y[i]);
    return e;
}

// The mesh-transform step of one transform: `diff` (NULL when the hierarchy did not touch it) applied as
// transform.ModelMatrix = diff * transform.ModelMatrix (ModelManager.cs:500-506, GpuMeshTransform.cs:30-38), then the
// PrevModelMatrix rule. Returns the new "moved" bit.
IDK_ANIM_HD bool transformStep(GpuMeshTransform& x, const M4* diff) {
    X34 model, old;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) old.m[r][c] = x.ModelMatrix[r][c];
    model = old;
    if (diff) {
        model = to3x4(mul(*diff, to4x4(old)));
        const X34 inv = invert3x4(model);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) { x.ModelMatrix[r][c] = model.m[r][c]; x.InvModelMatrix[r][c] = inv.m[r][c]; }
    }
    for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) x.PrevModelMatrix[r][c] = old.m[r][c];
    return !eq34(old, model);
}

// JointMatrices[off + j] = Matrix4x4ToTranposed3x4(InverseJointMatrices[j] * Joints[j].Global * inverseNodeTransform)
IDK_ANIM_HD X34 jointMatrix(const M4& inverseJoint, const M4& jointGlobal, const M4& inverseNode) {
    return to3x4(mul(mul(inverseJoint, jointGlobal), inverseNode));
}

}  // namespace idkanim

#include <algorithm>
#include <string>
#include <vector>

namespace idkanim {

// What both sides build from a checked IdkPtAnimationDesc.
struct Group { uint32_t node, first, count, pad; };   // one (node, property): pairs[first, +count) in application order
struct Plan {
    std::vector<IdkPtNode> nodes;
    std::vector<IdkPtNodeAnimation> channels;
    std::vector<IdkPtModelAnimation> animations;
    std::vector<IdkPtSkin> skins;
    std::vector<uint32_t> jointNodes;
    std::vector<float> inverseJoints, times, data;
    std::vector<Group> groups;
    std::vector<uint32_t> pairs;          // per applied channel: channel id, animation id
    std::vector<uint32_t> levelNodes;     // nodes ordered by depth
    std::vector<uint32_t> levelStart;     // levels + 1 offsets into levelNodes
    std::vector<int32_t> owner;           // per mesh transform of the scene: the node whose range holds it, or -1
    std::vector<uint32_t> jointSlotSkin, jointSlotJoint;   // per joint matrix: the last skin writing it and its joint, or ~0u
    uint32_t jointMatrixCount = 0;
};

// Checks `d` against a scene with `transformCount` mesh transforms and `blasCount` BLASes and builds the plan. Returns an
// empty string or what is wrong.
static inline std::string buildPlan(const IdkPtAnimationDesc* d, uint64_t transformCount, uint64_t blasCount, Plan& p) {
    if (!d) return "null desc";
    if ((!d->Nodes && d->NodeCount) || (!d->Channels && d->ChannelCount) || (!d->Animations && d->AnimationCount) ||
        (!d->Skins && d->SkinCount) || ((!d->JointNodes || !d->InverseJointMatrices) && d->JointCount) ||
        (!d->KeyFrameTimes && d->KeyFrameTimeCount) || (!d->KeyFrameData && d->KeyFrameDataCount))
        return "a NULL array with a count";
    const uint64_t lim = 1ull << 31;
    if (d->NodeCount >= lim || d->ChannelCount >= lim || d->AnimationCount >= lim || d->SkinCount >= lim || d->JointCount >= lim ||
        d->KeyFrameTimeCount >= lim || d->KeyFrameDataCount >= (1ull << 32))
        return "an array of 2^31 or more elements";
    const uint64_t N = d->NodeCount;
    std::vector<std::pair<uint64_t, uint64_t>> ranges;
    for (uint64_t i = 0; i < N; i++) {
        const IdkPtNode& n = d->Nodes[i];
        if (n.Parent < -1 || (int64_t)n.Parent >= (int64_t)i) return "node " + std::to_string(i) + ": Parent must be -1 or below the node's own index";
        if ((uint64_t)n.MeshTransformsStart + n.MeshTransformsCount > transformCount) return "node " + std::to_string(i) + ": mesh transform range outside the scene's transforms";
        if (n.MeshTransformsCount) ranges.push_back({n.MeshTransformsStart, (uint64_t)n.MeshTransformsStart + n.MeshTransformsCount});
    }
    std::sort(ranges.begin(), ranges.end());
    for (size_t i = 1; i < ranges.size(); i++)
        if (ranges[i].first < ranges[i - 1].second) return "two nodes' mesh transform ranges overlap";
    for (uint64_t c = 0; c < d->ChannelCount; c++) {
        const IdkPtNodeAnimation& ch = d->Channels[c];
        const std::string who = "channel " + std::to_string(c) + ": ";
        if (ch.TargetNode >= N) return who + "TargetNode out of range";
        if (ch.Type != IDKPT_ANIM_SCALE && ch.Type != IDKPT_ANIM_ROTATION && ch.Type != IDKPT_ANIM_TRANSLATION) return who + "unknown Type";
        if (ch.Mode != IDKPT_ANIM_STEP && ch.Mode != IDKPT_ANIM_LINEAR) return who + "unknown Mode";
        if (ch.KeyFrameCount < 2) return who + "fewer than 2 keyframes";
        if ((uint64_t)ch.KeyFrameOffset + ch.KeyFrameCount > d->KeyFrameTimeCount) return who + "key times past KeyFrameTimes";
        const uint64_t w = ch.Type == IDKPT_ANIM_ROTATION ? 4 : 3;
        if ((uint64_t)ch.DataOffset + w * ch.KeyFrameCount > d->KeyFrameDataCount) return who + "key data past KeyFrameData";
    }
    for (uint64_t a = 0; a < d->AnimationCount; a++) {
        const IdkPtModelAnimation& an = d->Animations[a];
        if ((uint64_t)an.FirstChannel + an.ChannelCount > d->ChannelCount) return "animation " + std::to_string(a) + ": channel range outside Channels";
    }
    uint64_t jointMatrices = 0;
    for (uint64_t s = 0; s < d->SkinCount; s++) {
        const IdkPtSkin& k = d->Skins[s];
        const std::string who = "skin " + std::to_string(s) + ": ";
        if (k.SkinnedNode >= N) return who + "SkinnedNode out of range";
        if ((uint64_t)k.FirstJoint + k.JointCount > d->JointCount) return who + "joint range outside JointNodes";
        if (k.BlasId >= blasCount) return who + "BlasId out of range";
        if ((uint64_t)k.JointMatricesOffset + k.JointCount >= lim) return who + "JointMatricesOffset + JointCount reaches 2^31";
        jointMatrices = std::max(jointMatrices, (uint64_t)k.JointMatricesOffset + k.JointCount);
    }
    for (uint64_t j = 0; j < d->JointCount; j++)
        if (d->JointNodes[j] >= N) return "JointNodes[" + std::to_string(j) + "] out of range";

    p = Plan();
    p.nodes.assign(d->Nodes, d->Nodes + N);
    p.channels.assign(d->Channels, d->Channels + d->ChannelCount);
    p.animations.assign(d->Animations, d->Animations + d->AnimationCount);
    p.skins.assign(d->Skins, d->Skins + d->SkinCount);
    p.jointNodes.assign(d->JointNodes, d->JointNodes + d->JointCount);
    p.inverseJoints.assign(d->InverseJointMatrices, d->InverseJointMatrices + 16 * d->JointCount);
    p.times.assign(d->KeyFrameTimes, d->KeyFrameTimes + d->KeyFrameTimeCount);
    p.data.assign(d->KeyFrameData, d->KeyFrameData + d->KeyFrameDataCount);
    // sampling groups: (node, property) in first-application order; each keeps its channels in application order
    std::vector<std::vector<uint32_t>> lists;
    std::vector<int64_t> groupOf(3 * N, -1);
    for (uint32_t a = 0; a < d->AnimationCount; a++)
        for (uint32_t c = d->Animations[a].FirstChannel; c < d->Animations[a].FirstChannel + d->Animations[a].ChannelCount; c++) {
            const uint64_t key = 3 * (uint64_t)d->Channels[c].TargetNode + (uint64_t)d->Channels[c].Type;
            if (groupOf[key] < 0) { groupOf[key] = (int64_t)lists.size(); lists.emplace_back(); p.groups.push_back({d->Channels[c].TargetNode, 0, 0, 0}); }
            lists[groupOf[key]].push_back(c);
            lists[groupOf[key]].push_back(a);
        }
    for (size_t g = 0; g < lists.size(); g++) {
        p.groups[g].first = (uint32_t)(p.pairs.size() / 2);
        p.groups[g].count = (uint32_t)(lists[g].size() / 2);
        p.pairs.insert(p.pairs.end(), lists[g].begin(), lists[g].end());
    }
    // hierarchy levels
    std::vector<uint32_t> depth(N);
    uint32_t levels = 0;
    for (uint64_t i = 0; i < N; i++) {
        depth[i] = d->Nodes[i].Parent < 0 ? 0 : depth[d->Nodes[i].Parent] + 1;
        levels = std::max(levels, depth[i] + 1);
    }
    p.levelStart.assign(levels + 1, 0);
    for (uint64_t i = 0; i < N; i++) p.levelStart[depth[i] + 1]++;
    for (uint32_t l = 0; l < levels; l++) p.levelStart[l + 1] += p.levelStart[l];
    p.levelNodes.resize(N);
    std::vector<uint32_t> fill(p.levelStart.begin(), p.levelStart.end());
    for (uint64_t i = 0; i < N; i++) p.levelNodes[fill[depth[i]]++] = (uint32_t)i;
    p.owner.assign(transformCount, -1);
    for (uint64_t i = 0; i < N; i++)
        for (uint32_t t = d->Nodes[i].MeshTransformsStart; t < d->Nodes[i].MeshTransformsStart + d->Nodes[i].MeshTransformsCount; t++) p.owner[t] = (int32_t)i;
    p.jointMatrixCount = (uint32_t)jointMatrices;
    p.jointSlotSkin.assign(jointMatrices, ~0u);
    p.jointSlotJoint.assign(jointMatrices, ~0u);
    for (uint32_t s = 0; s < d->SkinCount; s++)        // skins left to right: a later skin's write wins
        for (uint32_t j = 0; j < d->Skins[s].JointCount; j++) {
            p.jointSlotSkin[d->Skins[s].JointMatricesOffset + j] = s;
            p.jointSlotJoint[d->Skins[s].JointMatricesOffset + j] = j;
        }
    return std::string();
}

}  // namespace idkanim

#endif
