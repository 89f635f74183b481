// Host-side BLAS builder: C++ mirror of the reference's C# builder, which stays
// on the host in production (north_star: "the C# host keeps glTF load, SweepSAH
// BVH build and camera"). It exists here because this image has no .NET; it
// produces exactly the arrays the engine uploads to SSBO 20-23.
//
// Mirrors (file:line relative to the reference repository's IDKEngine/Source):
//   Bvh/PreSplitting.cs:26-160   PreSplit (early split clipping)
//   Bvh/BLAS.cs:128-157          GetBuildData (3 radix sorts by centroid key)
//   Bvh/BLAS.cs:159-274          Build / ProcessBuildTask / RemoveEmptySubtrees
//   Bvh/BLAS.cs:730-873          TrySplit (SweepSAH with early-outs)
//   Bvh/BLAS.cs:875-937          OptimizeStackSize
//   Bvh/BLAS.cs:441-466          GetUnindexedTriangles (refittable path)
//   Bvh/PreSplitting.cs:169-273  GetUnindexedTriangles (dedup + straddling)
//   Utils/Algorithms.cs:15-112,276-297  FloatToKey, RadixSort, StablePartition
//
// The scalar arithmetic (boxes, Triangle.Split, GetPriority, one pre-split step, the
// serial TrySplit, the SAH and collapse terms, the TLAS keys, the settings' defaults)
// lives in csrc/idk_bvh_math.h, which the device build (csrc/idk_blas_build.cuh)
// compiles too. This file keeps what only the host does: the thread pool, the wide
// split's six concurrent scans, the radix sort, processSubtree, the recursive
// collapse, both unindexings and the serial PLOC of the TLAS.
//
// Float semantics: compile with -ffp-contract=off (see idk_bvh_math.h).

#include <cstdint>
#include <cstring>
#include <cmath>
#include <cfloat>
#include <climits>
#include <vector>
#include <algorithm>
#include <thread>
#include <chrono>
#include <atomic>
#include <mutex>
#include <condition_variable>
#include <string>

#include "idk_bvh_math.h"

namespace {

using namespace idkbvh;

struct Settings : Params {
    int threads = 1;
};

struct Geometry {
    const PackedVec3* pos;
    const GpuBlasTriangle* tris;
    int triCount;
    Tri tri(int i) const {
        const GpuBlasTriangle& t = tris[i];
        return {{{{pos[t.X].x, pos[t.X].y, pos[t.X].z}}, {{pos[t.Y].x, pos[t.Y].y, pos[t.Y].z}}, {{pos[t.Z].x, pos[t.Z].y, pos[t.Z].z}}}};
    }
};

struct Fragments {
    std::vector<Box> bounds;
    std::vector<int> originalTriIds; // empty when not presplit
};

// ---------------------------------------------------------------- PreSplitting.PreSplit
static void preSplit(const Geometry& g, const Settings& s, Fragments& out) {
    // Priorities once (the reference evaluates GetPriority three times per triangle); the total is summed in triangle order
    // on one thread, exactly as PreSplitting.cs:33-37 does, because float addition order matters.
    std::vector<float> prio((size_t)g.triCount);
    auto chunked = [&](auto&& f) {
        const int workers = std::max(1, std::min(s.threads, g.triCount / 4096 + 1));
        if (workers == 1) { f(0, g.triCount); return; }
        std::vector<std::thread> pool;
        const int per = (g.triCount + workers - 1) / workers;
        for (int w = 0; w < workers; w++) pool.emplace_back([&, w]() { f(std::min(g.triCount, w * per), std::min(g.triCount, (w + 1) * per)); });
        for (auto& t : pool) t.join();
    };
    chunked([&](int b0, int e0) { for (int i = b0; i < e0; i++) prio[i] = priority(g.tri(i)); });
    float totalPriority = 0.0f;
    for (int i = 0; i < g.triCount; i++) totalPriority += prio[i];

    // every triangle emits exactly its split count (left + right counts always add up), so the output offsets are a prefix sum
    std::vector<size_t> offset((size_t)g.triCount + 1, 0);
    for (int i = 0; i < g.triCount; i++) offset[i + 1] = offset[i] + (size_t)splitCount(prio[i], totalPriority, g.triCount, s.splitFactor);
    out.bounds.resize(offset[g.triCount]);
    out.originalTriIds.resize(offset[g.triCount]);

    Box globalBox = boxEmpty();
    for (int i = 0; i < g.triCount; i++) {
        Tri t = g.tri(i);
        for (int k = 0; k < 3; k++) grow(globalBox, t.p[k]);
    }

    struct Item { Box box; int splits; };
    chunked([&](int b0, int e0) {
    std::vector<Item> stack(64 + 4096);
    for (int i = b0; i < e0; i++) {
        Tri tri = g.tri(i);
        size_t counter = offset[i];
        int sp = 0;
        stack[sp++] = {boxFromTri(tri), (int)(offset[i + 1] - offset[i])};
        while (sp > 0) {
            Item it = stack[--sp];
            if (it.splits == 1) {
                out.bounds[counter] = it.box;
                out.originalTriIds[counter] = i;
                counter++;
                continue;
            }
            Box lBox, rBox;
            const int leftCount = presplitStep(tri, it.box, it.splits, globalBox, lBox, rBox);
            if (sp + 2 > (int)stack.size()) stack.resize(stack.size() * 2);
            stack[sp++] = {rBox, it.splits - leftCount};
            stack[sp++] = {lBox, leftCount};
        }
    }
    });
}

// ---------------------------------------------------------------- BLAS.GetBuildData
struct BuildData {
    Fragments frags;
    std::vector<float> rightCostsAccum;
    std::vector<int> partitionAux;
    std::vector<uint8_t> fragLeftTable;
    std::vector<int> sorted[3];
    int n() const { return (int)frags.bounds.size(); }
};

// Algorithms.RadixSort: 3 x 11-bit LSD passes (stable).
static void radixSortFragments(const Fragments& f, int axis, std::vector<int>& output) {
    const int n = (int)f.bounds.size();
    const int radixSize = 11, binSize = 1 << radixSize, mask = binSize - 1;
    std::vector<uint32_t> keys(n);
    for (int i = 0; i < n; i++) keys[i] = floatToKey(f.bounds[i].mn[axis] + f.bounds[i].mx[axis]);
    std::vector<int> prefix(binSize * 3, 0);
    for (int i = 0; i < n; i++) {
        uint32_t k = keys[i];
        prefix[(k & mask)]++;
        prefix[((k >> 11) & mask) + binSize]++;
        prefix[((k >> 22) & mask) + 2 * binSize]++;
    }
    for (int p = 0; p < 3; p++) {
        int sum = 0;
        for (int i = 0; i < binSize; i++) { int t = prefix[i + p * binSize]; prefix[i + p * binSize] = sum; sum += t; }
    }
    std::vector<int> a(n), b(n);
    for (int i = 0; i < n; i++) a[i] = i;
    std::vector<int>* in = &a; std::vector<int>* outp = &b;
    for (int p = 0; p < 3; p++) {
        for (int j = 0; j < n; j++) {
            int el = (*in)[j];
            uint32_t r = (keys[el] >> (p * radixSize)) & mask;
            (*outp)[prefix[r + p * binSize]++] = el;
        }
        std::swap(in, outp);
    }
    output = *in; // after 3 passes the result lives in the buffer 'in' points to
}

static Box computeBoundingBox(int start, int count, const BuildData& bd, int axis) {
    return rangeBox(bd.frags.bounds.data(), bd.sorted[axis].data(), start, start + count);
}

// BLAS.TrySplit, serial; returns the split index, or -1 for a leaf
static int trySplit(const GpuBlasNode& parent, BuildData& bd, const Settings& s) {
    const Box parentBox = {{parent.Min[0], parent.Min[1], parent.Min[2]}, {parent.Max[0], parent.Max[1], parent.Max[2]}};
    int* const ids[3] = {bd.sorted[0].data(), bd.sorted[1].data(), bd.sorted[2].data()};
    return trySplitSerial(bd.frags.bounds.data(), ids, bd.rightCostsAccum.data(), bd.fragLeftTable.data(), bd.partitionAux.data(),
                          s, parentBox, parent.TriStartOrChild, parent.TriCount);
}


// ---- wide variant of TrySplit for the few huge nodes at the top of the tree --------------------------------------------------
// Same decisions as trySplit, bit for bit: the six box scans (prefix = left cost, suffix = right cost, per axis) are
// computed in full by up to six threads (min/max accumulation is exact, so a scan computed in full equals the
// reference's early-terminated one wherever the reference looks at it); the reference's sweep loop with its early-outs
// then runs over the precomputed costs. The two child boxes and the three stable partitions run concurrently as well.
struct WideScratch {
    std::vector<float> L[3], R[3];   // indexed by absolute fragment position
    void ensure(int n) { for (int a = 0; a < 3; a++) { if ((int)L[a].size() < n) { L[a].resize(n); R[a].resize(n); } } }
};

template <class F>
static void runTasks(int taskCount, int threads, F&& f) {
    const int workers = std::max(1, std::min(threads, taskCount));
    if (workers == 1) { for (int t = 0; t < taskCount; t++) f(t); return; }
    std::atomic<int> next(0);
    std::vector<std::thread> pool;
    for (int w = 0; w < workers - 1; w++) pool.emplace_back([&]() { for (;;) { int t = next.fetch_add(1); if (t >= taskCount) break; f(t); } });
    for (;;) { int t = next.fetch_add(1); if (t >= taskCount) break; f(t); }
    for (auto& th : pool) th.join();
}

static int trySplitWide(const GpuBlasNode& parent, BuildData& bd, const Settings& s, WideScratch& ws) {
    const Box parentBox = {{parent.Min[0], parent.Min[1], parent.Min[2]}, {parent.Max[0], parent.Max[1], parent.Max[2]}};
    if (parent.TriCount <= s.stopSplittingThreshold) return -1;
    const int start = parent.TriStartOrChild;
    const int end = parent.TriStartOrChild + parent.TriCount;
    const Box* fragBounds = bd.frags.bounds.data();
    ws.ensure(bd.n());

    runTasks(6, s.threads, [&](int task) {
        const int axis = task >> 1;
        const int* ids = bd.sorted[axis].data();
        if (task & 1) {           // suffix: R[i] = halfArea(box of [i, end)) * (end - i)
            Box acc = boxEmpty();
            float counter = 0.0f;
            float* R = ws.R[axis].data();
            for (int i = end - 1; i >= start + 1; i--) { counter++; acc = combine(acc, fragBounds[ids[i]]); R[i] = halfArea(acc) * counter; }
        } else {                  // prefix: L[i] = halfArea(box of [start, i]) * (i - start + 1)
            Box acc = boxEmpty();
            float counter = 0.0f;
            float* L = ws.L[axis].data();
            for (int i = start; i < end - 1; i++) { counter++; acc = combine(acc, fragBounds[ids[i]]); L[i] = halfArea(acc) * counter; }
        }
    });

    float bestCost = FLT_MAX;
    int bestAxis = 0, bestSplit = 0;
    for (int axis = 0; axis < 3; axis++) {   // BLAS.TrySplit's sweep, reading the precomputed costs
        const float* L = ws.L[axis].data();
        const float* R = ws.R[axis].data();
        int firstRight = start + 1;
        for (int i = end - 1; i >= firstRight; i--)
            if (R[i] >= bestCost) { firstRight = i + 1; break; }
        for (int i = firstRight - 1; i < end - 1; i++) {
            const float leftCost = L[i];
            const float cost = leftCost + R[i + 1];
            if (cost < bestCost) { bestSplit = i + 1; bestAxis = axis; bestCost = cost; }
            else if (leftCost >= bestCost) break;
        }
    }
    if (!keepSplit(s, parentBox, start, parent.TriCount, bestCost, bestAxis, bestSplit)) return -1;

    Box childBox[2];
    runTasks(2, s.threads, [&](int t) {
        childBox[t] = t == 0 ? computeBoundingBox(start, bestSplit - start, bd, bestAxis)
                             : computeBoundingBox(bestSplit, end - bestSplit, bd, bestAxis);
    });
    const bool swap = swapSides(childBox[0], childBox[1]);

    uint8_t* table = bd.fragLeftTable.data();
    int* ids = bd.sorted[bestAxis].data();
    runTasks(2, s.threads, [&](int t) {
        if (t == 0) for (int i = start; i < bestSplit; i++) table[ids[i]] = !swap;
        else for (int i = bestSplit; i < end; i++) table[ids[i]] = swap;
    });

    // three independent id arrays: each needs its own auxiliary range
    std::vector<int> auxB(parent.TriCount), auxC(parent.TriCount);
    int newSplit = bestSplit;
    runTasks(3, s.threads, [&](int t) {
        if (t == 0) { if (swap) newSplit = start + stablePartition(ids + start, parent.TriCount, bd.partitionAux.data() + start, table); }
        else if (t == 1) stablePartition(bd.sorted[(bestAxis + 1) % 3].data() + start, parent.TriCount, auxB.data(), table);
        else stablePartition(bd.sorted[(bestAxis + 2) % 3].data() + start, parent.TriCount, auxC.data(), table);
    });
    return newSplit;
}

// ---------------------------------------------------------------- BLAS.Build
struct BuildResult {
    std::vector<GpuBlasNode> nodes;
    int requiredStackSize = 0;
};

struct BuildTask { int parentNodeId; int newNodesId; };

static void processSubtree(BuildResult& blas, BuildData& bd, const Settings& s, BuildTask root,
                           std::vector<BuildTask>* spill, int spillThreshold) {
    std::vector<BuildTask> stack;
    stack.push_back(root);
    while (!stack.empty()) {
        BuildTask t = stack.back();
        stack.pop_back();
        GpuBlasNode& parent = blas.nodes[t.parentNodeId];
        setBounds(parent, computeBoundingBox(parent.TriStartOrChild, parent.TriCount, bd, 0));
        const int split = trySplit(parent, bd, s);
        if (split < 0) continue;

        GpuBlasNode left = {};
        left.TriStartOrChild = parent.TriStartOrChild;
        left.TriCount = split - left.TriStartOrChild;
        GpuBlasNode right = {};
        right.TriStartOrChild = split;
        right.TriCount = parent.TriCount - left.TriCount;

        int leftId = t.newNodesId, rightId = leftId + 1;
        blas.nodes[leftId] = left;
        blas.nodes[rightId] = right;
        parent.TriStartOrChild = leftId;
        parent.TriCount = 0;

        BuildTask lt = {leftId, rightId + 1};
        BuildTask rt = {rightId, rightId + (2 * left.TriCount - 1)};
        // Sub-tasks touch disjoint ranges of every array, so any execution order
        // yields the same tree (BLAS.cs:221-231 runs them on separate threads).
        if (spill && std::min(left.TriCount, right.TriCount) >= spillThreshold) {
            spill->push_back(lt);
            spill->push_back(rt);
        } else {
            stack.push_back(rt);
            stack.push_back(lt);
        }
    }
}

static int computeRequiredStackSize(const BuildResult& blas, int nodeId) {
    const GpuBlasNode& l = blas.nodes[nodeId];
    const GpuBlasNode& r = blas.nodes[nodeId + 1];
    bool tl = !(l.TriCount > 0), tr = !(r.TriCount > 0);
    if (tl || tr) {
        if (tl && tr) {
            int a = computeRequiredStackSize(blas, l.TriStartOrChild);
            int b = computeRequiredStackSize(blas, r.TriStartOrChild);
            return std::max(a, b) + 1;
        }
        return computeRequiredStackSize(blas, tl ? l.TriStartOrChild : r.TriStartOrChild);
    }
    return 0;
}

static double computeGlobalSAH(const BuildResult& blas, const Settings& s) {
    double cost = 0.0;
    double rootArea = 1.0 / (double)nodeHalfArea(blas.nodes[1]);
    std::vector<int> stack;
    stack.push_back(1);
    while (!stack.empty()) {
        const GpuBlasNode& n = blas.nodes[stack.back()];
        stack.pop_back();
        cost += sahTerm(n, rootArea, s.triangleCost);
        if (!(n.TriCount > 0)) {
            stack.push_back(n.TriStartOrChild + 1);
            stack.push_back(n.TriStartOrChild);
        }
    }
    return cost;
}

static void collapseDeepestLevel(BuildResult& blas, const Settings& s, int newStackSize, bool firstPass,
                                 double& nextCollapseCost, int parentId, int stackSize) {
    GpuBlasNode& parent = blas.nodes[parentId];
    const int childId = parent.TriStartOrChild;
    GpuBlasNode& l = blas.nodes[childId];
    GpuBlasNode& r = blas.nodes[childId + 1];

    if (!(l.TriCount > 0)) collapseDeepestLevel(blas, s, newStackSize, firstPass, nextCollapseCost, childId, stackSize + 1);
    if (!(r.TriCount > 0)) collapseDeepestLevel(blas, s, newStackSize, firstPass, nextCollapseCost, childId + 1, stackSize + 1);

    if (l.TriCount > 0 && r.TriCount > 0) {
        if (stackSize > newStackSize && !firstPass) {
            parent.TriStartOrChild = l.TriStartOrChild;
            parent.TriCount = l.TriCount + r.TriCount;
        }
        if ((stackSize == newStackSize && !firstPass) || (stackSize > newStackSize && firstPass)) {
            if ((float)(l.TriCount + r.TriCount) > STACK_OPT_MAX_LEAF_TRIANGLE_COUNT) {
                nextCollapseCost = (double)FLT_MAX;
                return;
            }
            nextCollapseCost += collapseTerm(parent, l, r, l.TriCount, r.TriCount, blas.nodes[1], s.triangleCost);
        }
    }
}

static void optimizeStackSize(BuildResult& blas, const Settings& s) {
    blas.requiredStackSize = computeRequiredStackSize(blas, 2);
    if (blas.requiredStackSize < s.stackOptThreshold) return;
    double currentCost = computeGlobalSAH(blas, s);
    double addedCost = 0.0;
    collapseDeepestLevel(blas, s, blas.requiredStackSize - 1, true, addedCost, 1, 0);
    double increasePercent = addedCost / currentCost;
    while (increasePercent <= (double)s.stackOptSahIncreaseAcceptance && blas.requiredStackSize > 0) {
        collapseDeepestLevel(blas, s, --blas.requiredStackSize, false, addedCost, 1, 0);
        increasePercent = addedCost / currentCost;
    }
}

static int removeEmptySubtrees(BuildResult& blas) {
    int nodeCounter = 2;
    std::vector<int> stack;
    stack.push_back(1);
    while (!stack.empty()) {
        int pid = stack.back();
        stack.pop_back();
        GpuBlasNode& parent = blas.nodes[pid];
        GpuBlasNode l = blas.nodes[parent.TriStartOrChild];
        GpuBlasNode r = blas.nodes[parent.TriStartOrChild + 1];
        int lid = nodeCounter, rid = nodeCounter + 1;
        blas.nodes[lid] = l;
        blas.nodes[rid] = r;
        parent.TriStartOrChild = lid;
        nodeCounter += 2;
        if (!(r.TriCount > 0)) stack.push_back(rid);
        if (!(l.TriCount > 0)) stack.push_back(lid);
    }
    return nodeCounter;
}

static int buildBlas(BuildResult& blas, BuildData& bd, const Settings& s) {
    const bool timing = getenv("IDKHOST_TIMING") != nullptr;
    auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t0 = now(), t1;
    auto lap = [&](const char* what) { if (timing) { t1 = now(); fprintf(stderr, "[idkhost]   %-14s %8.1f ms\n", what, (t1 - t0) * 1e3); t0 = t1; } };
    blas.nodes[0] = GpuBlasNode{};
    GpuBlasNode& root = blas.nodes[1];
    root = GpuBlasNode{};
    root.TriStartOrChild = 0;
    root.TriCount = bd.n();

    if (s.threads > 1 && bd.n() >= (1 << 14)) {
        // Task pool over the tree (BLAS.cs:221-231 runs sub-tasks on separate threads): a worker takes a node; a node
        // above the threshold is split once and its two children become tasks, a smaller one is finished serially.
        // Sub-tasks touch disjoint ranges of every array, so any execution order yields the same tree. The one or two
        // levels where there are fewer nodes than workers use the wide split (all threads on one node).
        const int threshold = std::max(1 << 13, bd.n() / (s.threads * 8)); // BLAS.THREADED_RECURSION_THRESHOLD
        const int wideThreshold = std::max(2 * threshold, bd.n() / 3);
        std::mutex mu;
        std::condition_variable cv;
        std::vector<BuildTask> queue;
        int active = 0;
        queue.push_back({1, 2});
        auto splitOnce = [&](BuildTask t, WideScratch* wide) {
            GpuBlasNode& parent = blas.nodes[t.parentNodeId];
            setBounds(parent, computeBoundingBox(parent.TriStartOrChild, parent.TriCount, bd, 0));
            const int split = wide ? trySplitWide(parent, bd, s, *wide) : trySplit(parent, bd, s);
            if (split < 0) return;
            GpuBlasNode left = {}; left.TriStartOrChild = parent.TriStartOrChild; left.TriCount = split - left.TriStartOrChild;
            GpuBlasNode right = {}; right.TriStartOrChild = split; right.TriCount = parent.TriCount - left.TriCount;
            int leftId = t.newNodesId, rightId = leftId + 1;
            blas.nodes[leftId] = left; blas.nodes[rightId] = right;
            parent.TriStartOrChild = leftId; parent.TriCount = 0;
            std::lock_guard<std::mutex> lk(mu);
            queue.push_back({leftId, rightId + 1});
            queue.push_back({rightId, rightId + (2 * left.TriCount - 1)});
        };
        {   // top of the tree: all threads on one node at a time
            WideScratch wide;
            for (;;) {
                size_t pick = queue.size();
                for (size_t i = 0; i < queue.size(); i++)
                    if (blas.nodes[queue[i].parentNodeId].TriCount >= wideThreshold) { pick = i; break; }
                if (pick == queue.size()) break;
                BuildTask t = queue[pick];
                queue.erase(queue.begin() + pick);
                splitOnce(t, &wide);
            }
        }
        lap("breadth");
        std::vector<std::thread> pool;
        for (int i = 0; i < s.threads; i++) {
            pool.emplace_back([&]() {
                std::unique_lock<std::mutex> lk(mu);
                for (;;) {
                    while (queue.empty() && active > 0) cv.wait(lk);
                    if (queue.empty()) break;                       // nothing queued and nobody working: done
                    BuildTask t = queue.back();
                    queue.pop_back();
                    active++;
                    lk.unlock();
                    if (blas.nodes[t.parentNodeId].TriCount >= 2 * threshold) splitOnce(t, nullptr);
                    else processSubtree(blas, bd, s, t, nullptr, 0);
                    lk.lock();
                    active--;
                    cv.notify_all();
                }
                cv.notify_all();
            });
        }
        for (auto& th : pool) th.join();
    } else {
        processSubtree(blas, bd, s, {1, 2}, nullptr, 0);
    }

    lap("subtrees");
    if (root.TriCount > 0) {
        blas.nodes[2] = root;
        blas.nodes[3] = root;
        root.TriStartOrChild = 2;
        root.TriCount = 0;
    }
    optimizeStackSize(blas, s);
    lap("stack opt");
    const int used = removeEmptySubtrees(blas);
    lap("compact");
    return used;
}

// ---------------------------------------------------------------- GetUnindexedTriangles
static std::vector<int> uniqueTriIds(const GpuBlasNode& leaf, const BuildData& bd) {
    std::vector<int> ids(leaf.TriCount);
    for (int i = 0; i < leaf.TriCount; i++) ids[i] = bd.frags.originalTriIds[bd.sorted[0][leaf.TriStartOrChild + i]];
    std::sort(ids.begin(), ids.end());
    ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
    return ids;
}

static bool contains(const std::vector<int>& v, int x) { return std::find(v.begin(), v.end(), x) != v.end(); }

// PreSplitting.GetUnindexedTriangles, Bvh/PreSplitting.cs:169-273
static void unindexPreSplit(BuildResult& blas, const BuildData& bd, const Geometry& g, std::vector<GpuBlasTriangle>& tris) {
    tris.assign(bd.n(), GpuBlasTriangle{});
    int counter = 0;
    std::vector<int> stack;
    stack.push_back(2);
    while (!stack.empty()) {
        int top = stack.back();
        stack.pop_back();
        GpuBlasNode& l = blas.nodes[top];
        GpuBlasNode& r = blas.nodes[top + 1];
        bool ll = l.TriCount > 0, rl = r.TriCount > 0;
        if (ll && rl) {
            std::vector<int> lu = uniqueTriIds(l, bd), ru = uniqueTriIds(r, bd);
            int onlyLeft = 0, backwards = 0;
            for (size_t i = 0; i < lu.size(); i++) {
                int id = lu[i];
                if (contains(ru, id)) tris[counter + (int)lu.size() - backwards++ - 1] = g.tris[id];
                else tris[counter + onlyLeft++] = g.tris[id];
            }
            int onlyRight = 0;
            for (size_t i = 0; i < ru.size(); i++) {
                int id = ru[i];
                if (!contains(lu, id)) tris[counter + (int)lu.size() + onlyRight++] = g.tris[id];
            }
            l.TriStartOrChild = counter;
            l.TriCount = (int)lu.size();
            r.TriStartOrChild = counter + onlyLeft;
            r.TriCount = (int)ru.size();
            counter += (r.TriStartOrChild + r.TriCount) - l.TriStartOrChild;
        } else if (ll || rl) {
            GpuBlasNode& leaf = ll ? l : r;
            std::vector<int> u = uniqueTriIds(leaf, bd);
            for (size_t i = 0; i < u.size(); i++) tris[counter + (int)i] = g.tris[u[i]];
            leaf.TriStartOrChild = counter;
            leaf.TriCount = (int)u.size();
            counter += (int)u.size();
        }
        if (!rl) stack.push_back(r.TriStartOrChild);
        if (!ll) stack.push_back(l.TriStartOrChild);
    }
    tris.resize(counter);
}

// BLAS.GetUnindexedTriangles, Bvh/BLAS.cs:441-466. The array holds n triangles; when the root stays a leaf, its two copies
// list all n each, and the reference writes the second copy's past the end of its array. Those writes are dropped: the
// result is the first copy's n triangles and the offset n for the second copy.
static void unindexPlain(BuildResult& blas, const BuildData& bd, const Geometry& g, std::vector<GpuBlasTriangle>& tris) {
    const int n = bd.n();
    tris.assign(n, GpuBlasTriangle{});
    int counter = 0;
    for (size_t i = 2; i < blas.nodes.size(); i++) {
        GpuBlasNode& node = blas.nodes[i];
        if (node.TriCount > 0) {
            for (int j = 0; j < node.TriCount && counter + j < n; j++) tris[counter + j] = g.tris[bd.sorted[0][node.TriStartOrChild + j]];
            node.TriStartOrChild = counter;
            counter += node.TriCount;
        }
    }
}

} // namespace

struct IdkBlasBuild {
    std::vector<GpuBlasNode> nodes;
    std::vector<GpuBlasTriangle> tris;
    int requiredStackSize = 0;
    int fragmentCount = 0;
    double sah = 0.0;
};

extern "C" {

// Settings blob mirrors BLAS.BuildSettings (BLAS.cs:31-48) + PreSplitting.Settings (PreSplitting.cs:17-24).
struct IdkBlasBuildSettings {
    int32_t StopSplittingThreshold;
    int32_t MaxLeafTriangleCount;
    float   TriangleCost;
    int32_t StackOptThreshold;
    float   StackOptSahIncreaseAcceptance;
    float   SplitFactor;
    int32_t DoPreSplit;   // !IsRefittable (BVH.cs:324-333)
    int32_t Threads;
};

__attribute__((visibility("default")))
void idkhost_default_build_settings(IdkBlasBuildSettings* s) {
    const Settings d;
    *s = {d.stopSplittingThreshold, d.maxLeafTriangleCount, d.triangleCost, d.stackOptThreshold,
          d.stackOptSahIncreaseAcceptance, d.splitFactor, d.doPreSplit, d.threads};
}

// One BLAS: BVH.BlasesBuild loop body, Bvh/BVH.cs:315-377.
__attribute__((visibility("default")))
IdkBlasBuild* idkhost_blas_build(const PackedVec3* positions, uint64_t vertexCount,
                                 const GpuBlasTriangle* triangles, uint64_t triangleCount,
                                 const IdkBlasBuildSettings* settings) {
    (void)vertexCount;
    Settings s;
    s.stopSplittingThreshold = settings->StopSplittingThreshold;
    s.maxLeafTriangleCount = settings->MaxLeafTriangleCount;
    s.triangleCost = settings->TriangleCost;
    s.stackOptThreshold = settings->StackOptThreshold;
    s.stackOptSahIncreaseAcceptance = settings->StackOptSahIncreaseAcceptance;
    s.splitFactor = settings->SplitFactor;
    s.doPreSplit = settings->DoPreSplit;
    s.threads = std::max(1, settings->Threads);

    const bool timing = getenv("IDKHOST_TIMING") != nullptr;
    auto now = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t0 = now(), t1;
    auto lap = [&](const char* what) { if (timing) { t1 = now(); fprintf(stderr, "[idkhost] %-14s %8.1f ms\n", what, (t1 - t0) * 1e3); t0 = t1; } };
    Geometry g = {positions, triangles, (int)triangleCount};
    BuildData bd;
    if (s.doPreSplit) {
        preSplit(g, s, bd.frags);
    } else {
        bd.frags.bounds.resize(g.triCount);
        for (int i = 0; i < g.triCount; i++) bd.frags.bounds[i] = boxFromTri(g.tri(i));
    }
    lap("presplit");
    const int n = bd.n();
    bd.fragLeftTable.assign(n, 0);
    bd.rightCostsAccum.assign(n, 0.0f);
    bd.partitionAux.assign(n, 0);
    if (s.threads > 1 && n >= (1 << 16)) {
        std::thread t0([&]() { radixSortFragments(bd.frags, 0, bd.sorted[0]); });
        std::thread t1([&]() { radixSortFragments(bd.frags, 1, bd.sorted[1]); });
        radixSortFragments(bd.frags, 2, bd.sorted[2]);
        t0.join(); t1.join();
    } else {
        for (int a = 0; a < 3; a++) radixSortFragments(bd.frags, a, bd.sorted[a]);
    }

    lap("radix sort");
    BuildResult blas;
    blas.nodes.assign(std::max(2 * n, 4), GpuBlasNode{});
    int used = buildBlas(blas, bd, s);
    blas.nodes.resize(used);
    lap("build+stackopt");

    IdkBlasBuild* out = new IdkBlasBuild();
    if (s.doPreSplit) unindexPreSplit(blas, bd, g, out->tris);
    else unindexPlain(blas, bd, g, out->tris);
    lap("unindex");
    out->sah = computeGlobalSAH(blas, s);
    lap("sah");
    out->nodes = std::move(blas.nodes);
    out->requiredStackSize = blas.requiredStackSize;
    out->fragmentCount = n;
    return out;
}

__attribute__((visibility("default"))) uint64_t idkhost_blas_node_count(const IdkBlasBuild* b) { return b->nodes.size(); }
__attribute__((visibility("default"))) uint64_t idkhost_blas_triangle_count(const IdkBlasBuild* b) { return b->tris.size(); }
__attribute__((visibility("default"))) int32_t idkhost_blas_required_stack_size(const IdkBlasBuild* b) { return b->requiredStackSize; }
__attribute__((visibility("default"))) int32_t idkhost_blas_fragment_count(const IdkBlasBuild* b) { return b->fragmentCount; }
__attribute__((visibility("default"))) double idkhost_blas_sah(const IdkBlasBuild* b) { return b->sah; }
__attribute__((visibility("default")))
void idkhost_blas_copy(const IdkBlasBuild* b, GpuBlasNode* nodes, GpuBlasTriangle* tris) {
    memcpy(nodes, b->nodes.data(), b->nodes.size() * sizeof(GpuBlasNode));
    memcpy(tris, b->tris.data(), b->tris.size() * sizeof(GpuBlasTriangle));
}
__attribute__((visibility("default"))) void idkhost_blas_free(IdkBlasBuild* b) { delete b; }

// BLAS.ComputeGlobalSAH (BLAS.cs:629-656) of any BLAS's nodes (node 1 the root): built, refitted or read back from the device.
__attribute__((visibility("default")))
double idkhost_blas_global_sah(const GpuBlasNode* nodes, uint64_t nodeCount, float triangleCost) {
    BuildResult blas;
    blas.nodes.assign(nodes, nodes + nodeCount);
    Settings s;
    s.triangleCost = triangleCost;
    return computeGlobalSAH(blas, s);
}

} // extern "C"

// ---------------------------------------------------------------- TLAS (Bvh/TLAS.cs:28-141, serial PLOC)
namespace {

static inline Box tlasBox(const GpuTlasNode& n) { return {{n.Min[0], n.Min[1], n.Min[2]}, {n.Max[0], n.Max[1], n.Max[2]}}; }
static inline void tlasSetBounds(GpuTlasNode& n, const Box& b) { for (int i = 0; i < 3; i++) { n.Min[i] = b.mn[i]; n.Max[i] = b.mx[i]; } }

static int findBestMatch(const GpuTlasNode* nodes, int start, int end, int nodeIndex) {
    float smallestArea = FLT_MAX;
    int best = -1;
    Box nodeBox = tlasBox(nodes[nodeIndex]);
    for (int i = start; i < end; i++) {
        if (i == nodeIndex) continue;
        float area = halfArea(combine(nodeBox, tlasBox(nodes[i])));
        if (area < smallestArea) { smallestArea = area; best = i; }
    }
    return best;
}

} // namespace

extern "C" {

// Box.Transformed(localBounds, modelMatrix) (Shapes/Box.cs:166-175): 8 corners through the (column-vector) 3x4 model matrix.
__attribute__((visibility("default")))
void idkhost_transform_box(const float mn[3], const float mx[3], const float model3x4[12], float outMin[3], float outMax[3]) {
    const Box b = transformedBox({{mn[0], mn[1], mn[2]}, {mx[0], mx[1], mx[2]}}, model3x4);
    for (int i = 0; i < 3; i++) { outMin[i] = b.mn[i]; outMax[i] = b.mx[i]; }
}

// idkhost_transform_box over n instances in one call: out[6 i ...] = Box.Transformed(roots[i], models[i]); roots = n x {min[3],
// max[3]}, models = n x 12 floats (the rows of each 3x4 model matrix).
__attribute__((visibility("default")))
void idkhost_transform_boxes(const float* roots, const float* models, int64_t n, float* out) {
    for (int64_t i = 0; i < n; i++) {
        const float* r = roots + 6 * i;
        const Box b = transformedBox({{r[0], r[1], r[2]}, {r[3], r[4], r[5]}}, models + 12 * i);
        for (int k = 0; k < 3; k++) { out[6 * i + k] = b.mn[k]; out[6 * i + 3 + k] = b.mx[k]; }
    }
}

// TLAS.Build: boxes = primitiveCount x {min[3], max[3]} (world space), nodes = 2*primitiveCount-1 GpuTlasNode, root at 0.
__attribute__((visibility("default")))
void idkhost_tlas_build(const float* boxes, int32_t primitiveCount, GpuTlasNode* nodes, int32_t searchRadius) {
    const int nodeCount = std::max(2 * primitiveCount - 1, 0);
    if (nodeCount == 0) return;
    std::vector<GpuTlasNode> temp(nodeCount);
    memset(nodes, 0, sizeof(GpuTlasNode) * (size_t)nodeCount);
    {
        GpuTlasNode* leaves = temp.data() + (nodeCount - primitiveCount);
        Box global = boxEmpty();
        for (int i = 0; i < primitiveCount; i++) {
            Box b = {{boxes[6 * i], boxes[6 * i + 1], boxes[6 * i + 2]}, {boxes[6 * i + 3], boxes[6 * i + 4], boxes[6 * i + 5]}};
            global = combine(global, b);
            GpuTlasNode n = {};
            tlasSetBounds(n, b);
            n.IsLeafAndChildOrInstanceId = (1u << 31) | (uint32_t)i;
            leaves[i] = n;
        }
        std::vector<std::pair<uint32_t, int>> keyed(primitiveCount);
        for (int i = 0; i < primitiveCount; i++) keyed[i] = {centreKey(tlasBox(leaves[i]), global), i};
        std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<uint32_t, int>& a, const std::pair<uint32_t, int>& b) { return a.first < b.first; });
        for (int i = 0; i < primitiveCount; i++) nodes[nodeCount - primitiveCount + i] = leaves[keyed[i].second];
    }
    int activeRangeCount = primitiveCount, activeRangeEnd = nodeCount;
    std::vector<int> pref(primitiveCount);
    while (activeRangeCount > 1) {
        const int activeRangeStart = activeRangeEnd - activeRangeCount;
        for (int i = 0; i < activeRangeCount; i++) {
            int a = activeRangeStart + i;
            int s = std::max(a - searchRadius, activeRangeStart), e = std::min(a + searchRadius + 1, activeRangeEnd);
            pref[i] = findBestMatch(nodes, s, e, a) - activeRangeStart;
        }
        int merged = 0;       // b < 0: the node found no half area below FLT_MAX (a box that is not finite)
        for (int i = 0; i < activeRangeCount; i++) { int b = pref[i]; if (b >= 0 && pref[b] == i && i < b) merged += 2; }
        if (merged == 0) return;   // nothing would ever merge again: the nodes are not a tree (the device build reports it)
        const int unmerged = activeRangeCount - merged, newNodes = merged / 2;
        int mergedHead = activeRangeEnd - merged;
        const int newBegin = mergedHead - unmerged - newNodes;
        int unmergedHead = newBegin;
        for (int i = 0; i < activeRangeCount; i++) {
            int b = pref[i];
            int aId = i + activeRangeStart;
            if (b >= 0 && pref[b] == i) {
                if (i < b) {
                    int bId = b + activeRangeStart;
                    temp[mergedHead] = nodes[aId];
                    temp[mergedHead + 1] = nodes[bId];
                    GpuTlasNode nn = {};
                    tlasSetBounds(nn, combine(tlasBox(temp[mergedHead]), tlasBox(temp[mergedHead + 1])));
                    nn.IsLeafAndChildOrInstanceId = (uint32_t)mergedHead;
                    temp[unmergedHead++] = nn;
                    mergedHead += 2;
                }
            } else {
                temp[unmergedHead++] = nodes[aId];
            }
        }
        memcpy(nodes + newBegin, temp.data() + newBegin, sizeof(GpuTlasNode) * (size_t)(activeRangeEnd - newBegin));
        activeRangeCount -= merged / 2;
        activeRangeEnd -= merged;
    }
}

} // extern "C"
