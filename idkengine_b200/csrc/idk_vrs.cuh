// Variable-rate deferred lighting for sm_90a: the lighting shading-rate classifier (LightingShadingRateClassifier.Compute,
// Source/Render/LightingShadingRateClassifier.cs) and the deferred lighting draw under its rate image (RasterPipeline.cs:441-463
// with IsVariableRateShading), restated on the device.
//
//   k_shading_rate           ShadingRateClassification/compute.glsl: one 256-thread CTA per 16x16 tile; the speed, luminance
//                            and squared-luminance sums of the tile in a pinned order (per warp an xor butterfly 16, 8, 4, 2, 1,
//                            then thread 0 adds the eight warp sums in order); one R8 palette index per tile and, in DebugMode
//                            2..4, the r32f value the shader stores
//   k_vrs_scan               one CTA: the coarse-fragment count of every tile and their exclusive scan (the last entry is the
//                            total), so the shading kernel's work scales with invocations rather than pixels
//   k_deferred_lighting_vrs  one thread per coarse fragment (256-thread CTAs, the lights staged in shared memory per CTA):
//                            deferred_shade (k_deferred_lighting's body, shared without changing that kernel's SASS) at the
//                            fragment's centre, the result written to every in-image pixel of the fragment
//
// The rules are spelled out in DESIGN.md 8f.1f and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_deferred.cuh"

#define IDK_VRS_TILE 16            // LightingShadingRateClassifier.TILE_SIZE, NV_shading_rate_image's texel footprint

struct ShadingRateArgs {
    const float4* color;           // rgba32f [h][w], the lit image (rgb read)
    const float2* velocity;        // RG float [h][w]
    int w, h;
    float deltaRenderTime, speedFactor, lumVarianceFactor;
    int debugMode;                 // 2 Speed, 3 Luminance, 4 LuminanceVariance: `debug` holds that value
    uint8_t* rates;                // R8 [ceil(h/16)][ceil(w/16)] palette indices 0..4
    float* debug;                  // r32f, same size, or null
};

// subgroupAdd in the pinned order: an xor butterfly over offsets 16, 8, 4, 2, 1. Lanes i and i^o add the same two values, so
// every lane ends with the same sum.
__device__ __forceinline__ float vrs_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

__global__ void __launch_bounds__(256) k_shading_rate(ShadingRateArgs a) {
    __shared__ float s_sums[3][8];  // SharedSpeedSums, SharedLumSums, SharedLumSquaredSums: one entry per warp
    const int lx = (int)threadIdx.x % IDK_VRS_TILE, ly = (int)threadIdx.x / IDK_VRS_TILE;
    const int x = (int)blockIdx.x * IDK_VRS_TILE + lx, y = (int)blockIdx.y * IDK_VRS_TILE + ly;
    // a lane outside the image reads colour 0 and velocity 0 (the robust-access result) and still counts in the mean
    float speed = 0.0f, lum = 0.0f;
    if (x < a.w && y < a.h) {
        const size_t p = (size_t)y * a.w + x;
        const float4 c = a.color[p];
        const float2 vel = a.velocity[p];
        lum = ((c.x + c.y) + c.z) * (1.0f / 3.0f);    // GetLuminance
        speed = sqrtf(vel.x * vel.x + vel.y * vel.y);  // length(velocity)
    }
    const float speedSum = vrs_warp_sum(speed), lumSum = vrs_warp_sum(lum), lumSqSum = vrs_warp_sum(lum * lum);
    if (threadIdx.x % 32 == 0) {
        const int warp = (int)threadIdx.x / 32;
        s_sums[0][warp] = speedSum; s_sums[1][warp] = lumSum; s_sums[2][warp] = lumSqSum;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    float ss = s_sums[0][0], ls = s_sums[1][0], lq = s_sums[2][0];
    for (int i = 1; i < 8; i++) { ss += s_sums[0][i]; ls += s_sums[1][i]; lq += s_sums[2][i]; }

    const float meanSpeed = (ss / 256.0f) / a.deltaRenderTime;
    const float lumMean = ls / 256.0f;
    uint32_t rate;
    float cov;
    if (lumMean <= 0.001f) {
        rate = 4u;                 // ENUM_SHADING_RATE_1_INVOCATION_PER_4X4_PIXELS_NV
        cov = 0.0f;
    } else {
        const float lumSqMean = lq / 256.0f;
        const float variance = lumSqMean - lumMean * lumMean;
        cov = sqrtf(variance) / lumMean;
        const float combined = mix1(0.0f, 4.0f, meanSpeed * a.speedFactor) + mix1(0.0f, 4.0f, a.lumVarianceFactor / cov);
        // round() half to even, then uint(): cvt.rzi.sat.u32 (NaN and negatives 0, overflow UINT_MAX), then clamp(.., 0, 4)
        rate = min(__float2uint_rz(rintf(combined)), 4u);
    }
    const size_t t = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
    a.rates[t] = (uint8_t)rate;
    if (a.debug) a.debug[t] = a.debugMode == 2 ? meanSpeed : a.debugMode == 3 ? lumMean : cov;
}

// The coarse fragment of palette index r (the engine's palette {1x1, 2x1, 2x2, 4x2, 4x4}): width cw, height ch in pixels.
__device__ __forceinline__ void vrs_fragment_size(uint32_t r, int& cw, int& ch) {
    cw = r == 0u ? 1 : r <= 2u ? 2 : 4;
    ch = r <= 1u ? 1 : r <= 3u ? 2 : 4;
}

struct VrsTiles {
    const uint8_t* rates;          // [tilesY][tilesX], the context's classifier image
    uint32_t* offsets;             // [tiles + 1]: first coarse fragment of each tile; offsets[tiles] = the fragment count
    int w, h, tilesX, tiles;
};

// Coarse fragments of tile t: ceil(tw / cw) * ceil(th / ch) over the tile's in-image extent tw x th.
__device__ __forceinline__ uint32_t vrs_tile_fragments(const VrsTiles& v, int t) {
    int cw, ch;
    vrs_fragment_size(v.rates[t], cw, ch);
    const int tw = min(IDK_VRS_TILE, v.w - (t % v.tilesX) * IDK_VRS_TILE), th = min(IDK_VRS_TILE, v.h - (t / v.tilesX) * IDK_VRS_TILE);
    return (uint32_t)(((tw + cw - 1) / cw) * ((th + ch - 1) / ch));
}

// One 1024-thread CTA: thread i counts a contiguous run of ceil(tiles / 1024) tiles, the CTA scans the run totals, and each
// thread writes its run's offsets. 8,160 tiles at 1080p, at most 1,048,576 at 16384^2 (a count of at most 2^28 fits).
__global__ void __launch_bounds__(1024) k_vrs_scan(VrsTiles v) {
    __shared__ uint32_t s_warp[32];
    const int per = (v.tiles + 1023) / 1024;
    const int begin = min((int)threadIdx.x * per, v.tiles), end = min(begin + per, v.tiles);
    uint32_t run = 0;
    for (int t = begin; t < end; t++) run += vrs_tile_fragments(v, t);
    const int lane = (int)threadIdx.x % 32, warp = (int)threadIdx.x / 32;
    uint32_t incl = run;           // inclusive scan within the warp, then over the warp totals
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, w, o);
            if (lane >= o) w += n;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    uint32_t offset = (incl - run) + (warp > 0 ? s_warp[warp - 1] : 0u);
    for (int t = begin; t < end; t++) {
        v.offsets[t] = offset;
        offset += vrs_tile_fragments(v, t);
    }
    if (threadIdx.x == 1023) v.offsets[v.tiles] = offset;
}

// NV_shading_rate_image under the engine's palette: the rate of pixel (x, y) is texel (x / 16, y / 16); a coarse fragment of
// cw x ch pixels is aligned to multiples of (cw, ch) from (0, 0), so it never crosses a tile. The fragment shader runs once, at
// the centre of the fragment's area: uv = ((x0 + cw / 2) / W, (y0 + ch / 2) / H) and imgCoord = ivec2(gl_FragCoord) =
// (x0 + cw / 2, y0 + ch / 2) in integers, clamped to the last column / row where the centre lies outside an odd-sized image.
// Its one result goes to every in-image pixel of the fragment.
__global__ void __launch_bounds__(256) k_deferred_lighting_vrs(DeferredArgs a, VrsTiles v) {
    const uint32_t total = v.offsets[v.tiles];
    if (blockIdx.x * 256u >= total) return;   // the grid is sized for all 1x1; CTAs past the fragment count leave at once
    __shared__ GpuLight s_lights[IDK_GPU_MAX_UBO_LIGHT_COUNT];
    volatile __shared__ uint32_t s_span[256];
    for (int i = threadIdx.x; i < a.lightCount; i += blockDim.x) s_lights[i] = a.lights[i];
    __syncthreads();
    const uint32_t f = blockIdx.x * 256u + threadIdx.x;
    if (f >= total) return;
    int lo = 0, hi = v.tiles - 1;  // the fragment's tile: the last t with offsets[t] <= f (every tile has a fragment)
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (__ldg(v.offsets + mid) <= f) lo = mid; else hi = mid - 1;
    }
    const int t = lo, tx = t % v.tilesX, ty = t / v.tilesX;
    int cw, ch;
    vrs_fragment_size(v.rates[t], cw, ch);
    const int tw = min(IDK_VRS_TILE, a.g.w - tx * IDK_VRS_TILE);
    const int nx = (tw + cw - 1) / cw, local = (int)(f - __ldg(v.offsets + t));
    const int x0 = tx * IDK_VRS_TILE + (local % nx) * cw, y0 = ty * IDK_VRS_TILE + (local / nx) * ch;
    const int ix = min(x0 + cw / 2, a.g.w - 1), iy = min(y0 + ch / 2, a.g.h - 1);
    // the fragment's in-image pixels wait in shared memory while it is shaded (in registers they spill at the 80 ptxas allots
    // for three CTAs per SM): the first pixel's index (< 2^28) and the column and row counts less one (1..4 each)
    s_span[threadIdx.x] = (uint32_t)(y0 * a.g.w + x0) | ((uint32_t)(min(x0 + cw, a.g.w) - x0 - 1) << 28) |
                          ((uint32_t)(min(y0 + ch, a.g.h) - y0 - 1) << 30);
    deferred_shade(a, s_lights, (size_t)iy * a.g.w + ix,
                   [&]() { return make_float2(((float)x0 + 0.5f * (float)cw) / (float)a.g.w, ((float)y0 + 0.5f * (float)ch) / (float)a.g.h); },
                   [&](float4 c) {
                       const uint32_t span = s_span[threadIdx.x], first = span & 0x0FFFFFFFu;
                       const int cols = (int)((span >> 28) & 3u) + 1, rows = (int)(span >> 30) + 1;
                       for (int y = 0; y < rows; y++)
                           for (int x = 0; x < cols; x++) a.out[(size_t)first + (size_t)y * a.g.w + x] = c;
                   });
}
