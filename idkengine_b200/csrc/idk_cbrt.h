// Single-precision cube root equal, bit for bit, to glibc's cbrtf on every non-NaN float.
//
// PreSplitting.GetPriority (PreSplitting.cs) takes MathF.Cbrt, which on Linux is libm's cbrtf; the host mirror
// (host_mirror/bvh_build.cpp, priority()) calls it directly. glibc's cbrtf is not correctly rounded: it differs from
// (float)cbrt((double)x) on about a tenth of all positive floats, so neither CUDA's cbrtf nor a double-precision cube
// root reproduces the host's split counts. This is glibc's algorithm restated (sysdeps/ieee754/flt-32/s_cbrtf.c):
// a quadratic first guess of the mantissa's cube root in double, one Halley step, a power-of-two correction for the
// exponent modulo 3. frexp and ldexp are done on the bits so that host and device run the same code; the result of
// the ldexp is always a normal float (|exponent| / 3 <= 50), so adding to the exponent field is exact.
//
// tests/test_blas_build.py compiles this header with g++ -ffp-contract=off and compares it with the running libm's
// cbrtf on all 2^32 bit patterns. Device code needs -fmad=false (libidkpt's flags): the double expressions below
// must not be contracted.
#ifndef IDK_CBRT_H
#define IDK_CBRT_H

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define IDK_CBRT_HD __host__ __device__ __forceinline__
#else
#define IDK_CBRT_HD static inline
#endif

IDK_CBRT_HD uint32_t idk_cbrt_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
IDK_CBRT_HD float idk_cbrt_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

IDK_CBRT_HD float idk_cbrtf(float x) {
    const uint32_t bits = idk_cbrt_bits(x);
    const uint32_t mag = bits & 0x7FFFFFFFu;
    if (mag == 0u || mag >= 0x7F800000u) return x + x;          // +-0, +-inf, NaN
    // frexpf(|x|, &xe): |x| = xm * 2^xe, xm in [0.5, 1)
    uint32_t m = mag;
    int xe = 0;
    if (m < 0x00800000u) {                                      // subnormal: scale by 2^25 (exact) first
        m = idk_cbrt_bits(idk_cbrt_float(m) * 33554432.0f);
        xe = -25;
    }
    xe += (int)(m >> 23) - 126;
    const float xm = idk_cbrt_float((m & 0x007FFFFFu) | (126u << 23));

    const double cbrt2 = 1.2599210498948731648, sqrCbrt2 = 1.5874010519681994748;   // 2^(1/3), 2^(2/3)
    const double factor[5] = {1.0 / sqrCbrt2, 1.0 / cbrt2, 1.0, cbrt2, sqrCbrt2};
    const float u = (float)(0.492659620528969547 + (0.697570460207922770 - 0.191502161678719066 * (double)xm) * (double)xm);
    const float t2 = u * u * u;
    const float ym = (float)((double)u * ((double)t2 + 2.0 * (double)xm) / (2.0 * (double)t2 + (double)xm) * factor[2 + xe % 3]);
    // ldexpf(x > 0 ? ym : -ym, xe / 3)
    const uint32_t yb = idk_cbrt_bits(ym) + ((uint32_t)(xe / 3) << 23);
    return idk_cbrt_float(yb | (bits & 0x80000000u));
}

#endif
