// Complex arithmetic on float2 = (re, im), one IEEE round-to-nearest FP32 add / mul / fma per lane.  Hopper has no
// packed FP32 instructions, so every helper is two scalar instructions per float2 operation (FADD / FMUL / FFMA); the
// same code runs in the host lane emulator (tests/emu) and gives bit-identical results.
#pragma once
#include "gb_common.cuh"

namespace gb {

GB_HD GB_INLINE float2 gb_add2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
GB_HD GB_INLINE float2 gb_mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
GB_HD GB_INLINE float2 gb_fma2(float2 a, float2 b, float2 c) {
    return make_float2(__builtin_fmaf(a.x, b.x, c.x), __builtin_fmaf(a.y, b.y, c.y));
}
#define GB_ADD2(a, b) gb_add2(a, b)
#define GB_MUL2(a, b) gb_mul2(a, b)
#define GB_FMA2(a, b, c) gb_fma2(a, b, c)

GB_HD GB_INLINE float2 c_add(float2 a, float2 b) { return GB_ADD2(a, b); }                                  // a + b
GB_HD GB_INLINE float2 c_sub(float2 a, float2 b) { return GB_ADD2(a, make_float2(-b.x, -b.y)); }            // a - b
GB_HD GB_INLINE float2 c_add_mj(float2 a, float2 b) { return GB_ADD2(a, make_float2(b.y, -b.x)); }          // a + (-j) b
GB_HD GB_INLINE float2 c_sub_mj(float2 a, float2 b) { return GB_ADD2(a, make_float2(-b.y, b.x)); }          // a - (-j) b = a + j b
GB_HD GB_INLINE float2 c_fma(float c, float2 x, float2 y) { return GB_FMA2(x, make_float2(c, c), y); }      // y + c x   (c real)
GB_HD GB_INLINE float2 c_fma_j(float c, float2 x, float2 y) {                                               // y + c (j x)
    return GB_FMA2(make_float2(-x.y, x.x), make_float2(c, c), y);
}
GB_HD GB_INLINE float2 c_scale(float c, float2 x) { return GB_MUL2(x, make_float2(c, c)); }                 // c x
GB_HD GB_INLINE float2 c_scale_j(float c, float2 x) { return GB_MUL2(make_float2(-x.y, x.x), make_float2(c, c)); }  // c (j x)
// Complex products: a multiply of the rotated operand by the imaginary part, then an fma by the real part.
// z * w = (fma(zr, wr, -(zi wi)), fma(zi, wr, zr wi))
GB_HD GB_INLINE float2 cmul(float2 z, float2 w) {
    const float2 p = GB_MUL2(make_float2(-z.y, z.x), make_float2(w.y, w.y));
    return GB_FMA2(z, make_float2(w.x, w.x), p);
}
// z * conj(w) = (fma(zr, wr, zi wi), fma(zi, wr, -(zr wi)))
GB_HD GB_INLINE float2 cmulc(float2 z, float2 w) {
    const float2 p = GB_MUL2(make_float2(z.y, -z.x), make_float2(w.y, w.y));
    return GB_FMA2(z, make_float2(w.x, w.x), p);
}
// e + o * conj(w) = (fma(or, wr, fma(oi, wi, er)), fma(oi, wr, fma(-or, wi, ei)))
GB_HD GB_INLINE float2 cfmac(float2 e, float2 o, float2 w) {
    const float2 t = GB_FMA2(make_float2(o.y, -o.x), make_float2(w.y, w.y), e);
    return GB_FMA2(o, make_float2(w.x, w.x), t);
}

}  // namespace gb
