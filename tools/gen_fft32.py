"""Emit gypsum_b200/csrc/fft32_gen.cuh: straight-line split-radix DFT codelets (length 32 and 64, forward and inverse) on
float2 = (re, im) register arrays, natural order in and out, written with the float2 helpers of cplx2.cuh (one
helper per complex add, per rotation by +-j and per real-times-complex multiply-add).

Twiddle constants are folded (1, -j, (1-j)/sqrt2 ... are special-cased) and every split-radix butterfly with non-trivial
twiddles is written in the factored ("tangent") form, in which the two twiddle products, their sum / difference and the four
outputs are 8 packed multiply-adds (16 scalar ones) instead of 20 scalar operations:
    w^k z = c1 (z + t1 (j z)),  t1 = tan,  and likewise w^3k z' = c3 (...), so that
    w^k z +- w^3k z' = c1 (a' +- (c3/c1) b')  and  out = u +- c1 (...)  -- each line one FFMA2.
The inverse codelets are the same graphs with conjugated twiddles (tangents negated, -j <-> +j); they are unnormalised.
Every lane of every emitted operation is one IEEE add / fma, in the same order as the scalar re[] / im[] codelets of round 1,
so results are bit-identical to those.
Run:  python tools/gen_fft32.py
"""
import math
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Emitter:
    def __init__(self, inverse: bool):
        self.lines = []
        self.n = 0
        self.ops = 0
        self.sg = -1.0 if inverse else 1.0  # multiplies every twiddle angle: forward exp(-j..), inverse exp(+j..)
        # rotation helpers: forward uses -j where the inverse uses +j
        self.add_rot, self.sub_rot = ("c_sub_mj", "c_add_mj") if inverse else ("c_add_mj", "c_sub_mj")

    def tmp(self, expr):
        name = f"t{self.n}"
        self.n += 1
        self.lines.append(f"    const float2 {name} = {expr};")
        self.ops += 1
        return name

    def lit(self, v):
        return f"{v:.9e}f"

    def add(self, a, b):
        return self.tmp(f"c_add({a}, {b})")

    def sub(self, a, b):
        return self.tmp(f"c_sub({a}, {b})")

    def add_rot_of(self, a, b):  # a + (-+j) b   (forward: -j)
        return self.tmp(f"{self.add_rot}({a}, {b})")

    def sub_rot_of(self, a, b):  # a - (-+j) b
        return self.tmp(f"{self.sub_rot}({a}, {b})")

    def fma(self, c, x, y):  # y + c x
        return self.tmp(f"c_fma({self.lit(c)}, {x}, {y})")

    def fma_j(self, c, x, y):  # y + c (j x)
        return self.tmp(f"c_fma_j({self.lit(c)}, {x}, {y})")

    def fft(self, x):
        n = len(x)
        if n == 1:
            return x
        if n == 2:
            return [self.add(x[0], x[1]), self.sub(x[0], x[1])]
        u = self.fft(x[0::2])
        z = self.fft(x[1::4])
        zp = self.fft(x[3::4])
        out = [None] * n
        q = n // 4
        for k in range(q):
            if k == 0:
                a, b = z[0], zp[0]
                s = self.add(a, b)
                d = self.sub(a, b)  # enters below rotated by -+j
                out[k] = self.add(u[k], s)
                out[k + 2 * q] = self.sub(u[k], s)
                out[k + q] = self.add_rot_of(u[k + q], d)
                out[k + 3 * q] = self.sub_rot_of(u[k + q], d)
                continue
            # a = w^k z = c1 * a1, b = w^3k z' = c3 * b1 with a1, b1 one packed operation each
            if 8 * k == n:  # w = (1 -+ j)/sqrt2, w^3 = (-1 -+ j)/sqrt2: c1 = c3 = 1/sqrt2
                a1 = self.add_rot_of(z[k], z[k])     # z -+ j z
                nb1 = self.sub_rot_of(zp[k], zp[k])  # z' +- j z' = -b1
                c1 = math.sqrt(0.5)
                s1 = self.sub(a1, nb1)
                d1 = self.add(a1, nb1)
            else:
                th1, th3 = -2.0 * math.pi * k / n, -2.0 * math.pi * 3 * k / n
                c1, c3 = math.cos(th1), math.cos(th3)
                t1, t3, rho = self.sg * math.tan(th1), self.sg * math.tan(th3), c3 / c1
                a1 = self.fma_j(t1, z[k], z[k])      # (zr - t1 zi, zi + t1 zr)
                b1 = self.fma_j(t3, zp[k], zp[k])
                s1 = self.fma(rho, b1, a1)
                d1 = self.fma(-rho, b1, a1)
            out[k] = self.fma(c1, s1, u[k])
            out[k + 2 * q] = self.fma(-c1, s1, u[k])
            # forward: -j (a - b) = c1 * (d1.im, -d1.re); inverse: +j (a - b)
            out[k + q] = self.fma_j(-self.sg * c1, d1, u[k + q])
            out[k + 3 * q] = self.fma_j(self.sg * c1, d1, u[k + q])
        return out


def emit(n, inverse):
    e = Emitter(inverse)
    xin = []
    for i in range(n):  # snapshot inputs so the in-place writes below cannot alias
        e.lines.append(f"    const float2 x{i} = x[{i}];")
        xin.append(f"x{i}")
    y = e.fft(xin)
    for k in range(n):
        e.lines.append(f"    x[{k}] = {y[k]};")
    name, sign = ("inv", "+") if inverse else ("fwd", "-")
    head = (f"// {'inverse (unnormalised)' if inverse else 'forward'} DFT-{n}, X[k] = sum_n x[n] exp({sign}2 pi i n k / {n}); {e.ops} packed operations\n"
            f"GB_HD GB_INLINE void fft{n}_{name}(float2 (&x)[{n}]) {{\n")
    return head + "\n".join(e.lines) + "\n}\n"


def main():
    out = ["// GENERATED by tools/gen_fft32.py -- do not edit.", "#pragma once", '#include "cplx2.cuh"', "", "namespace gb {", ""]
    for n in (32, 64):
        out.append(emit(n, False))
        out.append(emit(n, True))
    out.append("}  // namespace gb")
    path = os.path.join(ROOT, "gypsum_b200", "csrc", "fft32_gen.cuh")
    with open(path, "w") as f:
        f.write("\n".join(out) + "\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
