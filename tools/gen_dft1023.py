"""Emit gypsum_b200/csrc/dft1023_gen.cuh: straight-line DFT codelets of the prime-factor (Good-Thomas) 1023-point transform,
1023 = 31 x 33 and 33 = 3 x 11, on float2 = (re, im) register arrays, natural order in and out, written with the float2
helpers of cplx2.cuh so the host lane emulator runs the same IEEE operations.

The prime lengths p = 3, 11, 31 use the symmetric direct form: with a_k = x_k + x_{p-k} and b_k = x_k - x_{p-k} (k = 1..(p-1)/2),
    X_0 = x_0 + sum a_k,   X_j, X_{p-j} = A_j -+ j B_j   (forward),   A_j = x_0 + sum cos(2 pi jk/p) a_k,   B_j = sum sin(2 pi jk/p) b_k,
every product-sum one packed multiply-add.  DFT-33 is the Good-Thomas composition of DFT-3 and DFT-11: coprime lengths, so no
twiddles between the stages.  The inverse codelets are the same graphs with the sines negated; they are unnormalised.
Each codelet is checked against numpy's FFT when this script runs.  The file also holds the per-lane coefficient table of the
31-point row that warp_pfa.cuh spreads over a warp.
Run:  python tools/gen_dft1023.py
"""
import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Emitter:
    """Records one line per packed operation and evaluates the same graph on numpy complex values."""

    def __init__(self, inverse: bool, values):
        self.lines = []
        self.n = 0
        self.ops = 0
        self.sg = -1.0 if inverse else 1.0
        self.val = dict(values)

    def tmp(self, expr, v):
        name = f"t{self.n}"
        self.n += 1
        self.lines.append(f"    const float2 {name} = {expr};")
        self.ops += 1
        self.val[name] = v
        return name

    @staticmethod
    def lit(v):
        return f"{v:.9e}f"

    def add(self, a, b):
        return self.tmp(f"c_add({a}, {b})", self.val[a] + self.val[b])

    def sub(self, a, b):
        return self.tmp(f"c_sub({a}, {b})", self.val[a] - self.val[b])

    def fma(self, c, x, y):  # y + c x
        return self.tmp(f"c_fma({self.lit(c)}, {x}, {y})", self.val[y] + c * self.val[x])

    def fma_j(self, c, x, y):  # y + c (j x)
        return self.tmp(f"c_fma_j({self.lit(c)}, {x}, {y})", self.val[y] + c * 1j * self.val[x])

    def scale_j(self, c, x):  # c (j x)
        return self.tmp(f"c_scale_j({self.lit(c)}, {x})", c * 1j * self.val[x])

    def prime(self, x):
        p = len(x)
        m = (p - 1) // 2
        a = [self.add(x[k], x[p - k]) for k in range(1, m + 1)]
        b = [self.sub(x[k], x[p - k]) for k in range(1, m + 1)]
        out = [None] * p
        s = x[0]
        for k in range(m):
            s = self.add(s, a[k])
        out[0] = s
        for j in range(1, m + 1):
            acc = x[0]
            for k in range(1, m + 1):
                acc = self.fma(math.cos(2.0 * math.pi * j * k / p), a[k - 1], acc)
            # forward X_j = A - j B, X_{p-j} = A + j B; the inverse swaps the signs
            sn = [self.sg * math.sin(2.0 * math.pi * j * k / p) for k in range(1, m + 1)]
            if m == 1:
                out[j] = self.fma_j(-sn[0], b[0], acc)
                out[p - j] = self.fma_j(sn[0], b[0], acc)
                continue
            bj = self.scale_j(sn[0], b[0])
            for k in range(2, m + 1):
                bj = self.fma_j(sn[k - 1], b[k - 1], bj)
            out[j] = self.sub(acc, bj)
            out[p - j] = self.add(acc, bj)
        return out

    def pfa(self, x, n1, n2):
        """Good-Thomas DFT of length n1 n2 (coprime, both prime): x[(n2 i1 + n1 i2) % n] -> X[CRT(k1, k2)]."""
        n = n1 * n2
        u, v = pow(n2, -1, n1), pow(n1, -1, n2)
        y = [[None] * n2 for _ in range(n1)]
        for i2 in range(n2):
            col = self.prime([x[(n2 * i1 + n1 * i2) % n] for i1 in range(n1)])
            for k1 in range(n1):
                y[k1][i2] = col[k1]
        out = [None] * n
        for k1 in range(n1):
            row = self.prime(y[k1])
            for k2 in range(n2):
                out[(n2 * u * k1 + n1 * v * k2) % n] = row[k2]
        return out


def emit(n, inverse, rng):
    vals = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    e = Emitter(inverse, {f"x{i}": vals[i] for i in range(n)})
    xin = []
    for i in range(n):  # snapshot inputs so the in-place writes below cannot alias
        e.lines.append(f"    const float2 x{i} = x[{i}];")
        xin.append(f"x{i}")
    y = e.pfa(xin, 3, 11) if n == 33 else e.prime(xin)
    got = np.array([e.val[t] for t in y])
    want = np.fft.ifft(vals) * n if inverse else np.fft.fft(vals)
    assert np.allclose(got, want, rtol=0, atol=1e-9 * n), (n, inverse)
    for k in range(n):
        e.lines.append(f"    x[{k}] = {y[k]};")
    name, sign = ("inv", "+") if inverse else ("fwd", "-")
    head = (f"// {'inverse (unnormalised)' if inverse else 'forward'} DFT-{n}, X[k] = sum_n x[n] exp({sign}2 pi i n k / {n}); {e.ops} packed operations\n"
            f"GB_HD GB_INLINE void dft{n}_{name}(float2 (&x)[{n}]) {{\n")
    return head + "\n".join(e.lines) + "\n}\n"


def row31_table():
    """Per-lane coefficients of the 31-point row that warp_pfa.cuh spreads over a warp (see row31_dot there)."""
    rows = []
    for lane in range(32):
        if lane == 0:
            c = [1.0] * 15
        elif lane <= 15:
            c = [math.cos(2.0 * math.pi * lane * k / 31) for k in range(1, 16)]
        elif lane <= 30:
            c = [math.sin(2.0 * math.pi * (lane - 15) * k / 31) for k in range(1, 16)]
        else:
            c = [0.0] * 15
        rows.append("    {" + ", ".join(Emitter.lit(v) for v in c + [0.0]) + "}")
    return ("// Initialiser of the [32][16] float table of the 31-point row spread over a warp, k = 1..15: lane 0 sums (1), lane\n"
            "// j = 1..15 takes cos(2 pi j k / 31), lane 15 + j takes sin(2 pi j k / 31), lane 31 is idle (0); column 15 pads to 16.\n"
            "#define GB_ROW31_COEF \\\n  { \\\n" + ", \\\n".join(rows) + " \\\n  }\n")


def main():
    rng = np.random.default_rng(1023)
    out = ["// GENERATED by tools/gen_dft1023.py -- do not edit.", "#pragma once", '#include "cplx2.cuh"', "", "namespace gb {", ""]
    for n in (31, 33):
        out.append(emit(n, False, rng))
        out.append(emit(n, True, rng))
    out.append(row31_table())
    out.append("}  // namespace gb")
    path = os.path.join(ROOT, "gypsum_b200", "csrc", "dft1023_gen.cuh")
    with open(path, "w") as f:
        f.write("\n".join(out) + "\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
