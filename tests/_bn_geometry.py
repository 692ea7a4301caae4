"""Launch geometry of the channels_last BatchNorm chain kernels (statistics and backward reduction), the
host-side mirror of ``chain_launch`` in ``batchnorm_cl.cu``. Run it to print the geometry per shape:

    python tests/_bn_geometry.py

BY, GY: ATen's ``flexible_launch_configs(M, C, coop=true)`` (GY = 1 when it is below 8: no grid merge).
L: rows per chain; chains of more than 16 rows run on wide blocks (512 threads, up to 8 vector groups).
U: rows in flight per thread in the statistics kernel (4 when L <= 4, else 8).
G, W: vector groups and channels of a slab. CTAs per SM follow from each kernel's ``-Xptxas -v`` registers
for the 16-bit vector path: at 256 threads statistics 64 / 80 registers with U = 4 / 8, reduction 78, with
the ReLU mask 80 where L <= 4 (its parameters read from shared memory), else 118; wide blocks one per SM. Shared memory is sized
to the launch (16.6 KB for ResNet-50's short-chain blocks) and does not limit these counts.
"""
from __future__ import annotations

SMS = 132  # H100 SXM
LONG_CHAIN = 16
STATS_CTAS_PER_SM = {4: 4, 8: 3}
REDUCE_CTAS_PER_SM = {False: 3, True: 3}  # with the mask: 2 where 4 < L <= 16


def last_pow2(n: int) -> int:
    p = 1
    while p * 2 <= n:
        p *= 2
    return p


def cdiv(a: int, b: int) -> int:
    return (a + b - 1) // b


def geometry(M: int, C: int, vec: int) -> dict:
    """vec: 8 for 16-bit, 4 for fp32, 1 for the one-element path"""
    bx = min(last_pow2(C), 32)
    by = min(last_pow2(cdiv(M, 16)), 512 // bx)
    gy = min(cdiv(M, by * 16), 128)
    gy = 1 if gy < 8 else gy
    L = 1 + (M - 1) // (by * gy * 4)
    wide = L > LONG_CHAIN
    G = min(32 if vec == 1 else (8 if wide else 4), cdiv(C, vec))
    W = G * vec
    return {"BY": by, "GY": gy, "L": L, "wide": wide, "U": 4 if L <= 4 and not wide else 8, "G": G, "W": W,
            "slabs": cdiv(C, W), "partial_slab": C % W != 0, "CTAs": cdiv(C, W) * gy,
            "threads": G * min(4 * by, (512 if wide else 256) // G), "staged_per_slot": cdiv(gy, by) if gy > 1 else 0}


def shape_geometry(shape, vec: int = 8) -> dict:
    n, c, h, w = shape
    return geometry(n * h * w, c, vec)


RESNET50 = [(128, 64, 112, 112), (128, 64, 56, 56), (128, 256, 56, 56), (128, 128, 56, 56),
            (128, 128, 28, 28), (128, 512, 28, 28), (128, 256, 28, 28), (128, 256, 14, 14),
            (128, 1024, 14, 14), (128, 512, 14, 14), (128, 512, 7, 7), (128, 2048, 7, 7)]
SMALL = [(4, 64, 5, 5), (8, 3, 17, 19), (2, 16, 33, 31), (4, 96, 9, 7), (3, 100, 11, 13), (16, 1000, 3, 3),
         (64, 256, 1, 1), (5, 40, 1, 1), (1, 8, 2, 3), (2, 5, 1, 1), (8, 100, 16, 16)]


def main():
    print(f"{'shape':>22} {'vec':>3} {'BY':>3} {'GY':>3} {'L':>3} {'U':>2} {'G':>2} {'W':>2} {'slabs':>5} "
          f"{'threads':>7} {'CTAs':>5} {'stats/SM':>8} {'waves':>5} {'red/SM':>6} {'waves':>5} {'relu':>4} {'waves':>5}")
    print("CTAs per SM are those of the 16-bit vector kernels")
    for title, shapes in (("ResNet-50, batch 128", RESNET50), ("SMALL test shapes (16-bit vector path where C % 8 == 0)",
                                                                 SMALL)):
        print(title)
        for s in shapes:
            vec = 8 if s[1] % 8 == 0 else 1
            g = shape_geometry(s, vec)
            st = 1 if g["wide"] else STATS_CTAS_PER_SM[g["U"]]
            rd, rr = (1, 1) if g["wide"] else (REDUCE_CTAS_PER_SM[False], REDUCE_CTAS_PER_SM[True] if g["L"] <= 4 else 2)
            print(f"{'x'.join(map(str, s)):>22} {vec:>3} {g['BY']:>3} {g['GY']:>3} {g['L']:>3} {g['U']:>2} {g['G']:>2} "
                  f"{g['W']:>2} {g['slabs']:>5} {g['threads']:>7} {g['CTAs']:>5} {st:>8} "
                  f"{g['CTAs'] / (SMS * st):>5.1f} {rd:>6} {g['CTAs'] / (SMS * rd):>5.1f} {rr:>4} "
                  f"{g['CTAs'] / (SMS * rr):>5.1f}")


if __name__ == "__main__":
    main()
