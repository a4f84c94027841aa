"""Float32 restatement of the mesh rasterizer's rules (include/dss_b200.h, dss_rasterize_mesh): per pixel, every face in
index order.  numpy rounds every float32 operation on its own (no contraction), in the order written here, which is the
order of the kernel's explicit __fmul_rn / __fsub_rn / __fadd_rn / __fdiv_rn: the two agree bit for bit.

The input is the screen-space vertices of each view, (N,V,3) {NDC x, NDC y, view z}; on the GPU the tests take them
from ``preprocess_points`` on the vertices, the expression the kernel uses for its own transform."""
import numpy as np

f32 = np.float32
EPS = f32(1e-8)


def pix_to_ndc(i, S):
    """-1 + (2 i + 1) / S in float32 (common.cuh pix_to_ndc)."""
    return f32(-1) + (f32(2) * np.asarray(i, dtype=np.float32) + f32(1)) / f32(S)


def edge(px, py, ax, ay, bx, by):
    """E(p, a, b) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x)."""
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def rasterize_mesh_naive(screen, faces, S):
    """screen (N,V,3) f32, faces (F,3) int -> pix_to_face (N,S,S) i32, zbuf (N,S,S) f32 (-1 where uncovered).

    Image row r, column c has the centre (pix_to_ndc(S-1-c), pix_to_ndc(S-1-r)).  A face is skipped where
    max(z) < 0 (fmax: NaN ignored), where |E(v0, v1, v2)| <= 1e-8, and at pixels outside its closed bounding box; the
    pixels inside are tested face by face in index order, and a face replaces the current one only at a strictly smaller
    depth, so exact ties stay with the smaller index."""
    screen = np.asarray(screen, dtype=np.float32)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    N = screen.shape[0]
    ndc = pix_to_ndc(np.arange(S), S)            # by pixel index, before the flip
    p2f = np.full((N, S, S), -1, np.int32)
    zbuf = np.full((N, S, S), -1, np.float32)
    with np.errstate(all="ignore"):
        for n in range(N):
            best_z = np.zeros((S, S), np.float32)    # indexed [y index, x index]
            best_f = np.full((S, S), -1, np.int64)
            for f, (i0, i1, i2) in enumerate(faces):
                v0, v1, v2 = screen[n, i0], screen[n, i1], screen[n, i2]
                zmax = np.fmax(np.fmax(v0[2], v1[2]), v2[2])
                if zmax < 0:
                    continue
                area = edge(v0[0], v0[1], v1[0], v1[1], v2[0], v2[1])
                if -EPS <= area <= EPS:
                    continue
                xmin, xmax = np.fmin(np.fmin(v0[0], v1[0]), v2[0]), np.fmax(np.fmax(v0[0], v1[0]), v2[0])
                ymin, ymax = np.fmin(np.fmin(v0[1], v1[1]), v2[1]), np.fmax(np.fmax(v0[1], v1[1]), v2[1])
                xs = np.nonzero((ndc >= xmin) & (ndc <= xmax))[0]
                ys = np.nonzero((ndc >= ymin) & (ndc <= ymax))[0]
                if not len(xs) or not len(ys):
                    continue
                px, py = ndc[xs][None, :], ndc[ys][:, None]
                den = edge(v2[0], v2[1], v0[0], v0[1], v1[0], v1[1]) + EPS
                w0 = edge(px, py, v1[0], v1[1], v2[0], v2[1]) / den
                w1 = edge(px, py, v2[0], v2[1], v0[0], v0[1]) / den
                w2 = edge(px, py, v0[0], v0[1], v1[0], v1[1]) / den
                pz = (w0 * v0[2] + w1 * v1[2]) + w2 * v2[2]
                cov = (w0 > 0) & (w1 > 0) & (w2 > 0) & (pz >= 0)
                sub_z, sub_f = best_z[np.ix_(ys, xs)], best_f[np.ix_(ys, xs)]
                take = cov & ((sub_f < 0) | (pz < sub_z))
                sub_z[take] = pz[take]
                sub_f[take] = f
                best_z[np.ix_(ys, xs)], best_f[np.ix_(ys, xs)] = sub_z, sub_f
            hit = best_f >= 0
            # pixel index (x, y) -> image row S-1-y, column S-1-x
            p2f[n] = np.where(hit, best_f, -1)[::-1, ::-1]
            zbuf[n] = np.where(hit, best_z, f32(-1))[::-1, ::-1]
    return p2f, zbuf
