"""Float64 oracle of the screened Poisson reconstruction (csrc/poisson.cu, rules in include/dss_b200.h).

The system is assembled from its definition, independently of the kernel's hard-coded stencils: on the tensor-product
basis of trilinear hats the operators are Kronecker products of the 1-D mass M1, stiffness K1 and D1[n, m] = int phi_n'
phi_m, and the sample terms come from the sparse (P, nodes) matrix of hat values.  ``solve`` then solves it with
scipy (R <= 32 keeps this quick).  ``marching_tetrahedra`` restates the extraction in numpy with the kernel's float32
operations in the kernel's order, so that its vertices and faces can be compared bit for bit."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

ALPHA = 4.0
F32 = np.float32


def usable(points, normals):
    """rows with finite coordinates and normal and |n| > 0"""
    p, n = np.asarray(points, F32), np.asarray(normals, F32)
    n64 = n.astype(np.float64)
    return np.isfinite(p).all(1) & np.isfinite(n).all(1) & ((n64 * n64).sum(1) > 0)


def domain(points, normals):
    """(usable mask, c (3,) float32, L float32) by the rule of the header"""
    ok = usable(points, normals)
    if not ok.any():
        return ok, np.zeros(3, F32), F32(0)
    q = np.asarray(points, F32)[ok].astype(np.float64)
    lo, hi = q.min(0), q.max(0)
    c = (0.5 * (lo + hi)).astype(F32)
    return ok, c, F32(1.1 * float((hi - lo).max()))


def mats_1d(R):
    """M1, K1, D1 on the nodes [0, R] of [0, 1], h = 1 / R (dense float64)"""
    h, N1 = 1.0 / R, R + 1
    M = np.zeros((N1, N1))
    K = np.zeros((N1, N1))
    D = np.zeros((N1, N1))
    for i in range(R):          # element [x_i, x_i+1]: phi_i = 1 - s, phi_i+1 = s
        M[i:i + 2, i:i + 2] += h * np.array([[1 / 3, 1 / 6], [1 / 6, 1 / 3]])
        K[i:i + 2, i:i + 2] += (1 / h) * np.array([[1, -1], [-1, 1]])
        # D[n, m] = int phi_n' phi_m: phi_i' = -1/h, phi_i+1' = 1/h, int phi = h/2
        D[i:i + 2, i:i + 2] += np.array([[-0.5, -0.5], [0.5, 0.5]])
    return M, K, D


def hat_matrix(u, R):
    """(P, (R+1)^3) sparse matrix of the trilinear hats at the samples u (P,3) in [0,1]^3"""
    N1 = R + 1
    s = u * R
    cell = np.clip(np.floor(s).astype(np.int64), 0, R - 1)
    x = np.clip(s - cell, 0.0, 1.0)
    rows, cols, vals = [], [], []
    P = len(u)
    for a in range(8):
        d = np.array([(a >> 2) & 1, (a >> 1) & 1, a & 1])
        w = np.prod(np.where(d, x, 1.0 - x), axis=1)
        node = ((cell[:, 0] + d[0]) * N1 + cell[:, 1] + d[1]) * N1 + cell[:, 2] + d[2]
        rows.append(np.arange(P))
        cols.append(node)
        vals.append(w)
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(P, N1 ** 3)), cell


def assemble(points, normals, R):
    """the system of the header: dict(A, K, Q, b, a, u, Phi, c, L, usable)"""
    ok, c, L = domain(points, normals)
    p = np.asarray(points, F32)[ok].astype(np.float64)
    n = np.asarray(normals, F32)[ok].astype(np.float64)
    n = n / np.sqrt((n * n).sum(1, keepdims=True))
    u = (p - c.astype(np.float64)) / np.float64(L) + 0.5
    h = 1.0 / R
    Phi, cell = hat_matrix(u, R)
    occ = len(np.unique((cell[:, 0] * R + cell[:, 1]) * R + cell[:, 2]))
    a = h * h * occ / len(p)
    V = (a / h ** 3) * (Phi.T @ n)                       # (nodes, 3)
    M1, K1, D1 = (sp.csr_matrix(m) for m in mats_1d(R))
    kron3 = lambda x, y, z: sp.kron(x, sp.kron(y, z, format="csr"), format="csr")
    K = kron3(K1, M1, M1) + kron3(M1, K1, M1) + kron3(M1, M1, K1)
    b = kron3(D1, M1, M1) @ V[:, 0] + kron3(M1, D1, M1) @ V[:, 1] + kron3(M1, M1, D1) @ V[:, 2]
    Q = (Phi.T @ Phi).tocsr()
    A = (K + ALPHA * a * Q).tocsr()
    return {"A": A, "K": K, "Q": Q, "b": b, "a": a, "u": u, "Phi": Phi, "c": c, "L": L, "usable": ok}


def solve(points, normals, R):
    """chi ((R+1)^3 float64) of the system (relative residual 1e-13), the assembled pieces"""
    s = assemble(points, normals, R)
    A, b = s["A"], s["b"]
    # Jacobi-preconditioned CG in float64 far below the kernel's tolerance (a direct solve is slower at R = 32)
    Minv = sp.diags(1.0 / A.diagonal())
    chi, info = spla.cg(A, b, rtol=1e-13, atol=0.0, maxiter=100000, M=Minv)
    assert info == 0
    return chi, s


# ---- marching tetrahedra -------------------------------------------------------------------------------------------

TETS = [(0, 4, 6, 7), (0, 5, 4, 7), (0, 6, 2, 7), (0, 2, 3, 7), (0, 1, 5, 7), (0, 3, 1, 7)]
OPP = [(1, 2, 3), (0, 3, 2), (0, 1, 3), (0, 2, 1)]


def _tet_triangles(m):
    """triangles of one tetrahedron whose local vertices in bitmask m are inside: lists of three (local a, local b)
    edges, by the rules of the header"""
    ins = [v for v in range(4) if (m >> v) & 1]
    outs = [v for v in range(4) if not (m >> v) & 1]
    if len(ins) in (0, 4):
        return []
    if len(ins) in (1, 3):
        o = ins[0] if len(ins) == 1 else outs[0]
        j = OPP[o] if len(ins) == 1 else (OPP[o][0], OPP[o][2], OPP[o][1])
        return [[(o, j[0]), (o, j[1]), (o, j[2])]]
    perm = ins + outs
    inv = sum(perm[a] > perm[b] for a in range(4) for b in range(a + 1, 4))
    if inv & 1:
        outs = [outs[1], outs[0]]
    q = [(ins[0], outs[0]), (ins[0], outs[1]), (ins[1], outs[1]), (ins[1], outs[0])]
    return [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]


def marching_tetrahedra(chi, center, side):
    """(verts (V,3) float32, faces (F,3) int64) of the chi = 0 surface of the node grid chi (R+1)^3"""
    chi = np.ascontiguousarray(np.asarray(chi, F32))
    R = chi.shape[0] - 1
    N1 = R + 1
    flat = chi.reshape(-1)
    inside = chi < 0
    cross = np.zeros((N1, N1, N1, 8), bool)
    for d in range(1, 8):
        dx, dy, dz = (d >> 2) & 1, (d >> 1) & 1, d & 1
        a = inside[:N1 - dx, :N1 - dy, :N1 - dz]
        b = inside[dx:, dy:, dz:]
        cross[:N1 - dx, :N1 - dy, :N1 - dz, d] = a != b
    idx = np.nonzero(cross.reshape(-1))[0]
    vid = np.full(cross.size, -1, np.int64)
    vid[idx] = np.arange(len(idx))
    node, d = idx // 8, idx % 8
    ijk = [node // (N1 * N1), (node // N1) % N1, node % N1]
    dd = [(d >> 2) & 1, (d >> 1) & 1, d & 1]
    ca = flat[node]
    cb = flat[node + dd[0] * N1 * N1 + dd[1] * N1 + dd[2]]
    t = (F32(0) - ca) / (cb - ca)
    h = F32(1) / F32(R)
    c = np.asarray(center, F32).reshape(3)
    L = F32(side)
    verts = np.empty((len(idx), 3), F32)
    for k in range(3):
        g = np.where(dd[k] == 1, ijk[k].astype(F32) + t, ijk[k].astype(F32)).astype(F32)
        verts[:, k] = c[k] + (g * h - F32(0.5)) * L

    # faces: per tetrahedron and inside pattern, vectorised over the cubes
    ci, cj, ck = np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing="ij")
    ci, cj, ck = ci.reshape(-1), cj.reshape(-1), ck.reshape(-1)
    cube = np.arange(R ** 3)
    n0 = (ci * N1 + cj) * N1 + ck
    corner_in = np.stack([inside[ci + ((a >> 2) & 1), cj + ((a >> 1) & 1), ck + (a & 1)] for a in range(8)], 1)
    keys, tris = [], []
    for t_i, tet in enumerate(TETS):
        m = sum(corner_in[:, tet[v]].astype(np.int64) << v for v in range(4))
        for pattern in range(1, 15):
            sel = m == pattern
            if not sel.any():
                continue
            for f_i, tri in enumerate(_tet_triangles(pattern)):
                ids = []
                for la, lb in tri:
                    A, B = tet[la], tet[lb]
                    s, dirn = A & B, A ^ B
                    nd = n0[sel] + ((s >> 2) & 1) * N1 * N1 + ((s >> 1) & 1) * N1 + (s & 1)
                    ids.append(vid[nd * 8 + dirn])
                tris.append(np.stack(ids, 1))
                keys.append(np.stack([cube[sel], np.full(sel.sum(), t_i), np.full(sel.sum(), f_i)], 1))
    if not tris:
        return verts, np.zeros((0, 3), np.int64)
    tris, keys = np.concatenate(tris), np.concatenate(keys)
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    faces = tris[order]
    assert (faces >= 0).all()
    return verts, faces


# ---- mesh checks ---------------------------------------------------------------------------------------------------

def closed_manifold(faces):
    """every directed edge appears exactly once and its reverse exactly once"""
    f = np.asarray(faces, np.int64)
    if len(f) == 0:
        return True
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = e[:, 0] * (int(f.max()) + 1) + e[:, 1]
    rkey = e[:, 1] * (int(f.max()) + 1) + e[:, 0]
    uniq, counts = np.unique(key, return_counts=True)
    return bool((counts == 1).all() and np.isin(rkey, uniq).all())


def euler_characteristic(verts, faces):
    f = np.asarray(faces, np.int64)
    used = len(np.unique(f))
    return used - 3 * len(f) // 2 + len(f)


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float((a * np.cross(b, c)).sum() / 6.0)
