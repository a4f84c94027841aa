"""Float64 restatement of the fused shading's gradients with an error bound per output (csrc/shading.cuh: shade_light,
shade_point, normalize3_bwd; csrc/render.cu: shade_backward_kernel, shade_backward_packed_kernel,
camera_partials_kernel<true>, light_partials_kernel).

The shading is DSS/core/lighting.py (dss_b200/core/lighting.py): colour = albedo * (ambient + diffuse) + specular with
F.normalize(eps=1e-6) on the normal, the light direction (or location - point) and the view direction (camera - point).
`shade_grads` evaluates, for each (view, point) slot and its d L / d shaded `gc`, every gradient the kernels take from
the slot: per light the direction / location row, the diffuse and specular colours, the ambient colour, the camera
centre, and the albedo, normal and position.  It follows the kernels' expression order once, generically over the
number type, so the same code gives:

  - `Bounded`: the float64 value of every intermediate together with a running bound on what a float32 evaluation of
    the same expression may differ from it: every operation adds u·|result| (u = 2^-24), products and sums carry their
    operands' bounds weighted by the other operand's magnitude, that is c·u·Σ|terms| with c counted along each term's
    path, as the preprocess bound (tests/test_preprocess_bound.py) does.  No FMA is assumed, so the bound holds for any
    contraction.  A result of exact operands that float32 represents is exact (zeros, x - 0, the norm of a vector
    along an axis), so n·d = 0 and |x| = eps exactly stay decided; a result that may underflow adds half the subnormal
    spacing.  powf adds 4 ulp, and alpha^(shin-1) / alpha^shin are counted at alpha + e_alpha.  A branch
    (n·d > 0, alpha > 0, |x| >= eps) whose operand lies within its own bound of the threshold may go either way: the
    bound there also holds the distance between the two sides.  Elsewhere the branch is the float64 one.
  - `Rounded(bits)`: the same expressions with every operation rounded to `bits` significant bits (24: float32
    without FMA), the CPU stand-in for the kernels.

The eps rule is float32 F.normalize's: x / clamp_min(|x|, eps) with eps = float32(1e-6); the gradient passes through
the norm where |x| >= eps, at equality too, and only below it is the map linear (g / eps).

`SAFETY` multiplies the bound for the higher-order terms; `within` adds half an ulp for the final float32 rounding.
Below shininess 1 the reference's pow backward is NaN at alpha = 0 (0^(shin-1)); the kernels gate it, so shininess < 1
is left out of the tests."""
import numpy as np

U = 2.0 ** -24
EPS32 = float(np.float32(1e-6))
POW_ULP = 4            # powf: CUDA's maximum error in ulp (1 ulp <= 2u relative)
TINY = 2.0 ** -150     # half the subnormal spacing: the absolute rounding error of a result that underflows
SAFETY = 1.5


def _rnd(v, e):
    """the rounding of a result within e of v: u relative, or half the subnormal spacing where it may underflow; a
    result of exact operands (e = 0) that float32 represents (0, x - 0, Sterbenz differences, ...) rounds to itself"""
    m = np.abs(v) + e
    with np.errstate(over="ignore", invalid="ignore"):
        exact = (e == 0) & (np.asarray(v, np.float64).astype(np.float32).astype(np.float64) == v)
    return np.where(exact, 0.0, U * m + np.where((m > 0) & (m < 2.0 ** -125), TINY, 0.0))


# ---- number types ---------------------------------------------------------------------------------------------------
class Bounded:
    """float64 value `v` and a bound `e` on the distance of a float32 evaluation from it"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else e

    @staticmethod
    def lift(x):
        return x if isinstance(x, Bounded) else Bounded(x)

    def __add__(self, o):
        o = Bounded.lift(o)
        v = self.v + o.v
        e = self.e + o.e
        return Bounded(v, e + _rnd(v, e))

    __radd__ = __add__

    def __sub__(self, o):
        o = Bounded.lift(o)
        v = self.v - o.v
        e = self.e + o.e
        return Bounded(v, e + _rnd(v, e))

    def __rsub__(self, o):
        return Bounded.lift(o) - self

    def __neg__(self):
        return Bounded(-self.v, self.e)

    def __mul__(self, o):
        o = Bounded.lift(o)
        v = self.v * o.v
        e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e
        return Bounded(v, e + _rnd(v, e))

    __rmul__ = __mul__

    def sqrt(self):
        v = np.sqrt(self.v)
        lo = np.sqrt(np.maximum(self.v - self.e, 0.0))
        e = 2 * self.e / np.maximum(np.sqrt(self.v + self.e) + lo, 1e-300)
        e = np.where(self.e == 0, 0.0, e)
        return Bounded(v, e + _rnd(v, e))

    def rcp(self):
        v = 1.0 / self.v
        lo = self.v - self.e
        e = np.where(lo > 0, self.e / (np.abs(self.v) * np.maximum(lo, 1e-300)), np.inf)
        e = np.where(self.e == 0, 0.0, e)
        return Bounded(v, e + _rnd(v, e))

    def fmax(self, c):
        v = np.maximum(self.v, c)                              # exact; a bound that stays below c vanishes
        e = np.maximum(np.maximum(self.v + self.e, c) - v, v - np.maximum(self.v - self.e, c))
        return Bounded(v, e)

    def pow(self, s):
        a = np.maximum(self.v, 0.0)
        hi = (a + self.e) ** s
        v = a ** s
        e = np.maximum(hi - v, v - np.maximum(a - self.e, 0.0) ** s)
        return Bounded(v, e + POW_ULP * (2 * U * hi + 2 * TINY))

    @staticmethod
    def select(x, t, a, b, strict=True):
        """x > t (strict) or x >= t ? a : b"""
        a, b = Bounded.lift(a), Bounded.lift(b)
        take = x.v > t if strict else x.v >= t
        v = np.where(take, a.v, b.v)
        e = np.where(take, a.e, b.e)
        lo, hi = x.v - x.e, x.v + x.e
        sure = (lo > t) | (hi < t) | ((hi <= t) if strict else (lo >= t))
        flip = np.abs(a.v - b.v) + a.e + b.e
        e = np.where(sure | np.isnan(x.v), e, np.maximum(e, flip))
        return Bounded(v, e)

    @staticmethod
    def keep(mask, a):
        """a where mask, exactly 0 elsewhere (the kernels skip slots with d L / d shaded == 0)"""
        return Bounded(np.where(mask, a.v, 0.0), np.where(mask, a.e, 0.0))


def rounded(bits):
    """the number type that rounds every operation to `bits` significant bits"""
    if bits == 24:
        def r(v):
            with np.errstate(over="ignore", invalid="ignore"):
                return np.asarray(v, np.float64).astype(np.float32).astype(np.float64)
    else:
        def r(v):
            v = np.asarray(v, np.float64)
            m, e = np.frexp(v)
            return np.ldexp(np.round(m * 2.0 ** bits) / 2.0 ** bits, e)

    class Rounded:
        __slots__ = ("v",)

        def __init__(self, v):
            self.v = np.asarray(v, np.float64)

        @staticmethod
        def lift(x):
            return x if isinstance(x, Rounded) else Rounded(r(x))

        def __add__(self, o):
            return Rounded(r(self.v + Rounded.lift(o).v))

        __radd__ = __add__

        def __sub__(self, o):
            return Rounded(r(self.v - Rounded.lift(o).v))

        def __rsub__(self, o):
            return Rounded.lift(o) - self

        def __neg__(self):
            return Rounded(-self.v)

        def __mul__(self, o):
            return Rounded(r(self.v * Rounded.lift(o).v))

        __rmul__ = __mul__

        def sqrt(self):
            return Rounded(r(np.sqrt(self.v)))

        def rcp(self):
            return Rounded(r(1.0 / self.v))

        def fmax(self, c):
            return Rounded(np.where(np.isnan(self.v), r(c), np.maximum(self.v, r(c))))   # fmaxf ignores a NaN

        def pow(self, s):
            return Rounded(r(np.maximum(self.v, 0.0) ** s))

        @staticmethod
        def select(x, t, a, b, strict=True):
            a, b = Rounded.lift(a), Rounded.lift(b)
            return Rounded(np.where(x.v > r(t) if strict else x.v >= r(t), a.v, b.v))

        @staticmethod
        def keep(mask, a):
            return Rounded(np.where(mask, a.v, 0.0))

    return Rounded


# ---- the kernels' expressions ---------------------------------------------------------------------------------------
def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _add(a, b):
    return tuple(x + y for x, y in zip(a, b))


def _sub(a, b):
    return tuple(x - y for x, y in zip(a, b))


def _mul(a, s):
    return tuple(x * s for x in a)


def _normalize(a, T):
    """-> (a / max(|a|, eps), clamped length, raw length)"""
    raw = _dot(a, a).sqrt()
    if T is Bounded:
        # sqrtf(fl(x * x)) is |x| exactly (no underflow): a vector along an axis has an exact norm, so the eps branch
        # of normalize3_bwd is decided at |x| = eps exactly and one ulp either side
        axis = (sum((x.v != 0).astype(int) for x in a) == 1) & (sum(x.e for x in a) == 0)
        raw = Bounded(np.where(axis, sum(np.abs(x.v) for x in a), raw.v), np.where(axis, 0.0, raw.e))
    ln = raw.fmax(EPS32)
    return _mul(a, ln.rcp()), ln, raw


def _normalize_bwd(y, ln, raw, gy, T):
    inv = ln.rcp()
    proj = _mul(_sub(gy, _mul(y, _dot(y, gy))), inv)
    lin = _mul(gy, inv)
    return tuple(T.select(raw, EPS32, pc, lc, strict=False) for pc, lc in zip(proj, lin))


def _shade_light(L, light_type, shin, p, nh, v, alb, gc, T):
    """shade_light<true>: -> dict(d, dlen, draw, lam, pw, g_d, g_nh, g_v) of one light (g_nh / g_v: its share)"""
    zero = T.lift(np.zeros_like(p[0].v))
    draw = _sub(L[0:3], p) if light_type else tuple(L[0:3])
    d, dlen, dr = _normalize(draw, T)
    cd, cs = L[3:6], L[6:9]
    cos = _dot(nh, d)
    lam = cos.fmax(0.0)
    r = _add(_mul(d, -1.0), _mul(nh, 2.0 * cos))
    vr = _dot(v, r)
    alpha = T.select(cos, 0.0, vr.fmax(0.0), zero)
    pw = T.select(alpha, 0.0, alpha.pow(shin), zero)
    g_cos = T.select(cos, 0.0, gc[0] * alb[0] * cd[0] + gc[1] * alb[1] * cd[1] + gc[2] * alb[2] * cd[2], zero)
    g_alpha = T.select(alpha, 0.0, _dot(gc, cs) * shin * alpha.pow(shin - 1.0), zero)
    g_r = _mul(v, g_alpha)
    g_v = _mul(r, g_alpha)
    g_cos = g_cos + 2.0 * _dot(g_r, nh)
    g_nh = _add(_mul(g_r, 2.0 * cos), _mul(d, g_cos))
    g_d = _add(_mul(g_r, -1.0), _mul(nh, g_cos))
    return dict(d=d, dlen=dlen, draw=dr, lam=lam, pw=pw, g_d=g_d, g_nh=g_nh, g_v=g_v)


def shade_grads(T, p, n, alb, cam, lights, amb, gc, light_type, shin):
    """Per slot, in number type T.  p, n, alb, cam, amb, gc: (M,3); lights (M,L,9) the slot's light rows.
    -> dict of T triples: alb, nrm, pos, cam (the shading kernels) and, per light l, vec[l], cd[l], cs[l], and amb
    (light_partials_kernel).  Slots with gc == 0 give exactly 0."""
    M, L = lights.shape[0], lights.shape[1]
    col = lambda a, k: T.lift(np.asarray(a, np.float64)[:, k])
    P, N_, A, C, G, AM = ([col(a, k) for k in range(3)] for a in (p, n, alb, cam, gc, amb))
    live = np.asarray(gc != 0).any(1)
    nh, nlen, nraw = _normalize(tuple(N_), T)
    v, vlen, vraw = _normalize(_sub(C, P), T)
    zero3 = tuple(T.lift(np.zeros(M)) for _ in range(3))
    diff, g_nh, g_v, g_pos = zero3, zero3, zero3, zero3
    out = dict(vec=[], cd=[], cs=[])
    ga = tuple(G[k] * A[k] for k in range(3))
    for l in range(L):
        row = [col(lights[:, l], k) for k in range(9)]
        t = _shade_light(row, light_type, shin, P, nh, v, A, G, T)
        diff = _add(diff, _mul(row[3:6], t["lam"]))
        g_nh = _add(g_nh, t["g_nh"])
        g_v = _add(g_v, t["g_v"])
        gvec = _normalize_bwd(t["d"], t["dlen"], t["draw"], t["g_d"], T)
        if light_type:
            g_pos = _sub(g_pos, gvec)
        out["vec"].append(gvec)
        out["cd"].append(tuple(ga[k] * t["lam"] for k in range(3)))
        out["cs"].append(tuple(G[k] * t["pw"] for k in range(3)))
    out["amb"] = ga
    out["alb"] = tuple(G[k] * (AM[k] + diff[k]) for k in range(3))
    out["nrm"] = _normalize_bwd(nh, nlen, nraw, g_nh, T)
    g_cam = _normalize_bwd(v, vlen, vraw, g_v, T)
    out["pos"] = _sub(g_pos, g_cam)
    out["cam"] = g_cam
    keep = lambda tr: tuple(T.keep(live, x) for x in tr)
    return {k: ([keep(x) for x in val] if isinstance(val, list) else keep(val)) for k, val in out.items()}


def stack(tr):
    """a triple of per-slot numbers -> (M,3) values (and (M,3) bounds for Bounded)"""
    v = np.stack([x.v for x in tr], 1)
    return (v, np.stack([x.e for x in tr], 1)) if isinstance(tr[0], Bounded) else v


def slot_outputs(T, s):
    """shade_grads on a slot dict (p, n, alb, cam, lights, amb, gc, light_type, shin) -> dict name -> (M, ..., 3)
    arrays: alb, nrm, pos, cam, amb (M,3), vec / cd / cs (M,L,3); Bounded: (values, bounds) pairs"""
    o = shade_grads(T, s["p"], s["n"], s["alb"], s["cam"], s["lights"], s["amb"], s["gc"], s["light_type"], s["shin"])
    res = {}
    for k in ("alb", "nrm", "pos", "cam", "amb"):
        res[k] = stack(o[k])
    for k in ("vec", "cd", "cs"):
        per = [stack(x) for x in o[k]]
        res[k] = (np.stack([x[0] for x in per], 1), np.stack([x[1] for x in per], 1)) if T is Bounded else \
            np.stack(per, 1)
    return res


def within(got, want, bound, safety=SAFETY):
    """-> (ratio of |got - want| to the bound (+ half an ulp of the float32 result), NaN agreement mask).  NaN in
    `want` must be NaN in `got`; the ratio there is 0."""
    got, want, bound = (np.asarray(x, np.float64) for x in (got, want, bound))
    nan_w, nan_g = np.isnan(want), np.isnan(got)
    same_nan = nan_w == nan_g
    with np.errstate(invalid="ignore", over="ignore"):
        tol = safety * bound + U * np.abs(want) + 2.0 ** -149
        ratio = np.where(nan_w | nan_g, 0.0, np.abs(got - want) / tol)
        ratio = np.where(np.isnan(ratio), np.inf, ratio)
    return ratio, same_nan


# ---- slot families --------------------------------------------------------------------------------------------------
def _f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def _up(x):
    return float(np.nextafter(np.float32(x), np.float32(np.inf)))


def _down(x):
    return float(np.nextafter(np.float32(x), np.float32(-np.inf)))


def edge_slots(kind, L, shin, seed=0):
    """The hand-built edge slots, one light row set per slot (light 0 carries the edge, the others are ordinary).
    -> (slot dict, list of family labels per slot).  Every vector is exact in float32."""
    rng = np.random.default_rng(seed)
    lt = 1 if kind == "point" else 0
    rows, labels = [], []

    def add(label, p, n, cam, d0=None, loc0=None, cd=None, cs=None, alb=(0.7, 0.5, 0.3), gc=None):
        lr = np.zeros((L, 9))
        for l in range(L):
            vec = rng.normal(size=3) * (1.0 if lt == 0 else 1.5)
            lr[l] = np.concatenate([vec, 0.6 * rng.random(3), 0.5 * rng.random(3)])
        if lt == 0 and d0 is not None:
            lr[0, :3] = d0
        if lt == 1:
            lr[0, :3] = loc0 if loc0 is not None else (np.asarray(p) + np.asarray(d0 if d0 is not None else (1, 0, 0)))
        if cd is not None:
            lr[:, 3:6] = cd
        if cs is not None:
            lr[:, 6:9] = cs
        g = rng.normal(size=3) if gc is None else gc
        rows.append(dict(p=p, n=n, alb=alb, cam=cam, lights=_f32(lr), gc=g))
        labels.append(label)

    p0 = np.array([0.5, 0.25, -0.125])
    # n.d = 0 exactly (axis-aligned), and n.d = +-2^-40 exactly; the camera in the mirror direction keeps the
    # specular live wherever the mask lets it
    for lab, dz in (("n.d=0", 0.0), ("n.d=+tiny", 2.0 ** -40), ("n.d=-tiny", -(2.0 ** -40))):
        add(lab, p0, (0.0, 0.0, 2.0), p0 + np.array([-1.5, 0.0, 0.0]), d0=(1.0, 0.0, dz))
        add(lab, p0, (0.0, 0.0, 2.0), p0 + np.array([-1.0, 0.0, 0.5]), d0=(1.0, 0.0, dz))
    # v.r = 0 exactly (light head-on, camera along x) and v.r = 2^-30 exactly
    for lab, vz in (("v.r=0", 0.0), ("v.r=+tiny", 2.0 ** -30)):
        add(lab, p0, (0.0, 0.0, 1.0), p0 + np.array([1.0, 0.0, vz]), d0=(0.0, 0.0, 1.0))
    # zero normals
    add("zero normal", p0, (0.0, 0.0, 0.0), p0 + np.array([0.3, -1.0, 0.8]), d0=(0.2, 0.3, 1.0))
    # normals of length float32(1e-6) exactly, one ulp below and one above
    for lab, ln in (("|n|=eps", EPS32), ("|n|=eps-ulp", _down(EPS32)), ("|n|=eps+ulp", _up(EPS32))):
        add(lab, p0, (0.0, 0.0, ln), p0 + np.array([0.3, -0.5, 1.0]), d0=(0.2, 0.3, 1.0))
        add(lab, p0, (ln, 0.0, 0.0), p0 + np.array([1.0, 0.4, 0.2]), d0=(1.0, 0.1, 0.3))
    # a point at the camera centre, and 1e-6f (and one ulp either side) from it
    pc = np.array([0.0, 0.5, 0.25])
    for lab, off in (("at camera", 0.0), ("camera eps", EPS32), ("camera eps-ulp", _down(EPS32)),
                     ("camera eps+ulp", _up(EPS32))):
        add(lab, pc, (0.3, 0.4, 1.0), pc + np.array([off, 0.0, 0.0]), d0=(0.2, 0.3, 1.0))
    # a point at the point light and 1e-6f from it (sun lights: an ordinary slot)
    for lab, off in (("at light", 0.0), ("light eps", EPS32), ("light eps-ulp", _down(EPS32)),
                     ("light eps+ulp", _up(EPS32))):
        add(lab, pc, (0.3, 0.4, 1.0), pc + np.array([-0.5, 0.6, 1.0]), d0=(off, 0.0, 0.0) if lt else (0.2, 0.3, 1.0),
            loc0=pc + np.array([off, 0.0, 0.0]))
    # light and camera 1e4 away from the origin, close to the point (cancellation in loc - p and cam - p)
    pf = _f32([1.0e4, -2.0e4, 5.0e3])
    for k in range(2):
        add("far", pf, (0.3, -0.2, 1.0), _f32(pf + np.array([-0.4, 0.1, 0.9 + 0.1 * k])),
            d0=(0.3, -0.2, 1.0), loc0=_f32(pf + np.array([0.3, -0.25, 0.5 + 0.1 * k])))
    # zero light colours
    add("zero colours", p0, (0.1, 0.2, 1.0), p0 + np.array([0.2, 0.1, 1.0]), d0=(0.1, 0.1, 1.0), cd=0.0, cs=0.0)
    s = {k: _f32(np.stack([np.asarray(r[k], np.float64) for r in rows])) for k in ("p", "n", "alb", "cam", "lights", "gc")}
    s["amb"] = _f32(0.2 * rng.random((len(rows), 3)))
    s.update(light_type=lt, shin=shin)
    return s, labels


def ordinary_slots(M, kind, L, shin, seed=0):
    """M slots of a unit sphere seen from outside with lights around it, un-normalised normals"""
    rng = np.random.default_rng(seed)
    lt = 1 if kind == "point" else 0
    p = rng.normal(size=(M, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    n = p * rng.uniform(0.5, 2.0, (M, 1)) + 0.2 * rng.normal(size=(M, 3))
    cam = rng.normal(size=(M, 3))
    cam = 2.0 * cam / np.linalg.norm(cam, axis=1, keepdims=True)
    vec = rng.normal(size=(M, L, 3)) * (1.0 if lt == 0 else 2.0)
    lights = np.concatenate([vec, 0.6 * rng.random((M, L, 3)), 0.5 * rng.random((M, L, 3))], 2)
    s = dict(p=_f32(p), n=_f32(n), alb=_f32(rng.random((M, 3))), cam=_f32(cam), lights=_f32(lights),
             amb=_f32(0.2 * rng.random((M, 3))), gc=_f32(rng.normal(size=(M, 3))))
    s.update(light_type=lt, shin=shin)
    return s
