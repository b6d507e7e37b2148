"""NumPy restatement of what b2v_ws_flood computes (TEST INFRASTRUCTURE): the exact minimax cost
field of the chosen algorithm, then labels along cost-optimal edges — fewer hops first, then the
smaller label — and the label SET of every voxel (which labels can reach it along cost-optimal
edges: two different ones = the reference's answer there depends on its queue order).
6-connected. mode 0 = scipy.ndimage.watershed_ift's cost (max |dI| over the path's edges) with
SciPy's flat-array neighbourhood; mode 1 = skimage's (max I over the path), proper bounds.

Written for clarity (whole-array Jacobi sweeps), staged like the C ABI so that the Z-shard
protocol tests can drive it: planes outside [fz0, fz1) are frozen (only plane merges change them).
"""
import numpy as np

INF_C = np.uint32(0xFFFFFFFF)
INF_K = np.uint64(0xFFFFFFFFFFFFFFFF)
HOP = np.uint64(1 << 32)
EMPTY, MULTI = 32768, 0x10000      # label sets as the engines store them (uint32): label + 32768, or these


def _shifted(a, off, fill, mode, shape):
    """b[p] = a[p - off] where the predecessor p - off is a neighbour of p, else `fill`.
    off = (dz, dy, dx) with one non-zero entry."""
    nz, ny, nx = shape
    if mode == 0:                       # flat-array neighbourhood
        f = a.reshape(-1)
        o = (off[0] * ny + off[1]) * nx + off[2]
        b = np.full(f.shape, fill, f.dtype)
        if o > 0:
            b[o:] = f[:-o]
        else:
            b[:o] = f[-o:]
        return b.reshape(shape)
    b = np.full(shape, fill, a.dtype)
    src = [slice(None)] * 3
    dst = [slice(None)] * 3
    ax = [i for i in range(3) if off[i]][0]
    if off[ax] > 0:
        dst[ax] = slice(1, None); src[ax] = slice(0, -1)
    else:
        dst[ax] = slice(0, -1); src[ax] = slice(1, None)
    b[tuple(dst)] = a[tuple(src)]
    return b


OFFS = [(0, 0, 1), (0, 0, -1), (0, 1, 0), (0, -1, 0), (1, 0, 0), (-1, 0, 0)]


class Model:
    def __init__(self, img_u16, markers, mode, frozen_lo=False, frozen_hi=False):
        self.I = np.ascontiguousarray(img_u16).astype(np.int64)
        self.shape = self.I.shape
        self.mode = mode
        m = np.ascontiguousarray(markers).astype(np.int64)
        self.marker = m != 0
        self.C = np.where(self.marker, 0 if mode == 0 else self.I, int(INF_C)).astype(np.uint32)
        self.K = np.where(self.marker, (m + 32768).astype(np.uint64), INF_K).astype(np.uint64)
        self.S = np.where(self.marker, m + 32768, EMPTY).astype(np.int64)
        self.free = np.ones(self.shape, bool)
        if frozen_lo:
            self.free[0] = False
        if frozen_hi:
            self.free[-1] = False
        self.adm = None

    def _via(self, off):
        """cost of reaching p through its neighbour p - off (INF where there is none)."""
        Cv = _shifted(self.C, off, INF_C, self.mode, self.shape)
        if self.mode == 0:
            Iv = _shifted(self.I, off, 0, self.mode, self.shape)
            w = np.abs(self.I - Iv).astype(np.uint32)
        else:
            w = self.I.astype(np.uint32)
        return np.where(Cv == INF_C, INF_C, np.maximum(Cv, w))

    def converge_cost(self):
        while True:
            best = self.C.copy()
            for off in OFFS:
                best = np.minimum(best, self._via(off))
            best = np.where(self.free, best, self.C)
            if np.array_equal(best, self.C):
                return
            self.C = best

    def label_begin(self):
        adm = []
        if self.mode == 0:
            for off in OFFS:
                via = self._via(off)
                adm.append((via != INF_C) & (via == self.C))
        else:
            cvs = [_shifted(self.C, off, INF_C, self.mode, self.shape) for off in OFFS]
            cmin = np.minimum.reduce(cvs)
            for cv in cvs:
                adm.append((cv != INF_C) & (cv == cmin))
        ok = self.free & ~self.marker & (self.C != INF_C)
        self.adm = [a & ok for a in adm]

    def converge_labels(self):
        while True:
            K, S = self.K.copy(), self.S.copy()
            for off, a in zip(OFFS, self.adm):
                Kv = _shifted(self.K, off, INF_K, self.mode, self.shape)
                Sv = _shifted(self.S, off, EMPTY, self.mode, self.shape)
                use = a & (Kv != INF_K)
                K = np.where(use & (Kv + HOP < K), Kv + HOP, K)
                j = use & (Sv != EMPTY)
                joined = np.where(S == EMPTY, Sv, np.where((S == Sv) & (Sv != MULTI), S, MULTI))
                S = np.where(j, joined, S)
            if np.array_equal(K, self.K) and np.array_equal(S, self.S):
                return
            self.K, self.S = K, S

    # ---- frozen planes
    def get_plane(self, what, z):
        if what == 0:
            return self.C[z].copy()
        return self.K[z].copy(), self.S[z].copy()

    def merge_plane(self, what, z, plane):
        if what == 0:
            new = np.minimum(self.C[z], plane)
            ch = not np.array_equal(new, self.C[z])
            self.C[z] = new
            return ch
        k, s = plane
        newk = np.minimum(self.K[z], k)
        S = self.S[z]
        joined = np.where(S == EMPTY, s, np.where((S == s) & (s != MULTI), S, MULTI))
        news = np.where(s != EMPTY, joined, S)
        ch = not (np.array_equal(newk, self.K[z]) and np.array_equal(news, S))
        self.K[z], self.S[z] = newk, news
        return ch

    def labels(self):
        lab = np.where(self.K == INF_K, 0, (self.K & np.uint64(0xFFFFFFFF)).astype(np.int64) - 32768).astype(np.int16)
        return lab, (self.S == MULTI).astype(np.uint8)


def flood(img_u16, markers, mode):
    m = Model(img_u16, markers, mode)
    m.converge_cost()
    m.label_begin()
    m.converge_labels()
    return m.labels()
