"""Host mirror of the reference's ``bn128`` package for the prove path
(bn128/g1.go, bn128/g2.go): same method names and argument meaning, bodies are
calls into libb200snark (CUDA).  Points are Jacobian tuples of Python ints —
G1: (X, Y, Z); G2: ((X0, X1), (Y0, Y1), (Z0, Z1)) — like ``[3]*big.Int`` and
``[3][2]*big.Int``.

Extra (not in the reference, which has no MSM routine): ``BaseSet`` — a
device-resident CRS array — and ``G1.MSM`` / ``G2.MSM``.
"""
import numpy as np

from . import _lib
from ._lib import check, ints_to_limbs, lib, limbs_to_ints, ptr

# bn128/bn128.go:40-83
Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def _flatten_g1(points):
    flat = []
    for p in points:
        flat.extend((p[0], p[1], p[2]))
    return ints_to_limbs(flat)


def _flatten_g2(points):
    flat = []
    for p in points:
        flat.extend((p[0][0], p[0][1], p[1][0], p[1][1], p[2][0], p[2][1]))
    return ints_to_limbs(flat)


def _unflatten_g1(arr):
    v = limbs_to_ints(arr)
    return [tuple(v[i:i + 3]) for i in range(0, len(v), 3)]


def _unflatten_g2(arr):
    v = limbs_to_ints(arr)
    return [((v[i], v[i + 1]), (v[i + 2], v[i + 3]), (v[i + 4], v[i + 5])) for i in range(0, len(v), 6)]


def reduce_scalar(e):
    """The m in [0, r) with the reference's MulScalar(P, e) == m * P as group elements, for every P of order r.

    MulScalar consumes |e| (Fq.Copy goes through Bytes(), fields/fq.go:138-140) and runs its MSB-first double-and-add
    over every bit of it (bn128/g1.go:140-155, g2.go:142-181) with an Add that has no doubling branch (SURVEY H6).
    Below r the accumulator never meets P, so m = |e|.  For |e| >= r it can: when the doubled prefix is P itself and the
    next bit is set, Add(P, P) returns infinity and the walk restarts from there.  So m is |e| mod r only when no
    prefix hits that case; e = r + 2 gives m = 0, not 2.  The C ABI takes m and refuses scalars >= r (B200_ERANGE)."""
    e = abs(int(e))
    if e < R:
        return e
    m = 0
    for i in range(e.bit_length() - 1, -1, -1):
        d = 2 * m % R
        m = (0 if d == 1 else (d + 1) % R) if (e >> i) & 1 else d   # d == 1 and the bit set: Add(P, P) -> infinity
    return m


class BaseSet:
    """A CRS array (e.g. Pk.G1.At) uploaded once: normalised to affine Montgomery
    form and window-precomputed on the device (b200_g*_bases_load)."""

    def __init__(self, group, points=None, limbs=None, window_bits=0, acc_mode=0, table_windows=0):
        """acc_mode: 0 auto, 1 batched-affine, 2 XYZZ bucket accumulation (b200_config; same result).
        table_windows: stored window rows t (B200_CFG_TABLE_WINDOWS; 0 = all, same result, t < all: less memory)."""
        assert group in (1, 2)
        self.group = group
        if limbs is None:
            limbs = _flatten_g1(points) if group == 1 else _flatten_g2(points)
        words = 12 if group == 1 else 24
        limbs = np.ascontiguousarray(limbs, dtype=np.uint64).reshape(-1)
        assert limbs.size % words == 0
        self.n = limbs.size // words
        h = _lib._h(0)
        fn = lib().b200_g1_bases_load if group == 1 else lib().b200_g2_bases_load
        check(lib().b200_config(_lib.CFG_ACC_MODE, acc_mode))
        try:
            with _lib.table_windows(table_windows):
                check(fn(ptr(limbs), self.n, window_bits, h))
        finally:
            check(lib().b200_config(_lib.CFG_ACC_MODE, _lib.ACC_AUTO))
        self.handle = h.value

    def table_windows(self):
        t = _lib._int(0)
        check(lib().b200_bases_table_windows(self.handle, t))
        return t.value

    def device_bytes(self):
        v = _lib._sz(0)
        check(lib().b200_bases_device_bytes(self.handle, v))
        return v.value

    def acc_mode(self):
        m = _lib._int(0)
        check(lib().b200_bases_acc_mode(self.handle, m))
        return m.value

    def info(self):
        n, g, c, nw = _lib._sz(0), _lib._int(0), _lib._int(0), _lib._int(0)
        check(lib().b200_bases_info(self.handle, n, g, c, nw))
        return {"n": n.value, "group": g.value, "window_bits": c.value, "n_windows": nw.value}

    def msm(self, scalars=None, limbs=None):
        """sum_i scalars[i] * P_i  ->  Jacobian (x, y, 1) (infinity: all zero)."""
        if limbs is None:
            limbs = ints_to_limbs([reduce_scalar(s) for s in scalars])
        limbs = np.ascontiguousarray(limbs, dtype=np.uint64).reshape(-1, 4)
        n = limbs.shape[0]
        out = np.zeros(12 if self.group == 1 else 24, dtype=np.uint64)
        fn = lib().b200_g1_msm if self.group == 1 else lib().b200_g2_msm
        check(fn(self.handle, ptr(limbs), n, ptr(out)))
        return _unflatten_g1(out)[0] if self.group == 1 else _unflatten_g2(out)[0]

    def msm_device_batch(self, d_scalars, n, k, d_out, stride=None, mont=0, stream=None):
        """k MSMs over the first n bases in one set of launches (b200_msm_device_batch): record p of ``d_out`` (k XYZZ
        records of 16 / 32 u64 words, device memory) is sum_i scalar[p*stride + i] * P_i.  ``d_scalars`` / ``d_out`` are
        device pointers or objects with ``data_ptr()`` (torch tensors); ``stream`` a cudaStream_t or an object with
        ``cuda_stream``; ``stride`` defaults to n.  No host synchronisation."""
        def _p(x):
            return None if x is None else (x.data_ptr() if hasattr(x, "data_ptr") else int(x))
        st = getattr(stream, "cuda_stream", stream)
        check(lib().b200_msm_device_batch(self.handle, _p(d_scalars), n, k, n if stride is None else stride, mont,
                                          _p(d_out), st))

    def free(self):
        if self.handle:
            check(lib().b200_bases_free(self.handle))
            self.handle = 0


class _Group:
    _group = 0

    def MulScalarBatch(self, points, scalars):
        """[MulScalar(p_i, e_i)] with the reference's own double-and-add and
        formulas (X,Y,Z-exact; bn128/g1.go:140-155, g2.go:142-181)."""
        n = len(scalars)
        s = ints_to_limbs([reduce_scalar(e) for e in scalars])
        words = 12 if self._group == 1 else 24
        out = np.zeros(n * words, dtype=np.uint64)
        flat = _flatten_g1 if self._group == 1 else _flatten_g2
        if len(points) == 1 and n != 1:
            fn = lib().b200_g1_mul_batch_bcast if self._group == 1 else lib().b200_g2_mul_batch_bcast
        else:
            assert len(points) == n
            fn = lib().b200_g1_mul_batch if self._group == 1 else lib().b200_g2_mul_batch
        p = flat(points)
        check(fn(ptr(p), ptr(s), n, ptr(out)))
        return _unflatten_g1(out) if self._group == 1 else _unflatten_g2(out)

    def MulScalar(self, p, e):
        """bn128.G1.MulScalar / bn128.G2.MulScalar.  NOTE: the reference consumes
        all bits of |e|; this mirror first maps e with reduce_scalar (the same
        group element for every e; identical X,Y,Z whenever |e| < r)."""
        return self.MulScalarBatch([p], [e])[0]

    # element-wise group law with the reference's formulas (X,Y,Z-exact): g1.go:32-170 / g2.go:32-200
    def _op(self, name, pts, qts=None, out_fe=3):
        n = len(pts)
        flat = _flatten_g1 if self._group == 1 else _flatten_g2
        words = (4 if self._group == 1 else 8) * out_fe
        out = np.zeros(n * words, dtype=np.uint64)
        fn = getattr(lib(), f"b200_g{self._group}_{name}_batch")
        if qts is None:
            check(fn(ptr(flat(pts)), n, ptr(out)))
        else:
            check(fn(ptr(flat(pts)), ptr(flat(qts)), n, ptr(out)))
        return out

    def Add(self, p1, p2):
        return (_unflatten_g1 if self._group == 1 else _unflatten_g2)(self._op("add", [p1], [p2]))[0]

    def Double(self, p):
        return (_unflatten_g1 if self._group == 1 else _unflatten_g2)(self._op("double", [p]))[0]

    def Neg(self, p):
        return (_unflatten_g1 if self._group == 1 else _unflatten_g2)(self._op("neg", [p]))[0]

    def Sub(self, a, b):                      # g1.go:98-100
        return self.Add(a, self.Neg(b))

    def IsZero(self, p):                      # g1.go:28-30
        z = p[2]
        return z == 0 if self._group == 1 else (z[0] == 0 and z[1] == 0)

    def Affine(self, p):
        """G1.Affine -> (x, y), infinity (0, 0) (g1.go:157-170); G2.Affine -> (x, y, one), infinity
        ((0,0),(1,0),(0,0)) (g2.go:183-200)."""
        v = limbs_to_ints(self._op("affine", [p], out_fe=2))
        if self._group == 1:
            return (v[0], v[1])
        if self.IsZero(p):
            return ((0, 0), (1, 0), (0, 0))
        return ((v[0], v[1]), (v[2], v[3]), (1, 0))

    def Equal(self, p1, p2):                  # g1.go:172-193: same point <=> same affine coordinates
        if self.IsZero(p1) or self.IsZero(p2):
            return self.IsZero(p1) and self.IsZero(p2)
        return self.Affine(p1) == self.Affine(p2)

    def MSM(self, points, scalars, window_bits=0):
        bs = BaseSet(self._group, points, window_bits=window_bits)
        try:
            return bs.msm(scalars)
        finally:
            bs.free()


class G1(_Group):
    _group = 1
    G = (1, 2, 1)                                   # bn128/bn128.go:52-55


class G2(_Group):
    _group = 2
    G = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
          11559732032986387107991004021392285783925812861821192530917403151452391805634),
         (8495653923123431417604973247489272438418190587263600148770280649306958101930,
          4082367875863433681332203403145435568316851327593401208105741076214120093531),
         (1, 0))                                    # bn128/bn128.go:57-83


class Bn128:
    """bn128.Bn128 (bn128/bn128.go:11-36): the pairing entry point."""
    G1 = G1()
    G2 = G2()

    def PairingBatch(self, p1s, p2s):
        n = len(p1s)
        a, b = _flatten_g1(p1s), _flatten_g2(p2s)
        out = np.zeros(n * 48, dtype=np.uint64)
        check(lib().b200_pairing_batch(ptr(a), ptr(b), n, ptr(out)))
        v = limbs_to_ints(out)
        return [tuple(tuple((v[12 * i + 6 * h + 2 * k], v[12 * i + 6 * h + 2 * k + 1]) for k in range(3)) for h in range(2))
                for i in range(n)]

    @staticmethod
    def _flatten_fq12(vals):
        return ints_to_limbs([c for v in vals for h in v for f2 in h for c in f2])

    def Fq12MulBatch(self, xs, ys):         # fields/fq12.go:72-84, element-wise over two lists
        n = len(xs)
        out = np.zeros(n * 48, dtype=np.uint64)
        check(lib().b200_fq12_mul_batch(ptr(self._flatten_fq12(xs)), ptr(self._flatten_fq12(ys)), n, ptr(out)))
        v = limbs_to_ints(out)
        return [tuple(tuple((v[12 * i + 6 * h + 2 * k], v[12 * i + 6 * h + 2 * k + 1]) for k in range(3)) for h in range(2))
                for i in range(n)]

    def Fq12Mul(self, x, y):
        return self.Fq12MulBatch([x], [y])[0]

    def Pairing(self, p1, p2):              # bn128.go:179-186 -> [2][3][2] tuple of ints
        return self.PairingBatch([p1], [p2])[0]
