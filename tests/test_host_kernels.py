"""CPU: the per-thread bucket kernels of csrc/bucket_affine.cuh — the product backward kernel and the experiment
variants (_lr: short live ranges, _sp: three-deep staged fetches, prefetch) — run one emulated thread at a time over all
rounds of a small slice forest (csrc/host_kernel_test.cpp over csrc/host_stub), against the oracle's group sums.
Covers the kernels' index logic: pair <-> slice <-> entry mapping, signs, infinity operands, doublings, cancellations,
ragged and empty slices, several CTAs, and that the x-only forward denominators equal the full ones."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import ref_py as o

R_ = o.R


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_kernels())


def _u32(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint32).copy()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _scenario(group, R, nslices, seed):
    G = o.BN.G1 if group == 1 else o.BN.G2
    rng = random.Random(seed)
    npts = 40
    pts = [G.affine(G.mul_scalar(G.G, rng.randrange(1, R_)))[:2] for _ in range(npts - 2)]
    zero = (0, 0) if group == 1 else ((0, 0), (0, 0))
    pts += [zero, pts[3]]                                   # an infinity point and a repeated point in the table
    S = 1 << R
    slices = [[], [(0, 0)], [(0, 0), (0, 0)], [(1, 0), (1, 1)], [(2, 0)] * 4, [(npts - 2, 0), (5, 1)], [(5, 0), (npts - 2, 1)],
              [(3, 0), (npts - 1, 0)], [(3, 0), (npts - 1, 1), (7, 0)], [(i % npts, i & 1) for i in range(S)],
              [(4, 0), (4, 0), (4, 1), (4, 1)], [(npts - 2, 0), (npts - 2, 1)]]
    slices = [s[:S] for s in slices]
    while len(slices) < nslices:
        cnt = min(S, rng.choice([0, 1, 2, 3, S - 1, S, rng.randrange(S + 1)]))
        slices.append([(rng.randrange(npts), rng.randrange(2)) for _ in range(cnt)])
    rng.shuffle(slices)
    entries, starts, ends = [], [], []
    for s in slices:
        starts.append(len(entries))
        entries += [(i << 1) | sg for i, sg in s]
        ends.append(len(entries))
    entries += [0] * 4
    exp = []
    for s in slices:
        acc = G.zero3()
        one = 1 if group == 1 else (1, 0)
        for i, sg in s:
            if pts[i] == zero:
                continue
            p = (pts[i][0], pts[i][1], one)
            acc = G.add_or_double(acc, G.neg(p) if sg else p) if hasattr(G, "add_or_double") else _add(G, acc, G.neg(p) if sg else p)
        exp.append(zero if G.is_zero(acc) else G.affine(acc)[:2])
    flat = []
    for p in pts:
        for c in p:
            flat.extend(c if isinstance(c, tuple) else (c,))
    return _u32(flat), npts, np.array(entries, dtype=np.uint32), np.array(starts, dtype=np.uint32), np.array(ends, dtype=np.uint32), exp


def _add(G, a, b):
    """Group addition that also doubles (the reference's Add returns infinity for P + P, SURVEY H6)."""
    if G.is_zero(a):
        return b
    if G.is_zero(b):
        return a
    if G.affine(a)[:2] == G.affine(b)[:2]:
        return G.double(a)
    return G.add(a, b)


def _run(lib, group, variant, T, R, nslices, seed, fwd=-1):
    table, npts, entries, starts, ends, exp = _scenario(group, R, nslices, seed)
    w = 8 if group == 1 else 16
    out = np.zeros(nslices * 2 * w, dtype=np.uint32)
    rc = lib.t_affine_rounds(group, variant, fwd, T, _ptr(table), npts, _ptr(entries), _ptr(starts), _ptr(ends), nslices, R, _ptr(out))
    assert rc == 0
    raw = out.tobytes()
    vals = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    got = []
    for s in range(nslices):
        v = vals[s * (2 * w // 8):(s + 1) * (2 * w // 8)]
        got.append((v[0], v[1]) if group == 1 else ((v[0], v[1]), (v[2], v[3])))
    assert got == exp


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("T,R,nslices", [(8, 4, 300), (8, 3, 37), (32, 5, 520)])
def test_g1_backward_kernels(lib, variant, T, R, nslices):
    """variant 0: k_affine_backward (register loads); 1: k_affine_backward_staged — warp-leader TMA bulk copies +
    per-warp mbarrier in rounds >= 2, per-thread cp.async gathers from the forward pass's pair ids in round 1 (the copies
    are synchronous in the emulation, the mbarrier a warp barrier): index logic, phase parity, tail blocks, signs."""
    _run(lib, 1, variant, T, R, nslices, seed=100 * T + R)


@pytest.mark.parametrize("variant", [0, 1])
def test_g2_backward_kernels(lib, variant):
    _run(lib, 2, variant, 8, 3, 70, seed=9)


@pytest.mark.parametrize("T,R,nslices", [(8, 4, 300), (32, 5, 520)])
def test_g1_forward_kernel_cta_emulation(lib, T, R, nslices):
    """The forward KERNEL (x-only denominators, per-thread prefix products, warp-shuffle + shared-memory block scan)
    runs CTA by CTA with one OS thread per CUDA thread; its pre / others / btot equal the host restatement in every
    round, and the proof-of-the-pudding sums come out right."""
    _run(lib, 1, 0, T, R, nslices, seed=7 * T + R, fwd=0)


def test_g2_forward_kernel_cta_emulation(lib):
    _run(lib, 2, 0, 8, 3, 70, seed=11, fwd=0)


@pytest.mark.parametrize("group,nbuckets,seg", [(1, 300, 4), (1, 37, 1), (1, 700, 4), (2, 90, 4),
                                                # seg = 0: rows / columns + bit planes + Horner tail, nbuckets = 2^(c-1)
                                                (1, 64, 0), (1, 128, 0), (1, 2048, 0), (2, 256, 0)])
def test_msm_tail_kernels(lib, group, nbuckets, seg):
    """k_merge_slices_affine (thread-per-bucket path and the warp path for buckets with > 24 slices, ballot + shuffles),
    then the engine's tails (msm_host.cuh): launch_segment_tail — k_bucket_reduce (running sums + small scalar multiple per
    segment), launch_tree_sum (one and two levels) — or launch_bucket_tail, and k_finalize: sum_b b * (sum of the slices
    of bucket b) against the oracle."""
    G = o.BN.G1 if group == 1 else o.BN.G2
    rng = random.Random(50 + nbuckets)
    zero = (0, 0) if group == 1 else ((0, 0), (0, 0))
    one = 1 if group == 1 else (1, 0)
    pool = [G.affine(G.mul_scalar(G.G, rng.randrange(1, R_)))[:2] for _ in range(24)] + [zero]
    slice_off = [0, 0]                                # slice_off[b] for b = 0 (unused) and 1
    pts = []
    acc = G.zero3()
    for b in range(1, nbuckets + 1):
        cnt = rng.choice([0, 1, 1, 2, 3, 12, 13, 24, 25, 40]) if b % 7 else rng.choice([0, 33])
        bsum = G.zero3()
        for _ in range(cnt):
            p = rng.choice(pool)
            pts.append(p)
            if p != zero:
                bsum = _add(G, bsum, (p[0], p[1], one))
        slice_off.append(slice_off[-1] + cnt)
        if not G.is_zero(bsum):
            acc = _add(G, acc, G.mul_scalar(bsum, b))
    flat = []
    for p in pts or [zero]:
        for c in p:
            flat.extend(c if isinstance(c, tuple) else (c,))
    w = 8 if group == 1 else 16
    out = np.zeros(3 * w, dtype=np.uint32)
    so = np.array(slice_off, dtype=np.uint32)
    assert lib.t_msm_tail(group, _ptr(_u32(flat)), _ptr(so), nbuckets, seg, _ptr(out)) == 0
    raw = out.tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    if G.is_zero(acc):
        assert all(x == 0 for x in v)
    else:
        e = G.affine(acc)
        got = (v[0], v[1], v[2]) if group == 1 else ((v[0], v[1]), (v[2], v[3]), (v[4], v[5]))
        assert got == ((e[0], e[1], 1) if group == 1 else (e[0], e[1], (1, 0)))


@pytest.mark.parametrize("group,n,c,S", [(1, 150, 5, 0), (1, 150, 5, 16), (1, 97, 4, 64), (1, 40, 9, 0), (2, 48, 4, 8),
                                         (1, 300, 8, 8), (2, 60, 7, 0),
                                         # ~17 slices per bucket: above the old thread-path bound of k_merge_slices_affine (12), inside the new one (24)
                                         (1, 100, 6, 8), (2, 110, 6, 8)])
def test_whole_msm_pipeline_on_the_cpu(lib, group, n, c, S):
    """The library's own MSM engine (msm_host.cuh: window precompute, signed-digit recode, counting sort, slice tables,
    bucket accumulation in both modes — the batched-affine rounds with the staged backward pass, the XYZZ kernel with the
    lanes per slice it picks —, slice merge, bucket tail) and k_finalize on the CPU emulation == sum_i s_i * P_i by the
    oracle.  Scalars include 0, 1, r - 1, small values and repeated points."""
    G = o.BN.G1 if group == 1 else o.BN.G2
    rng = random.Random(1000 * group + n + c)
    ks = [rng.randrange(1, R_) for _ in range(n)]
    ks[5] = ks[6]                                           # a repeated point
    pts = [G.mul_scalar(G.G, k) for k in ks]                # Jacobian, Z != 1: k_load_bases normalises
    pts[7] = G.zero3()                                      # an infinity point in the CRS (SURVEY a11)
    ks[7] = 0
    sc = [rng.randrange(R_) for _ in range(n)]
    sc[0], sc[1], sc[2], sc[3] = 0, 1, R_ - 1, (1 << 16) - 1
    for i in range(10, 20):
        sc[i] = rng.randrange(1 << 12)
    flat = []
    for p in pts:
        for cc in p:
            flat.extend(cc if isinstance(cc, tuple) else (cc,))
    w = 8 if group == 1 else 16
    out = np.zeros(3 * w, dtype=np.uint32)
    rc = lib.t_msm_full(group, _ptr(_u32(flat)), _ptr(_u32(sc)), n, c, S, _ptr(out))
    assert rc == 0
    raw = out.tobytes()
    v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(len(raw) // 32)]
    e = G.affine(G.mul_scalar(G.G, sum(k * s_ for k, s_ in zip(ks, sc)) % R_))
    got = (v[0], v[1], v[2]) if group == 1 else ((v[0], v[1]), (v[2], v[3]), (v[4], v[5]))
    assert got == ((e[0], e[1], 1) if group == 1 else (e[0], e[1], (1, 0)))


@pytest.mark.parametrize("la,lb", [(1, 1), (7, 13), (64, 64), (100, 29), (129, 128)])
def test_ntt_kernels_polynomial_product(lib, la, lb):
    """PolynomialField.Mul (r1csqap.go:57-67) through the NTT kernels on the CPU emulation (twiddles, DIF stages,
    pointwise product, DIT stages; no bit-reversal pass) == the oracle's schoolbook product."""
    rng = random.Random(la * 1000 + lb)
    a = [rng.randrange(R_) for _ in range(la)]
    b = [rng.randrange(R_) for _ in range(lb)]
    a[0], b[-1] = R_ - 1, 1
    out = np.zeros(8 * (la + lb - 1), dtype=np.uint32)
    assert lib.t_poly_mul_kernels(_ptr(_u32(a)), la, _ptr(_u32(b)), lb, _ptr(out)) == 0
    raw = out.tobytes()
    got = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(la + lb - 1)]
    assert got == o.PF.mul(a, b)


@pytest.mark.parametrize("logn,dit,max_k", [(10, 0, 8), (10, 1, 8), (11, 0, 8), (11, 1, 8), (13, 0, 8), (13, 1, 8),
                                            (14, 0, 2), (14, 1, 2), (14, 0, 3), (15, 1, 1),   # several strided passes
                                            (18, 1, 8)])                                       # a full 8-stage strided pass
def test_fused_ntt_passes_equal_the_stage_kernels(lib, logn, dit, max_k):
    """k_ntt_fused (several stages per pass in a 1024-element shared-memory tile: strided passes + the contiguous last
    pass) produces exactly the per-stage kernels' transform, forward and inverse; and the forward one is the DFT."""
    n = 1 << logn
    rng = random.Random(logn * 2 + dit)
    vals = [rng.randrange(R_) for _ in range(n)]
    a, b = np.zeros(8 * n, dtype=np.uint32), np.zeros(8 * n, dtype=np.uint32)
    # inputs are taken as Montgomery representatives by the kernels; any residues do for an equality test
    assert lib.t_ntt_compare(_ptr(_u32(vals)), logn, dit, max_k, _ptr(a), _ptr(b)) == 0
    assert a.tobytes() == b.tobytes()
    assert a.tobytes() != _u32(vals).tobytes()


def _limbs_to_ints(a, n):
    raw = a.tobytes()
    return [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(n)]


def _horner(c, x):
    acc = 0
    for v in reversed(c):
        acc = (acc * x + v) % R_
    return acc


@pytest.mark.parametrize("n", [1, 2, 3, 7, 21, 33, 64, 100, 1024, 1500, 3000])
def test_interpolation_orchestration_on_the_cpu(lib, n):
    """The library's own host code for LagrangeInterpolation over {1..n} (r1csqap.go:150-158) at any n — QapDomain
    (factorial inverses, subproduct tree: schoolbook levels, batched sub-transforms on shared-memory tiles and fused
    strided passes above 2^10), Newton coefficients by one cyclic product, Newton -> monomial divide and conquer
    (qap_sparse.cuh) — on the emulated kernels == the oracle's coefficients / the interpolation conditions."""
    rng = random.Random(n)
    v = [rng.randrange(R_) for _ in range(n)]
    if n > 2:
        v[1], v[2] = 0, 5
    out = np.zeros(8 * n, dtype=np.uint32)
    assert lib.t_qap_interpolate(_ptr(_u32(v)), n, _ptr(out)) == 0
    c = _limbs_to_ints(out, n)
    if n <= 21:
        assert c == o.PF.lagrange_interpolation(v)
    for j in (range(n) if n <= 100 else rng.sample(range(n), 60)):
        assert _horner(c, j + 1) == v[j], (n, j)


@pytest.mark.parametrize("n", [1, 6, 20, 127, 128, 1100])
def test_zero_poly_orchestration_on_the_cpu(lib, n):
    """prod_{i=1..n}(x - i) (groth16.go:122-132) as the Newton basis element n through the subproduct tree."""
    out = np.zeros(8 * (n + 1), dtype=np.uint32)
    assert lib.t_qap_zero_poly(n, _ptr(out)) == 0
    z = _limbs_to_ints(out, n + 1)
    if n <= 20:
        exp = [1]
        for i in range(1, n + 1):
            exp = o.PF.mul(exp, [(-i) % R_, 1])
        assert z == exp
    else:
        assert z[n] == 1 and all(_horner(z, x) == 0 for x in random.Random(n).sample(range(1, n + 1), 30))
        t = 0x1234567
        e = 1
        for i in range(1, n + 1):
            e = e * (t - i) % R_
        assert _horner(z, t) == e


@pytest.mark.parametrize("n", [2, 3, 7, 16, 21, 40, 100, 1024, 1500])
def test_quotient_h_directly_from_the_values(lib, n):
    """h = DivisorPolynomial(px, Z) (r1csqap.go:213-216; groth16.go:266) without forming px: a, b, c are shifted from
    {1..n} to n+1..2n-1 in Newton form, h is formed there pointwise and interpolated once over the offset tree
    (qap_sparse.cuh: QapHDomain).  Equal to the oracle's exact quotient for small n; checked through the identity
    h(x) Z(x) = a(x) b(x) - c(x) at random points for the larger ones."""
    rng = random.Random(5000 + n)
    a = [rng.randrange(R_) for _ in range(n)]
    b = [rng.randrange(R_) for _ in range(n)]
    if n > 3:
        a[1], b[2] = 0, 1
    c = [x * y % R_ for x, y in zip(a, b)]              # a satisfied R1CS: (a b - c) vanishes on 1..n
    out = np.zeros(8 * max(n - 1, 1), dtype=np.uint32)
    assert lib.t_qap_h_direct(_ptr(_u32(a + b + c)), n, _ptr(out)) == 0
    h = _limbs_to_ints(out, n - 1)

    def interp(v):
        o_ = np.zeros(8 * n, dtype=np.uint32)
        assert lib.t_qap_interpolate(_ptr(_u32(v)), n, _ptr(o_)) == 0
        return _limbs_to_ints(o_, n)
    if n <= 40:
        ax, bx, cx = (o.PF.lagrange_interpolation(v) for v in (a, b, c))
        px = o.PF.sub(o.PF.mul(ax, bx), cx)
        z = [1]
        for i in range(1, n + 1):
            z = o.PF.mul(z, [(-i) % R_, 1])
        assert h == o.PF.divisor_polynomial(px, z)
    else:
        ax, bx, cx = interp(a), interp(b), interp(c)
        for _ in range(6):
            t = rng.randrange(R_)
            zt = 1
            for i in range(1, n + 1):
                zt = zt * (t - i) % R_
            assert _horner(h, t) * zt % R_ == (_horner(ax, t) * _horner(bx, t) - _horner(cx, t)) % R_


def _lagrange_at(n, t):
    """[l_j(t)], the Lagrange basis of {1..n} at t (t not in 1..n), from factorials and one batch inversion."""
    fact = [1] * n
    for i in range(1, n):
        fact[i] = fact[i - 1] * i % R_
    den = [(t - j - 1) * fact[j] % R_ * fact[n - 1 - j] % R_ for j in range(n)]
    pre, zt = [1] * (n + 1), 1
    for j in range(n):
        pre[j + 1] = pre[j] * den[j] % R_
        zt = zt * (t - j - 1) % R_
    inv, out = pow(pre[n], -1, R_), [0] * n
    for j in range(n - 1, -1, -1):
        v = zt * inv % R_ * pre[j] % R_
        out[j] = (R_ - v) % R_ if (n - 1 - j) & 1 else v
        inv = inv * den[j] % R_
    return out


@pytest.mark.parametrize("how", ["first", "last", "middle", "every", "c=0"])
@pytest.mark.parametrize("n", [2, 3, 7, 16, 21, 40, 100, 1024, 1500])
def test_quotient_h_directly_drops_the_remainder(lib, n, how):
    """Values of an UNSATISFIED R1CS (c_j != a_j b_j on one row — the first, the last or n/2 — on every row, or c = 0):
    groth16.GenerateProofs takes h = DivisorPolynomial(px, Z), the quotient with the remainder dropped
    (r1csqap.go:213-216), and so must the direct path.  Equal to the oracle's quotient for n <= 40; above, checked through
    h(t) Z(t) = a(t) b(t) - c(t) - rem(t) at random t, where rem = px mod Z is the interpolant of the row residuals
    a_j b_j - c_j (all from an independent Lagrange basis at t)."""
    rng = random.Random(7000 + n)
    a = [rng.randrange(R_) for _ in range(n)]
    b = [rng.randrange(R_) for _ in range(n)]
    c = [x * y % R_ for x, y in zip(a, b)]
    if how == "every":
        c = [rng.randrange(R_) for _ in range(n)]
    elif how == "c=0":
        c = [0] * n
    else:
        j = {"first": 0, "last": n - 1, "middle": n // 2}[how]
        c[j] = (c[j] + 1) % R_
    out = np.zeros(8 * max(n - 1, 1), dtype=np.uint32)
    assert lib.t_qap_h_direct(_ptr(_u32(a + b + c)), n, _ptr(out)) == 0
    h = _limbs_to_ints(out, n - 1)
    if n <= 40:
        ax, bx, cx = (o.PF.lagrange_interpolation(v) for v in (a, b, c))
        z = [1]
        for i in range(1, n + 1):
            z = o.PF.mul(z, [(-i) % R_, 1])
        assert h == o.PF.divisor_polynomial(o.PF.sub(o.PF.mul(ax, bx), cx), z)
    for _ in range(3 if n <= 40 else 5):
        t = rng.randrange(n + 1, R_)
        lag = _lagrange_at(n, t)
        at_, bt_, ct_ = (sum(v * l for v, l in zip(vs, lag)) % R_ for vs in (a, b, c))
        rem = sum((x * y - z_) * l for x, y, z_, l in zip(a, b, c, lag)) % R_
        zt = 1
        for i in range(1, n + 1):
            zt = zt * (t - i) % R_
        assert _horner(h, t) * zt % R_ == (at_ * bt_ - ct_ - rem) % R_, t


@pytest.mark.parametrize("na,nb", [(13, 7), (200, 101), (1023, 513), (2600, 1300)])
def test_division_orchestration_on_the_cpu(lib, na, nb):
    """poly_div_device (poly_host.cuh: Newton inverse series of the reversed divisor, cached transform, fused transform
    passes at >= 2^10 points) on the emulated kernels == PolynomialField.Div (r1csqap.go:70-84)."""
    rng = random.Random(na)
    b = [rng.randrange(R_) for _ in range(nb)]
    b[-1] = rng.randrange(1, R_)
    q0 = [rng.randrange(R_) for _ in range(na - nb + 1)]
    r0 = [rng.randrange(R_) for _ in range(nb - 1)]
    a = o.PF.add(o.PF.mul(q0, b), r0) if na <= 300 else None
    if a is None:                                  # larger: build a = q0*b + r0 with the emulated product kernels
        prod = np.zeros(8 * na, dtype=np.uint32)
        assert lib.t_poly_mul_kernels(_ptr(_u32(q0)), len(q0), _ptr(_u32(b)), nb, _ptr(prod)) == 0
        a = _limbs_to_ints(prod, na)
        a = [(x + (r0[i] if i < nb - 1 else 0)) % R_ for i, x in enumerate(a)]
    q = np.zeros(8 * (na - nb + 1), dtype=np.uint32)
    rem = np.zeros(8 * max(nb - 1, 1), dtype=np.uint32)
    assert lib.t_poly_div_orch(_ptr(_u32(a)), na, _ptr(_u32(b)), nb, _ptr(q), _ptr(rem)) == 0
    assert _limbs_to_ints(q, na - nb + 1) == q0
    assert _limbs_to_ints(rem, nb - 1) == r0


def test_warp_pairing_on_the_cpu(lib):
    """csrc/pairing_warp.cuh — one warp per pairing: F_q^12 in shared memory, the 27 F_q^2 products of a tower
    multiplication on 27 lanes, the line functions level by level — run as 32 emulated lanes: the tower operations
    (product, aliased square, Frobenius 1-3, x^u, conjugation, inversion) and a whole pairing agree coefficient for
    coefficient with the thread-per-pairing restatement of pairing.cuh, and e(25 G1, 30 G2) carries the literal of
    bn128_test.go:66."""
    rng = random.Random(77)
    for _ in range(3):
        a = _u32([rng.randrange(o.Q) for _ in range(12)])
        b = _u32([rng.randrange(o.Q) for _ in range(12)])
        o1, o2, o3 = (np.zeros(96, dtype=np.uint32) for _ in range(3))
        assert lib.t_f12_warp_ops(_ptr(a), _ptr(b), _ptr(o1), _ptr(o2), _ptr(o3)) == 0
    G1, G2 = o.BN.G1, o.BN.G2
    for k1, k2 in ((25, 30), (rng.randrange(1, R_), rng.randrange(1, R_))):
        p = G1.affine(G1.mul_scalar(G1.G, k1))
        q = G2.affine(G2.mul_scalar(G2.G, k2))
        out = np.zeros(96, dtype=np.uint32)
        assert lib.t_pairing_warp(_ptr(_u32([p[0], p[1]])), _ptr(_u32([q[0][0], q[0][1], q[1][0], q[1][1]])), _ptr(out)) == 0
        raw = out.tobytes()
        v = [int.from_bytes(raw[32 * i:32 * (i + 1)], "little") for i in range(12)]
        got = tuple(tuple((v[6 * h + 2 * k], v[6 * h + 2 * k + 1]) for k in range(3)) for h in range(2))
        assert got == o.BN.pairing((p[0], p[1], 1), (q[0], q[1], (1, 0)))
        if (k1, k2) == (25, 30):
            assert v[0] == 8016119724813186033542830391460394070015218389456422587891475873290878009957


def test_glv_half_warp_multiplication_on_the_cpu(lib):
    """csrc/glv.cuh — the sixteen-lane GLV scalar multiplication behind the prover's blinding products s*A, r*B1
    (groth16.go:272-273) and the verifier's public-input sum (groth16.go:283-286) — on an emulated warp, with the scalars
    split by the library's own glv_decompose: k * P equals the oracle's double-and-add (bn128/g1.go:140-155) as a group
    element for edge scalars (0, 1, 2, r-1, either side of 2^128, lambda-sized values), random full-width scalars, points in
    non-normalised Jacobian form, and the point at infinity."""
    G = o.BN.G1
    rng = random.Random(91)
    lam = 4407920970296243842393367215006156084916469457145843978461       # an element of order 3 mod r (the GLV eigenvalue's size)
    edge = [0, 1, 2, R_ - 1, R_ - 2, (1 << 128) - 1, 1 << 128, (1 << 128) + 1, (1 << 127), lam % R_, (R_ - lam) % R_, (1 << 253)]
    scalars = edge + [rng.randrange(R_) for _ in range(12)]
    if len(scalars) % 2:
        scalars.append(rng.randrange(R_))
    inf = (0, 0, 0)
    for i in range(0, len(scalars), 2):
        pts = []
        for j in range(2):
            if i == 4 and j == 1:
                pts.append(inf)                                   # the point at infinity times a scalar
            elif (i // 2 + j) % 3 == 0:
                pts.append(G.mul_scalar(G.G, rng.randrange(1, R_)))  # Jacobian with Z != 1 (the reference's own MulScalar output)
            else:
                a = G.affine(G.mul_scalar(G.G, rng.randrange(1, R_)))
                pts.append((a[0], a[1], 1))
        ks = scalars[i:i + 2]
        out = np.zeros(48, dtype=np.uint32)
        assert lib.t_glv_mul(_ptr(_u32([c for p in pts for c in p])), _ptr(_u32(ks)), _ptr(out)) == 0
        raw = out.tobytes()
        v = [int.from_bytes(raw[32 * n:32 * (n + 1)], "little") for n in range(6)]
        for j in range(2):
            got = (v[3 * j], v[3 * j + 1], v[3 * j + 2])
            exp = G.mul_scalar(pts[j], ks[j])
            if G.is_zero(exp):
                assert got[2] == 0, (ks[j], pts[j])
            else:
                assert got[2] != 0 and G.affine(got) == G.affine(exp), (ks[j], pts[j])
