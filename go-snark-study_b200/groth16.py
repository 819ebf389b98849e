"""Host mirror of the reference's ``groth16`` package prove path
(groth16/groth16.go:225-278) over libb200snark.

    pk  = {"G1": {"Alpha","Beta","Delta","At","BACGamma"}, "G2": {"Beta","Delta","BACGamma"},
           "BACDelta", "PowersTauDelta", "Z"}            (field names of groth16.Pk, groth16.go:15-32)
    proof = GenerateProofs(circuit, pk, w, px)           -> {"PiA","PiB","PiC"} Jacobian tuples

``circuit`` only needs ``NVars`` and ``NPublic`` (all the reference reads from it).
The proving key is uploaded once (``LoadProvingKey``) and cached per pk object.
"""
import secrets

import numpy as np

from . import _lib
from ._lib import check, ints_to_limbs, lib, ptr
from .bn128 import R, _flatten_g1, _flatten_g2, _unflatten_g1, _unflatten_g2, reduce_scalar


def _attr(obj, name):
    return obj[name] if isinstance(obj, dict) else getattr(obj, name)


def _n_signals(circuit, default):
    """len(circuit.Signals) (groth16.go:164, snark.go:171) for dict- and object-style circuits; NVars if absent."""
    if isinstance(circuit, dict):
        sig = circuit.get("Signals")
    else:
        sig = getattr(circuit, "Signals", None)
    return len(sig) if sig is not None else default


def rand_fr():
    """Fq.Rand over r (fields/fq.go:116-132): bitlen/8-1 = 30 random bytes, mod r."""
    return int.from_bytes(secrets.token_bytes(30), "big") % R


class DeviceProvingKey:
    """table_windows: stored window rows t per base set (B200_CFG_TABLE_WINDOWS; 0 = all, the fastest; 1 the smallest)."""

    def __init__(self, pk, n_vars, n_public, window_bits=0, table_windows=0):
        m = n_vars
        g1, g2 = pk["G1"], pk["G2"]
        assert len(g1["At"]) >= m and len(g1["BACGamma"]) >= m and len(g2["BACGamma"]) >= m and len(pk["BACDelta"]) >= m
        at = _flatten_g1(g1["At"][:m])
        b1 = _flatten_g1(g1["BACGamma"][:m])
        b2 = _flatten_g2(g2["BACGamma"][:m])
        cd = _flatten_g1(pk["BACDelta"][:m])
        ptd = _flatten_g1(pk["PowersTauDelta"])
        z = ints_to_limbs([int(x) % R for x in pk["Z"]])
        a1, be1, d1 = (_flatten_g1([g1[k]]) for k in ("Alpha", "Beta", "Delta"))
        be2, d2 = (_flatten_g2([g2[k]]) for k in ("Beta", "Delta"))
        h = _lib._h(0)
        with _lib.table_windows(table_windows):
            check(lib().b200_groth16_pk_load(ptr(at), ptr(b1), ptr(b2), ptr(cd), m, ptr(ptd), len(pk["PowersTauDelta"]),
                                             ptr(z), len(pk["Z"]), ptr(a1), ptr(be1), ptr(d1), ptr(be2), ptr(d2),
                                             n_public, window_bits, h))
        self.handle = h.value
        self.m = m

    @classmethod
    def from_handle(cls, handle, m):
        """Wrap a key already loaded with b200_groth16_pk_load(_shard)."""
        self = cls.__new__(cls)
        self.handle, self.m = handle, m
        return self

    def prove_limbs(self, w_limbs, px_limbs, r, s):
        pa = np.zeros(12, dtype=np.uint64)
        pb = np.zeros(24, dtype=np.uint64)
        pc = np.zeros(12, dtype=np.uint64)
        rr, ss = ints_to_limbs([r]), ints_to_limbs([s])
        check(lib().b200_groth16_prove(self.handle, ptr(w_limbs), w_limbs.shape[0], ptr(px_limbs), px_limbs.shape[0],
                                       ptr(rr), ptr(ss), ptr(pa), ptr(pb), ptr(pc)))
        return {"PiA": _unflatten_g1(pa)[0], "PiB": _unflatten_g2(pb)[0], "PiC": _unflatten_g1(pc)[0]}

    def prove_witness_limbs(self, r1cs, w_limbs, r, s):
        """The proof from the witness alone (b200_groth16_prove_witness): px, or the quotient directly, is computed on the
        device from ``r1cs`` (an r1csqap.SparseR1CS of the same circuit)."""
        pa = np.zeros(12, dtype=np.uint64)
        pb = np.zeros(24, dtype=np.uint64)
        pc = np.zeros(12, dtype=np.uint64)
        rr, ss = ints_to_limbs([r]), ints_to_limbs([s])
        check(lib().b200_groth16_prove_witness(self.handle, r1cs.handle, ptr(w_limbs), w_limbs.shape[0], ptr(rr), ptr(ss),
                                               ptr(pa), ptr(pb), ptr(pc)))
        return {"PiA": _unflatten_g1(pa)[0], "PiB": _unflatten_g2(pb)[0], "PiC": _unflatten_g1(pc)[0]}

    def prove_witness_batch_limbs(self, r1cs, w_limbs, rs):
        """k proofs in one call (b200_groth16_prove_witness_batch): ``w_limbs`` holds k witnesses (k x m x 4 limbs, or
        k*m x 4), ``rs`` a list of k (r, s) pairs.  Proof p is prove_witness_limbs(r1cs, w_limbs[p], *rs[p]).  On a key
        shard with a matching communicator (b200_comm_init, every rank calling with the same arguments) each rank
        computes its part of the k proofs, one all-gather of k records runs, and every rank gets all k proofs."""
        k = len(rs)
        w = np.ascontiguousarray(w_limbs, dtype=np.uint64).reshape(-1, 4)
        if k == 0 or w.shape[0] % k:
            raise ValueError("prove_witness_batch_limbs: need k >= 1 witnesses of equal length")
        rr = ints_to_limbs([r for r, _ in rs])
        ss = ints_to_limbs([s for _, s in rs])
        pa = np.zeros(12 * k, dtype=np.uint64)
        pb = np.zeros(24 * k, dtype=np.uint64)
        pc = np.zeros(12 * k, dtype=np.uint64)
        check(lib().b200_groth16_prove_witness_batch(self.handle, r1cs.handle, ptr(w), w.shape[0] // k, k, ptr(rr), ptr(ss),
                                                     ptr(pa), ptr(pb), ptr(pc)))
        a, b, c = _unflatten_g1(pa), _unflatten_g2(pb), _unflatten_g1(pc)
        return [{"PiA": a[p], "PiB": b[p], "PiC": c[p]} for p in range(k)]

    def device_bytes(self):
        return _lib.pk_device_bytes(self.handle)

    def free(self):
        if self.handle:
            check(lib().b200_pk_free(self.handle))
            self.handle = 0


class KeyCache:
    """Implicit proving-key cache of the drop-in ``GenerateProofs(circuit, pk, w, px)`` form (the reference takes the key
    by value on every call, groth16.go:225; uploading 384·n bytes and precomputing window tables per call would
    dominate).  An entry holds a STRONG reference to the caller's ``pk`` object and is matched by identity
    (``entry.pk is pk``) plus the shape it was loaded with — never by ``id()`` alone: a freed dict's address can be
    handed to a different key (round-1 bug: a proof under a stale key).  At most ``capacity`` keys stay resident;
    evicting one frees its device tables.  A caller that mutates ``pk`` in place must call ``Forget(pk)``."""

    def __init__(self, factory, capacity=2):
        self.factory, self.capacity, self.entries = factory, capacity, []

    def get(self, circuit, pk, window_bits=0, table_windows=0):
        shape = (_attr(circuit, "NVars"), _attr(circuit, "NPublic"), window_bits, table_windows)
        for k, (epk, eshape, dpk) in enumerate(self.entries):
            if epk is pk and eshape == shape:
                self.entries.append(self.entries.pop(k))          # most recently used last
                return dpk
        kw = {"table_windows": table_windows} if table_windows else {}
        dpk = self.factory(pk, shape[0], shape[1], window_bits, **kw)
        self.entries.append((pk, shape, dpk))
        while len(self.entries) > self.capacity:
            self.entries.pop(0)[2].free()
        return dpk

    def forget(self, pk=None):
        keep = []
        for e in self.entries:
            if pk is None or e[0] is pk:
                e[2].free()
            else:
                keep.append(e)
        self.entries = keep


_pk_cache = KeyCache(DeviceProvingKey)


def LoadProvingKey(circuit, pk, window_bits=0, table_windows=0):
    """Explicit handle form: the returned DeviceProvingKey can be passed as ``pk`` to GenerateProofs."""
    return _pk_cache.get(circuit, pk, window_bits, table_windows)


def Forget(pk=None):
    """Free the device copy of ``pk`` (all cached keys when None)."""
    _pk_cache.forget(pk)


def GenerateProofs(circuit, pk, w, px, r=None, s=None):
    """groth16.GenerateProofs(circuit, pk, w, px) (groth16.go:225).  r, s default
    to fresh randomness like the reference; pass them for reproducible proofs."""
    dpk = pk if isinstance(pk, DeviceProvingKey) else LoadProvingKey(circuit, pk)
    r = rand_fr() if r is None else int(r) % R
    s = rand_fr() if s is None else int(s) % R
    wl = ints_to_limbs([reduce_scalar(x) for x in w])
    pl = ints_to_limbs([int(x) % R for x in px])
    return dpk.prove_limbs(wl, pl, r, s)


def GenerateTrustedSetup(witnessLength, circuit, alphas, betas, gammas, toxic=None):
    """groth16.GenerateTrustedSetup (groth16/groth16.go:94-222) with the heavy loops on the GPU: the
    Eval(alphas[i], tau) evaluations (b200_poly_eval_batch), the z polynomial (b200_zero_poly) and every
    G.MulScalar(generator, k) (b200_g{1,2}_mul_batch_bcast — the reference's own double-and-add, so the
    points are X,Y,Z-identical to the reference's for the same toxic values).  ``toxic`` = dict
    T, Kalpha, Kbeta, Kgamma, Kdelta; drawn like the reference (Fq.Rand) when omitted.  ``witnessLength`` is
    unused, as in the reference.  Returns {"Toxic", "Pk", "Vk"} shaped like groth16.Setup."""
    from . import bn128
    from ._lib import limbs_to_ints
    n_vars, n_public = _attr(circuit, "NVars"), _attr(circuit, "NPublic")
    n_signals = _n_signals(circuit, n_vars)
    tox = {k: rand_fr() for k in ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta")} if toxic is None else toxic
    t, ka, kb, kg, kd = (int(tox[k]) % R for k in ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta"))
    if kg == 0 or kd == 0:
        raise ValueError("GenerateTrustedSetup: Kgamma and Kdelta must be invertible mod r (groth16.go:151,201)")
    m = len(alphas)
    nz = m - 2                                                   # z pol: prod_{i=1}^{len(alphas)-2} (x - i), :122-132
    zl = np.zeros((nz + 1, 4), dtype=np.uint64)
    check(lib().b200_zero_poly(nz, ptr(zl)))
    zpol = limbs_to_ints(zl)
    tl = ints_to_limbs([t])

    def evals(polys):
        n = len(polys[0])
        P = ints_to_limbs([int(x) % R for row in polys for x in row])
        out = np.zeros((len(polys), 4), dtype=np.uint64)
        check(lib().b200_poly_eval_batch(ptr(P), len(polys), n, ptr(tl), ptr(out)))
        return limbs_to_ints(out)

    zt = evals([zpol])[0]
    inv_delta = pow(kd, -1, R)
    zt_inv_delta = inv_delta * zt % R
    g1, g2 = bn128.G1(), bn128.G2()
    ptd_k, t_encr = [zt_inv_delta], t                            # :139-149
    for _ in range(1, len(zpol)):
        ptd_k.append(t_encr * zt_inv_delta % R)
        t_encr = t_encr * t % R
    at = evals(alphas[:n_signals])
    bt = evals(betas[:n_signals])
    ct = evals(gammas[:n_signals])
    inv_gamma = pow(kg, -1, R)
    c_k = [inv_delta * ((at[i] * kb + bt[i] * ka + ct[i]) % R) % R for i in range(n_public + 1, n_vars)]     # :181-200
    ic_k = [inv_gamma * ((at[i] * kb + bt[i] * ka + ct[i]) % R) % R for i in range(n_public + 1)]            # :202-219
    # one batched scalar multiplication of the G1 generator for every G1 point of the setup
    k1 = ptd_k + [ka, kb, kd] + at + bt + c_k + ic_k
    p1 = g1.MulScalarBatch([g1.G], k1)
    k2 = [kb, kg, kd] + bt
    p2 = g2.MulScalarBatch([g2.G], k2)
    o = 0
    ptd = p1[o:o + len(ptd_k)]; o += len(ptd_k)
    alpha1, beta1, delta1 = p1[o:o + 3]; o += 3
    At = p1[o:o + len(at)]; o += len(at)
    B1 = p1[o:o + len(bt)]; o += len(bt)
    Cd = p1[o:o + len(c_k)]; o += len(c_k)
    IC = p1[o:o + len(ic_k)]
    beta2, gamma2, delta2 = p2[:3]
    pk = {"BACDelta": [(0, 0, 0)] * (n_public + 1) + Cd, "Z": zpol, "PowersTauDelta": ptd,
          "G1": {"Alpha": alpha1, "Beta": beta1, "Delta": delta1, "At": At, "BACGamma": B1},
          "G2": {"Beta": beta2, "Gamma": gamma2, "Delta": delta2, "BACGamma": p2[3:]}}
    vk = {"IC": IC, "G1": {"Alpha": alpha1}, "G2": {"Beta": beta2, "Gamma": gamma2, "Delta": delta2}}
    return {"Toxic": {"T": t, "Kalpha": ka, "Kbeta": kb, "Kgamma": kg, "Kdelta": kd}, "Pk": pk, "Vk": vk}


def draw_toxic(names, n):
    """Toxic values drawn like the reference (Fq.Rand), T redrawn while it is one of the interpolation points 1..n."""
    tox = {k: rand_fr() for k in names}
    while 1 <= tox["T"] <= n:
        tox["T"] = rand_fr()
    return tox


def toxic_limbs(tox, names):
    return ints_to_limbs([int(tox[k]) for k in names])


class SparseSetup:
    """Groth16 key and Vk of GenerateTrustedSetupSparse as limb arrays (standard-form affine (x, y, 1) points, infinity
    all zero): at, b1, bacdelta (m G1), b2 (m G2), ptd (m-1 G1), z (m-1 coefficients), alpha1, beta1, delta1 (G1),
    beta2, gamma2, delta2 (G2), ic (npublic+1 G1).  A 2^20-constraint key is ~0.6 GB here; as tuples of Python ints it
    would take gigabytes, so ``pk_dict`` is for small circuits only."""
    TOXIC = ("T", "Kalpha", "Kbeta", "Kgamma", "Kdelta")

    def __init__(self, r1cs, n_public, toxic=None):
        m = self.m = r1cs.m
        self.n, self.npublic = r1cs.n, n_public
        tox = draw_toxic(self.TOXIC, r1cs.n) if toxic is None else dict(toxic)
        self.Toxic = {k: int(tox[k]) for k in self.TOXIC}
        g1 = lambda k: np.zeros((k, 12), dtype=np.uint64)
        g2 = lambda k: np.zeros((k, 24), dtype=np.uint64)
        self.at, self.b1, self.bacdelta, self.b2, self.ptd = g1(m), g1(m), g1(m), g2(m), g1(m - 1)
        self.z = np.zeros((m - 1, 4), dtype=np.uint64)
        self.alpha1, self.beta1, self.delta1 = g1(1), g1(1), g1(1)
        self.beta2, self.gamma2, self.delta2 = g2(1), g2(1), g2(1)
        self.ic = g1(n_public + 1)
        check(lib().b200_groth16_setup(r1cs.handle, n_public, ptr(toxic_limbs(self.Toxic, self.TOXIC)), ptr(self.at),
                                       ptr(self.b1), ptr(self.b2), ptr(self.bacdelta), ptr(self.ptd), ptr(self.z),
                                       ptr(self.alpha1), ptr(self.beta1), ptr(self.delta1), ptr(self.beta2),
                                       ptr(self.gamma2), ptr(self.delta2), ptr(self.ic)))
        self.Vk = {"IC": _unflatten_g1(self.ic), "G1": {"Alpha": _unflatten_g1(self.alpha1)[0]},
                   "G2": {"Beta": _unflatten_g2(self.beta2)[0], "Gamma": _unflatten_g2(self.gamma2)[0],
                          "Delta": _unflatten_g2(self.delta2)[0]}}

    def load_pk(self, window_bits=0, rank=0, world=1, table_windows=0):
        """The key on the device (b200_groth16_pk_load_shard): a DeviceProvingKey with prove_limbs / prove_witness_limbs.
        table_windows: stored window rows per base set (B200_CFG_TABLE_WINDOWS; 0 = all)."""
        h = _lib._h(0)
        with _lib.table_windows(table_windows):
            check(lib().b200_groth16_pk_load_shard(
                ptr(self.at), ptr(self.b1), ptr(self.b2), ptr(self.bacdelta), self.m, ptr(self.ptd), self.m - 1,
                ptr(self.z), self.m - 1, ptr(self.alpha1), ptr(self.beta1), ptr(self.delta1), ptr(self.beta2),
                ptr(self.delta2), self.npublic, window_bits, rank, world, h))
        return DeviceProvingKey.from_handle(h.value, self.m)

    def pk_dict(self):
        """The key in the shape GenerateTrustedSetup returns (Python ints; small circuits only)."""
        from ._lib import limbs_to_ints
        return {"BACDelta": _unflatten_g1(self.bacdelta), "Z": limbs_to_ints(self.z), "PowersTauDelta": _unflatten_g1(self.ptd),
                "G1": {"Alpha": _unflatten_g1(self.alpha1)[0], "Beta": _unflatten_g1(self.beta1)[0],
                       "Delta": _unflatten_g1(self.delta1)[0], "At": _unflatten_g1(self.at), "BACGamma": _unflatten_g1(self.b1)},
                "G2": {"Beta": self.Vk["G2"]["Beta"], "Gamma": self.Vk["G2"]["Gamma"], "Delta": self.Vk["G2"]["Delta"],
                       "BACGamma": _unflatten_g2(self.b2)}}


def GenerateTrustedSetupSparse(r1cs, nPublic, toxic=None):
    """groth16.GenerateTrustedSetup (groth16/groth16.go:94-222) for an r1csqap.SparseR1CS of any size, on the GPU
    (b200_groth16_setup): the same group elements as GenerateTrustedSetup for the same toxic values, as affine points.
    ``toxic`` = dict T, Kalpha, Kbeta, Kgamma, Kdelta; drawn like the reference when omitted (T never in 1..n)."""
    return SparseSetup(r1cs, nPublic, toxic)


class ResidentSetup:
    """A trusted setup made straight into a device-resident proving key: ``pk`` (a DeviceProvingKey), ``Vk`` (the dict
    VerifyProof takes) and ``Toxic`` (the toxic values it was made with)."""

    def __init__(self, pk, vk, toxic):
        self.pk, self.Vk, self.Toxic = pk, vk, toxic


def _resident_toxic(names, r1cs, toxic, world):
    if toxic is None and world > 1:
        raise ValueError("GenerateTrustedSetupResident: a sharded setup (world > 1) needs the toxic values every rank "
                         "shares; independently drawn ones would give an inconsistent key")
    tox = draw_toxic(names, r1cs.n) if toxic is None else dict(toxic)
    return {k: int(tox[k]) for k in names}


def GenerateTrustedSetupResident(r1cs, nPublic, toxic=None, window_bits=0, rank=0, world=1, table_windows=0):
    """GenerateTrustedSetupSparse(r1cs, nPublic, toxic).load_pk(window_bits, rank, world, table_windows) in one call
    (b200_groth16_setup_pk): the key is minted on the device straight into its tables, no CRS passes through host
    memory, and rank ``rank`` of ``world`` mints only the part of the key it holds.  Every rank must pass the same toxic
    values, so ``toxic`` is required when world > 1."""
    names = SparseSetup.TOXIC
    tox = _resident_toxic(names, r1cs, toxic, world)
    g1 = lambda k: np.zeros((k, 12), dtype=np.uint64)
    g2 = lambda k: np.zeros((k, 24), dtype=np.uint64)
    alpha1, beta2, gamma2, delta2, ic = g1(1), g2(1), g2(1), g2(1), g1(nPublic + 1)
    h = _lib._h(0)
    with _lib.table_windows(table_windows):
        check(lib().b200_groth16_setup_pk(r1cs.handle, nPublic, ptr(toxic_limbs(tox, names)), window_bits, rank, world, h,
                                          ptr(alpha1), ptr(beta2), ptr(gamma2), ptr(delta2), ptr(ic)))
    vk = {"IC": _unflatten_g1(ic), "G1": {"Alpha": _unflatten_g1(alpha1)[0]},
          "G2": {"Beta": _unflatten_g2(beta2)[0], "Gamma": _unflatten_g2(gamma2)[0], "Delta": _unflatten_g2(delta2)[0]}}
    return ResidentSetup(DeviceProvingKey.from_handle(h.value, r1cs.m), vk, tox)


def VerifyProof(vk, proof, publicSignals, debug=False):
    """groth16.VerifyProof(vk, proof, publicSignals, debug) (groth16/groth16.go:281-305) on the GPU:
    vk = {"IC", "G1": {"Alpha"}, "G2": {"Beta", "Gamma", "Delta"}}, proof = {"PiA", "PiB", "PiC"}."""
    import ctypes
    ic = _flatten_g1(vk["IC"])
    pub = ints_to_limbs([reduce_scalar(x) for x in publicSignals]) if len(publicSignals) else np.zeros((1, 4), dtype=np.uint64)
    ok = ctypes.c_int(0)
    check(lib().b200_groth16_verify(ptr(ic), len(vk["IC"]), ptr(_flatten_g1([vk["G1"]["Alpha"]])),
                                    ptr(_flatten_g2([vk["G2"]["Beta"]])), ptr(_flatten_g2([vk["G2"]["Gamma"]])),
                                    ptr(_flatten_g2([vk["G2"]["Delta"]])), ptr(_flatten_g1([proof["PiA"]])),
                                    ptr(_flatten_g2([proof["PiB"]])), ptr(_flatten_g1([proof["PiC"]])), ptr(pub),
                                    len(publicSignals), ctypes.byref(ok)))
    if debug:
        print("✓ groth16 verification passed" if ok.value else "❌ groth16 verification not passed")
    return bool(ok.value)


# status word of b200_groth16_verify_batch(_device) (include/b200snark.h)
VB_AGGREGATE, VB_PER_PROOF, VB_ROUTED, VB_RANGE = 1, 2, 4, 8


def draw_rho(k):
    """k randomisers for a batch verification: secrets.randbits(128), zeros redrawn."""
    out = []
    while len(out) < k:
        v = secrets.randbits(128)
        if v:
            out.append(v)
    return out


def _rho_limbs(rho):
    return np.array([w for v in rho for w in (int(v) & (2**64 - 1), int(v) >> 64)], dtype=np.uint64)


def _vk_args(vk):
    return (_flatten_g1(vk["IC"]), _flatten_g1([vk["G1"]["Alpha"]]), _flatten_g2([vk["G2"]["Beta"]]),
            _flatten_g2([vk["G2"]["Gamma"]]), _flatten_g2([vk["G2"]["Delta"]]))


def verify_batch_limbs(vk, proofs, publicSignalsList, rho=None):
    """b200_groth16_verify_batch: (list of k verdicts, status word).  ``rho``: k randomisers in 1..2^128 - 1 (drawn
    with draw_rho when None; pass them for reproducible runs)."""
    import ctypes
    k = len(proofs)
    if k == 0 or len(publicSignalsList) != k:
        raise ValueError("verify_batch: need k >= 1 proofs and one publicSignals list per proof")
    npub = len(publicSignalsList[0])
    if any(len(ps) != npub for ps in publicSignalsList):
        raise ValueError("verify_batch: every proof needs the same number of public signals")
    rho = draw_rho(k) if rho is None else list(rho)
    ic, a1, b2, g2, d2 = _vk_args(vk)
    pa = _flatten_g1([p["PiA"] for p in proofs])
    pb = _flatten_g2([p["PiB"] for p in proofs])
    pc = _flatten_g1([p["PiC"] for p in proofs])
    pub = (ints_to_limbs([reduce_scalar(x) for ps in publicSignalsList for x in ps]) if npub
           else np.zeros((1, 4), dtype=np.uint64))
    ok = np.zeros(k, dtype=np.int32)
    status = ctypes.c_uint32(0)
    check(lib().b200_groth16_verify_batch(ptr(ic), len(vk["IC"]), ptr(a1), ptr(b2), ptr(g2), ptr(d2), ptr(pa), ptr(pb),
                                          ptr(pc), ptr(pub), npub, k, ptr(_rho_limbs(rho)), ptr(ok), ctypes.byref(status)))
    return [bool(v) for v in ok], status.value


def VerifyProofBatch(vk, proofs, publicSignalsList, rho=None):
    """[groth16.VerifyProof(vk, proofs[i], publicSignalsList[i]) for every i] in one call (b200_groth16_verify_batch): one
    random linear combination of the regular proofs, k + 3 Miller loops and one final exponentiation; irregular proofs,
    and every proof of a batch whose combination fails, get the single call's verdict.  ``rho`` defaults to fresh
    128-bit randomisers (secrets.randbits), which is what makes an invalid proof's acceptance improbable."""
    return verify_batch_limbs(vk, proofs, publicSignalsList, rho)[0]


def VerifyProofBatchDevice(vk, d_proofs, d_public, k, n_public, rho=None, d_ok=None, stream=None):
    """b200_groth16_verify_batch_device on a batch in device memory: ``d_proofs`` is the output tensor of
    b200_groth16_prove_witness_batch_device (k x 48 words, PiA | PiC | PiB), ``d_public`` the k x n_public x 4 standard-form
    signals.  Queued on ``stream`` (a torch.cuda.Stream; None: the library's main stream) without waiting; returns the
    int32 tensor of k verdicts followed by the status word (``d_ok``, allocated when None)."""
    import torch
    rho = draw_rho(k) if rho is None else list(rho)
    if d_ok is None:
        d_ok = torch.zeros(k + 1, dtype=torch.int32, device=d_proofs.device)
    ic, a1, b2, g2, d2 = _vk_args(vk)
    check(lib().b200_groth16_verify_batch_device(ptr(ic), len(vk["IC"]), ptr(a1), ptr(b2), ptr(g2), ptr(d2),
                                                 d_proofs.data_ptr(), d_public.data_ptr() if n_public else None, n_public,
                                                 k, ptr(_rho_limbs(rho)), d_ok.data_ptr(),
                                                 None if stream is None else stream.cuda_stream))
    return d_ok
