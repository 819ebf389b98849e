"""Host mirror of the reference's root ``snark`` package (Pinocchio) over libb200snark: the prove path
(snark.go:254-289), and — SURVEY §8f rows 1-2 — the trusted setup (snark.go:98-251) and VerifyProof (:292-372).

    pk = {"A","Ap","B","Bp","C","Cp","Kp","G1T","Z"}   (snark.Pk, snark.go:16-26; B is in G2)
    proof = GenerateProofs(circuit, pk, w, px) -> PiA PiAp PiB PiBp PiC PiCp PiH PiKp
"""
import numpy as np

from . import _lib
from ._lib import check, ints_to_limbs, lib, ptr
from .bn128 import R, _flatten_g1, _flatten_g2, _unflatten_g1, _unflatten_g2, reduce_scalar
from .groth16 import KeyCache, _attr, _n_signals

_ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")


class DeviceProvingKey:
    """table_windows: stored window rows t per base set (B200_CFG_TABLE_WINDOWS; 0 = all, the fastest; 1 the smallest)."""

    def __init__(self, pk, n_vars, n_public, window_bits=0, table_windows=0):
        m = n_vars
        arr = {k: _flatten_g1(pk[k][:m]) for k in ("A", "Ap", "Bp", "C", "Cp", "Kp")}
        b2 = _flatten_g2(pk["B"][:m])
        g1t = _flatten_g1(pk["G1T"])
        z = ints_to_limbs([int(x) % R for x in pk["Z"]])
        h = _lib._h(0)
        with _lib.table_windows(table_windows):
            check(lib().b200_pinocchio_pk_load(ptr(arr["A"]), ptr(arr["Ap"]), ptr(b2), ptr(arr["Bp"]), ptr(arr["C"]),
                                               ptr(arr["Cp"]), ptr(arr["Kp"]), m, ptr(g1t), len(pk["G1T"]), ptr(z),
                                               len(pk["Z"]), n_public, window_bits, h))
        self.handle = h.value

    @classmethod
    def from_handle(cls, handle):
        """Wrap a key already loaded with b200_pinocchio_pk_load(_shard)."""
        self = cls.__new__(cls)
        self.handle = handle
        return self

    def prove_limbs(self, w_limbs, px_limbs):
        g1 = np.zeros(84, dtype=np.uint64)
        pb = np.zeros(24, dtype=np.uint64)
        check(lib().b200_pinocchio_prove(self.handle, ptr(w_limbs), w_limbs.shape[0], ptr(px_limbs),
                                         px_limbs.shape[0], ptr(g1), ptr(pb)))
        proof = dict(zip(_ORDER, _unflatten_g1(g1)))
        proof["PiB"] = _unflatten_g2(pb)[0]
        return proof

    def prove_witness_limbs(self, r1cs, w_limbs):
        """The proof from the witness alone (b200_pinocchio_prove_witness): px, or the quotient directly, is computed on
        the device from ``r1cs`` (an r1csqap.SparseR1CS of the same circuit)."""
        g1 = np.zeros(84, dtype=np.uint64)
        pb = np.zeros(24, dtype=np.uint64)
        check(lib().b200_pinocchio_prove_witness(self.handle, r1cs.handle, ptr(w_limbs), w_limbs.shape[0], ptr(g1), ptr(pb)))
        proof = dict(zip(_ORDER, _unflatten_g1(g1)))
        proof["PiB"] = _unflatten_g2(pb)[0]
        return proof

    def prove_witness_batch_limbs(self, r1cs, w_limbs):
        """k proofs in one call (b200_pinocchio_prove_witness_batch): ``w_limbs`` holds k witnesses (k x m x 4 limbs).
        Proof p is prove_witness_limbs(r1cs, w_limbs[p])."""
        w = np.ascontiguousarray(w_limbs, dtype=np.uint64)
        if w.ndim != 3 or w.shape[0] == 0 or w.shape[2] != 4:
            raise ValueError("prove_witness_batch_limbs: need k >= 1 witnesses as a k x m x 4 array")
        k, m = w.shape[0], w.shape[1]
        g1 = np.zeros(84 * k, dtype=np.uint64)
        pb = np.zeros(24 * k, dtype=np.uint64)
        check(lib().b200_pinocchio_prove_witness_batch(self.handle, r1cs.handle, ptr(w), m, k, ptr(g1), ptr(pb)))
        p1, p2 = _unflatten_g1(g1), _unflatten_g2(pb)
        proofs = [dict(zip(_ORDER, p1[7 * p:7 * p + 7])) for p in range(k)]
        for p in range(k):
            proofs[p]["PiB"] = p2[p]
        return proofs

    def device_bytes(self):
        return _lib.pk_device_bytes(self.handle)

    def free(self):
        if self.handle:
            check(lib().b200_pk_free(self.handle))
            self.handle = 0


_pk_cache = KeyCache(DeviceProvingKey)       # see groth16.KeyCache (identity + strong ref)


def LoadProvingKey(circuit, pk, window_bits=0, table_windows=0):
    return _pk_cache.get(circuit, pk, window_bits, table_windows)


def Forget(pk=None):
    _pk_cache.forget(pk)


def GenerateProofs(circuit, pk, w, px):
    """snark.GenerateProofs(circuit, pk, w, px) (snark.go:254). Deterministic."""
    dpk = pk if isinstance(pk, DeviceProvingKey) else LoadProvingKey(circuit, pk)
    wl = ints_to_limbs([reduce_scalar(x) for x in w])
    pl = ints_to_limbs([int(x) % R for x in px])
    return dpk.prove_limbs(wl, pl)


def GenerateTrustedSetup(witnessLength, circuit, alphas, betas, gammas, toxic=None):
    """snark.GenerateTrustedSetup (snark.go:98-251) with the heavy loops on the GPU: Eval(alphas[i], t) as one batched
    evaluation per matrix, every MulScalar as the reference's own double-and-add in batch kernels (so Jacobian X,Y,Z
    equal the reference's for the same toxic values), and the reference's k == a + b + c self-check (:194-199) as
    batched group additions.  ``toxic`` = dict T, Ka, Kb, Kc, Kbeta, Kgamma, RhoA, RhoB (RhoC = RhoA*RhoB, :150);
    drawn like the reference (Fq.Rand) when omitted.  Returns {"Toxic", "Pk", "Vk"} shaped like snark.Setup."""
    from . import bn128
    from ._lib import limbs_to_ints
    from .groth16 import rand_fr
    n_vars, n_public = _attr(circuit, "NVars"), _attr(circuit, "NPublic")
    n_signals = _n_signals(circuit, n_vars)
    tox = {k: rand_fr() for k in ("T", "Ka", "Kb", "Kc", "Kbeta", "Kgamma", "RhoA", "RhoB")} if toxic is None else dict(toxic)
    t, ka, kb, kc, kbeta, kgamma, rho_a, rho_b = (int(tox[k]) % R for k in
                                                  ("T", "Ka", "Kb", "Kc", "Kbeta", "Kgamma", "RhoA", "RhoB"))
    rho_c = rho_a * rho_b % R
    kbg = kbeta * kgamma % R
    nz = len(alphas) - 2                                         # z pol, :210-221
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
    ra = [rho_a * v % R for v in evals(alphas[:n_signals])]      # rhoAat, :173
    rb = [rho_b * v % R for v in evals(betas[:n_signals])]       # rhoBbt, :181
    rc = [rho_c * v % R for v in evals(gammas[:n_signals])]      # rhoCct, :188
    kt = [(ra[i] + rb[i] + rc[i]) % R for i in range(n_signals)]
    t_pows, t_encr = [], t                                       # G1T = [G, tG, t^2 G, ...], :230-237
    for _ in range(1, len(zpol)):
        t_pows.append(t_encr)
        t_encr = t_encr * t % R
    g1, g2 = bn128.G1(), bn128.G2()
    n = n_signals
    p1 = g1.MulScalarBatch([g1.G], [kb, kbg] + ra + rb + rc + kt + t_pows)
    vkb, g1kbg = p1[0], p1[1]
    A, Bg1, C, K = p1[2:2 + n], p1[2 + n:2 + 2 * n], p1[2 + 2 * n:2 + 3 * n], p1[2 + 3 * n:2 + 4 * n]
    g1t = [g1.G] + p1[2 + 4 * n:]
    p2 = g2.MulScalarBatch([g2.G], [ka, kc, kbg, kgamma, rho_c * zt % R] + rb)
    vka, vkc, g2kbg, g2kg, vkz = p2[:5]
    # the reference's self-check: Affine(G * kt) == Affine(a + bg1 + c), else os.Exit(1)
    ab = _unflatten_g1(g1._op("add", A, Bg1))
    abc = _unflatten_g1(g1._op("add", ab, C))
    if limbs_to_ints(g1._op("affine", abc, out_fe=2)) != limbs_to_ints(g1._op("affine", K, out_fe=2)):
        raise RuntimeError("GenerateTrustedSetup: k != a + b + c (snark.go:194-199)")
    pk = {"G1T": g1t, "A": A, "B": p2[5:], "C": C, "Z": zpol,
          "Ap": g1.MulScalarBatch(A, [ka] * n), "Bp": g1.MulScalarBatch(Bg1, [kb] * n),
          "Cp": g1.MulScalarBatch(C, [kc] * n), "Kp": g1.MulScalarBatch(K, [kbeta] * n)}
    vk = {"Vka": vka, "Vkb": vkb, "Vkc": vkc, "IC": A[:n_public + 1], "G1Kbg": g1kbg, "G2Kbg": g2kbg, "G2Kg": g2kg,
          "Vkz": vkz}
    toxic_out = {"T": t, "Ka": ka, "Kb": kb, "Kc": kc, "Kbeta": kbeta, "Kgamma": kgamma, "RhoA": rho_a, "RhoB": rho_b,
                 "RhoC": rho_c}
    return {"Toxic": toxic_out, "Pk": pk, "Vk": vk}


class SparseSetup:
    """Pinocchio key and Vk of GenerateTrustedSetupSparse as limb arrays (standard-form affine (x, y, 1) points, infinity
    all zero): a, ap, bp, c, cp, kp (m G1), b2 (m G2), g1t (m-1 G1), z (m-1 coefficients), vk_g1 = Vkb | G1Kbg,
    vk_g2 = Vka | Vkc | G2Kbg | G2Kg | Vkz.  ``pk_dict`` is for small circuits only."""
    TOXIC = ("T", "Ka", "Kb", "Kc", "Kbeta", "Kgamma", "RhoA", "RhoB")

    def __init__(self, r1cs, n_public, toxic=None):
        from .groth16 import draw_toxic, toxic_limbs
        m = self.m = r1cs.m
        self.n, self.npublic = r1cs.n, n_public
        tox = draw_toxic(self.TOXIC, r1cs.n) if toxic is None else dict(toxic)
        self.Toxic = {k: int(tox[k]) for k in self.TOXIC}
        self.Toxic["RhoC"] = self.Toxic["RhoA"] * self.Toxic["RhoB"] % R
        g1 = lambda k: np.zeros((k, 12), dtype=np.uint64)
        self.a, self.ap, self.bp, self.c, self.cp, self.kp = (g1(m) for _ in range(6))
        self.b2 = np.zeros((m, 24), dtype=np.uint64)
        self.g1t = g1(m - 1)
        self.z = np.zeros((m - 1, 4), dtype=np.uint64)
        self.vk_g1, self.vk_g2 = g1(2), np.zeros((5, 24), dtype=np.uint64)
        check(lib().b200_pinocchio_setup(r1cs.handle, n_public, ptr(toxic_limbs(self.Toxic, self.TOXIC)), ptr(self.a),
                                         ptr(self.ap), ptr(self.b2), ptr(self.bp), ptr(self.c), ptr(self.cp), ptr(self.kp),
                                         ptr(self.g1t), ptr(self.z), ptr(self.vk_g1), ptr(self.vk_g2)))
        self.Vk = dict(zip(("Vkb", "G1Kbg"), _unflatten_g1(self.vk_g1)))
        self.Vk.update(zip(("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz"), _unflatten_g2(self.vk_g2)))
        self.Vk["IC"] = _unflatten_g1(self.a[:n_public + 1])

    def load_pk(self, window_bits=0, rank=0, world=1, table_windows=0):
        """The key on the device (b200_pinocchio_pk_load_shard): a DeviceProvingKey with prove_limbs.
        table_windows: stored window rows per base set (B200_CFG_TABLE_WINDOWS; 0 = all)."""
        h = _lib._h(0)
        with _lib.table_windows(table_windows):
            check(lib().b200_pinocchio_pk_load_shard(
                ptr(self.a), ptr(self.ap), ptr(self.b2), ptr(self.bp), ptr(self.c), ptr(self.cp), ptr(self.kp), self.m,
                ptr(self.g1t), self.m - 1, ptr(self.z), self.m - 1, self.npublic, window_bits, rank, world, h))
        return DeviceProvingKey.from_handle(h.value)

    def pk_dict(self):
        """The key in the shape GenerateTrustedSetup returns (Python ints; small circuits only)."""
        from ._lib import limbs_to_ints
        pk = {k: _unflatten_g1(getattr(self, k.lower())) for k in ("A", "Ap", "Bp", "C", "Cp", "Kp")}
        pk.update({"B": _unflatten_g2(self.b2), "G1T": _unflatten_g1(self.g1t), "Z": limbs_to_ints(self.z)})
        return pk


def GenerateTrustedSetupSparse(r1cs, nPublic, toxic=None):
    """snark.GenerateTrustedSetup (snark.go:98-251) for an r1csqap.SparseR1CS of any size, on the GPU
    (b200_pinocchio_setup): the same group elements as GenerateTrustedSetup for the same toxic values, as affine points.
    ``toxic`` = dict T, Ka, Kb, Kc, Kbeta, Kgamma, RhoA, RhoB; drawn like the reference when omitted (T never in 1..n)."""
    return SparseSetup(r1cs, nPublic, toxic)


def GenerateTrustedSetupResident(r1cs, nPublic, toxic=None, window_bits=0, rank=0, world=1, table_windows=0):
    """GenerateTrustedSetupSparse(r1cs, nPublic, toxic).load_pk(window_bits, rank, world, table_windows) in one call
    (b200_pinocchio_setup_pk): the key is minted on the device straight into its tables, no CRS passes through host
    memory, and rank ``rank`` of ``world`` mints only the sets it holds.  Returns a groth16.ResidentSetup (``pk``, ``Vk``
    as VerifyProof takes it, ``Toxic`` with RhoC).  Every rank must pass the same toxic values, so ``toxic`` is required
    when world > 1."""
    from .groth16 import ResidentSetup, _resident_toxic, toxic_limbs
    names = SparseSetup.TOXIC
    tox = _resident_toxic(names, r1cs, toxic, world)
    vk_g1, vk_g2 = np.zeros((2, 12), dtype=np.uint64), np.zeros((5, 24), dtype=np.uint64)
    ic = np.zeros((nPublic + 1, 12), dtype=np.uint64)
    h = _lib._h(0)
    with _lib.table_windows(table_windows):
        check(lib().b200_pinocchio_setup_pk(r1cs.handle, nPublic, ptr(toxic_limbs(tox, names)), window_bits, rank, world, h,
                                            ptr(vk_g1), ptr(vk_g2), ptr(ic)))
    vk = dict(zip(("Vkb", "G1Kbg"), _unflatten_g1(vk_g1)))
    vk.update(zip(("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz"), _unflatten_g2(vk_g2)))
    vk["IC"] = _unflatten_g1(ic)
    tox["RhoC"] = tox["RhoA"] * tox["RhoB"] % R
    return ResidentSetup(DeviceProvingKey.from_handle(h.value), vk, tox)


def VerifyProof(vk, proof, publicSignals, debug=False):
    """snark.VerifyProof(vk, proof, publicSignals, debug) (snark.go:292-372): the twelve pairings of the five checks run
    as ONE batched GPU call (lock-step lanes of a warp), the two F_q^12 products as another; the checks are then
    evaluated in the reference's order, with its ✓/❌ lines when ``debug``."""
    from . import bn128
    bn = bn128.Bn128()
    g1, g2g = bn.G1, bn.G2.G
    vkxpia = vk["IC"][0]
    if len(publicSignals) > len(vk["IC"]) - 1:
        raise IndexError("VerifyProof: len(publicSignals) > len(vk.IC) - 1")     # the reference panics (index out of range)
    if publicSignals:
        terms = g1.MulScalarBatch(list(vk["IC"][1:len(publicSignals) + 1]), list(publicSignals))
        for term in terms:                                                       # :334-337
            vkxpia = g1.Add(vkxpia, term)
    vkx_a = g1.Add(vkxpia, proof["PiA"])
    vkx_a_c = g1.Add(vkx_a, proof["PiC"])
    e = bn.PairingBatch(
        [proof["PiA"], proof["PiAp"], vk["Vkb"], proof["PiBp"], proof["PiC"], proof["PiCp"],
         vkx_a, proof["PiH"], proof["PiC"], vkx_a_c, vk["G1Kbg"], proof["PiKp"]],
        [vk["Vka"], g2g, proof["PiB"], g2g, vk["Vkc"], g2g,
         proof["PiB"], vk["Vkz"], g2g, vk["G2Kbg"], proof["PiB"], vk["G2Kg"]])
    prod = bn.Fq12MulBatch([e[7], e[9]], [e[8], e[10]])
    checks = (
        (e[0] == e[1], "e(piA, Va) == e(piA', g2), valid knowledge commitment for A"),
        (e[2] == e[3], "e(Vb, piB) == e(piB', g2), valid knowledge commitment for B"),
        (e[4] == e[5], "e(piC, Vc) == e(piC', g2), valid knowledge commitment for C"),
        (e[6] == prod[0], "e(Vkx+piA, piB) == e(piH, Vkz) * e(piC, g2), QAP disibility checked"),
        (prod[1] == e[11], "e(Vkx+piA+piC, g2KbetaKgamma) * e(g1KbetaKgamma, piB) == e(piK, g2Kgamma)"),
    )
    for k, (ok, text) in enumerate(checks):
        if debug or (k == 4 and not ok):          # the last failure line is printed unconditionally (snark.go:360-363)
            print(("✓ " if ok else "❌ ") + text)
        if not ok:
            return False
    return True


def _vk_args(vk):
    return (_flatten_g1(vk["IC"]), _flatten_g1([vk["Vkb"], vk["G1Kbg"]]),
            _flatten_g2([vk["Vka"], vk["Vkc"], vk["G2Kbg"], vk["G2Kg"], vk["Vkz"]]))


def verify_batch_limbs(vk, proofs, publicSignalsList, rho=None):
    """b200_pinocchio_verify_batch: (list of k verdicts, status word; its bits are groth16.VB_*).  ``rho``: 5k randomisers in 1..2^128 - 1, rho[5 i + c - 1]
    for check c of proof i (drawn with groth16.draw_rho when None; pass them for reproducible runs)."""
    import ctypes
    from .groth16 import _rho_limbs, draw_rho
    k = len(proofs)
    if k == 0 or len(publicSignalsList) != k:
        raise ValueError("verify_batch: need k >= 1 proofs and one publicSignals list per proof")
    npub = len(publicSignalsList[0])
    if any(len(ps) != npub for ps in publicSignalsList):
        raise ValueError("verify_batch: every proof needs the same number of public signals")
    rho = draw_rho(5 * k) if rho is None else list(rho)
    if len(rho) != 5 * k:
        raise ValueError("verify_batch: need five randomisers per proof")
    ic, g1, g2 = _vk_args(vk)
    out_g1 = _flatten_g1([p[s] for p in proofs for s in _ORDER])
    pb = _flatten_g2([p["PiB"] for p in proofs])
    pub = (ints_to_limbs([reduce_scalar(x) for ps in publicSignalsList for x in ps]) if npub
           else np.zeros((1, 4), dtype=np.uint64))
    ok = np.zeros(k, dtype=np.int32)
    status = ctypes.c_uint32(0)
    check(lib().b200_pinocchio_verify_batch(ptr(ic), len(vk["IC"]), ptr(g1), ptr(g2), ptr(out_g1), ptr(pb), ptr(pub), npub, k,
                                            ptr(_rho_limbs(rho)), ptr(ok), ctypes.byref(status)))
    return [bool(v) for v in ok], status.value


def VerifyProofBatch(vk, proofs, publicSignalsList, rho=None):
    """[snark.VerifyProof(vk, proofs[i], publicSignalsList[i]) for every i] in one call (b200_pinocchio_verify_batch): one
    random linear combination of the five checks of the regular proofs, k + 6 Miller loops and one final exponentiation;
    irregular proofs, and every proof of a batch whose combination fails, get VerifyProof's verdict.  ``rho`` defaults to
    fresh 128-bit randomisers (secrets.randbits), five per proof, which is what makes an invalid proof's acceptance
    improbable."""
    return verify_batch_limbs(vk, proofs, publicSignalsList, rho)[0]


def VerifyProofBatchDevice(vk, d_proofs, d_public, k, n_public, rho=None, d_ok=None, stream=None):
    """b200_pinocchio_verify_batch_device on a batch in device memory: ``d_proofs`` is the output tensor of
    b200_pinocchio_prove_witness_batch_device (k x 108 words: PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp, PiB), ``d_public`` the
    k x n_public x 4 standard-form signals.  Queued on ``stream`` (a torch.cuda.Stream; None: the library's main stream)
    without waiting; returns the int32 tensor of k verdicts followed by the status word (``d_ok``, allocated when None)."""
    import torch
    from .groth16 import _rho_limbs, draw_rho
    rho = draw_rho(5 * k) if rho is None else list(rho)
    if len(rho) != 5 * k:
        raise ValueError("verify_batch: need five randomisers per proof")
    if d_ok is None:
        d_ok = torch.zeros(k + 1, dtype=torch.int32, device=d_proofs.device)
    ic, g1, g2 = _vk_args(vk)
    check(lib().b200_pinocchio_verify_batch_device(ptr(ic), len(vk["IC"]), ptr(g1), ptr(g2), d_proofs.data_ptr(),
                                                   d_public.data_ptr() if n_public else None, n_public, k,
                                                   ptr(_rho_limbs(rho)), d_ok.data_ptr(),
                                                   None if stream is None else stream.cuda_stream))
    return d_ok
