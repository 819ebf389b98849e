"""GPU: batched Groth16 verification (include/b200snark.h: b200_groth16_verify_batch, b200_groth16_verify_batch_device) on
proofs made by the batch prover under a real key (synthetic.CircuitGroth16).  Every verdict that the contract ties to
b200_groth16_verify is compared with b200_groth16_verify on that proof."""
import ctypes
import random

import numpy as np
import pytest

from oracle import ref_py as o

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
R, Q = o.R, o.Q
EINVAL, ERANGE = -3, -4
N = 1 << 10


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def limbs(vals):
    from gosnark_b200._lib import ints_to_limbs
    return ints_to_limbs(list(vals))


def _p(a):
    from gosnark_b200._lib import ptr
    return ptr(a)


def rho_limbs(rho):
    return np.array([w for v in rho for w in (v & (2**64 - 1), v >> 64)], dtype=np.uint64)


def to_dev(arr):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


class Batch:
    """64 proofs of distinct satisfying witnesses of CircuitGroth16(N), proved in one b200_groth16_prove_witness_batch_device
    call; ``d_out`` is the prover's output tensor, ``words`` its host copy (k x 48: PiA | PiC | PiB)."""

    def __init__(self, L, n=N, k=64, seed=0):
        import torch
        from gosnark_b200._lib import check
        from gosnark_b200.synthetic import CircuitGroth16, SyntheticCircuit
        self.syn = CircuitGroth16(n=n)
        self.pk = self.syn.load_pk()
        cs = [SyntheticCircuit(n, seed=0x5EED + 131 * seed + p) for p in range(k)]
        self.pubs = [c.public_signals for c in cs]
        rng = random.Random(seed)
        rs, ss = [rng.randrange(1, R) for _ in range(k)], [rng.randrange(1, R) for _ in range(k)]
        d_w = to_dev(limbs([v for c in cs for v in c.witness]))
        self.d_out = torch.zeros(48 * k, dtype=torch.int64, device="cuda")
        check(L.b200_groth16_prove_witness_batch_device(self.pk, self.syn.r1cs.handle, d_w.data_ptr(), self.syn.m, k,
                                                        _p(limbs(rs)), _p(limbs(ss)), self.d_out.data_ptr(), None))
        torch.cuda.synchronize()
        self.words = self.d_out.cpu().numpy().view(np.uint64).reshape(k, 48).copy()
        self.d_pub = to_dev(limbs([s for ps in self.pubs for s in ps]))
        self.vk = self.syn.vk_limbs()
        self.npub = len(self.pubs[0])


@pytest.fixture(scope="module")
def batch(L):
    b = Batch(L)
    yield b
    L.b200_pk_free(b.pk)


def split(words):
    words = np.ascontiguousarray(words, dtype=np.uint64).reshape(-1, 48)
    return (np.ascontiguousarray(words[:, :12]), np.ascontiguousarray(words[:, 24:48]), np.ascontiguousarray(words[:, 12:24]))


def vb_host(L, vk, words, pubs, rho, npub=None):
    """b200_groth16_verify_batch -> (rc, verdicts, status)."""
    ic, a1, b2, g2, d2 = vk
    k = len(words)
    npub = len(pubs[0]) if npub is None else npub
    pa, pb, pc = split(words)
    pub = limbs([s for ps in pubs for s in ps]) if npub else np.zeros((1, 4), np.uint64)
    ok = np.full(k, -1, np.int32)
    st = ctypes.c_uint32(0)
    rc = L.b200_groth16_verify_batch(_p(ic), ic.shape[0] if ic.ndim > 1 else len(ic) // 12, _p(a1), _p(b2), _p(g2), _p(d2),
                                     _p(pa), _p(pb), _p(pc), _p(pub), npub, k, _p(rho_limbs(rho)), _p(ok), ctypes.byref(st))
    return rc, [int(v) for v in ok], st.value


def vb_dev(L, vk, d_proofs, d_pub, npub, k, rho):
    """b200_groth16_verify_batch_device on device tensors -> (rc, verdicts, status)."""
    import torch
    ic, a1, b2, g2, d2 = vk
    d_ok = torch.full((k + 1,), -1, dtype=torch.int32, device="cuda")
    rc = L.b200_groth16_verify_batch_device(_p(ic), ic.shape[0] if ic.ndim > 1 else len(ic) // 12, _p(a1), _p(b2), _p(g2),
                                            _p(d2), d_proofs.data_ptr(), d_pub.data_ptr(), npub, k, _p(rho_limbs(rho)),
                                            d_ok.data_ptr(), None)
    torch.cuda.synchronize()
    out = d_ok.cpu().numpy()
    return rc, [int(v) for v in out[:k]], int(out[k].view(np.uint32))


def single(L, vk, words, pub):
    """b200_groth16_verify on one proof -> verdict (or the error code, negative)."""
    ic, a1, b2, g2, d2 = vk
    pa, pb, pc = split(words)
    ok = ctypes.c_int(-1)
    rc = L.b200_groth16_verify(_p(ic), ic.shape[0] if ic.ndim > 1 else len(ic) // 12, _p(a1), _p(b2), _p(g2), _p(d2), _p(pa),
                               _p(pb), _p(pc), _p(limbs(pub)), len(pub), ctypes.byref(ok))
    return ok.value if rc == 0 else rc


def rhos(k, seed=1):
    rng = random.Random(seed)
    return [rng.randrange(1, 1 << 128) for _ in range(k)]


def ints(words):
    raw = np.ascontiguousarray(words, dtype=np.uint64).tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


def words_of(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy()


def set_g1(words, off, p):
    words[off:off + 12] = words_of(list(p))


def get_g1(words, off):
    return tuple(ints(words[off:off + 12]))


@pytest.fixture
def kernel(L, request):
    from gosnark_b200 import _lib
    from gosnark_b200._lib import check
    check(L.b200_config(_lib.CFG_PAIRING_KERNEL, request.param))
    yield request.param
    check(L.b200_config(_lib.CFG_PAIRING_KERNEL, 0))


@pytest.mark.parametrize("kernel", [0, 1, 2], indirect=True)
@pytest.mark.parametrize("k", [1, 2, 7, 64])
def test_valid_batches_aggregate_only(L, batch, kernel, k):
    rho = rhos(k, seed=k)
    rc, ok, st = vb_host(L, batch.vk, batch.words[:k], batch.pubs[:k], rho)
    assert rc == 0 and ok == [1] * k and st == 1
    # the prover's d_out, with no host copy in between
    rc, ok, st = vb_dev(L, batch.vk, batch.d_out, batch.d_pub, batch.npub, k, rho)
    assert rc == 0 and ok == [1] * k and st == 1


@pytest.mark.timeout(900)
def test_4096_tiled(L, batch):
    import torch
    k = 4096
    words = np.tile(batch.words, (k // 64, 1))
    pubs = batch.pubs * (k // 64)
    rho = rhos(k, seed=4096)
    rc, ok, st = vb_host(L, batch.vk, words, pubs, rho)
    assert rc == 0 and ok == [1] * k and st == 1
    d_proofs = batch.d_out.view(64, 48).repeat(k // 64, 1).reshape(-1).contiguous()
    d_pub = batch.d_pub.view(64, -1).repeat(k // 64, 1).reshape(-1).contiguous()
    torch.cuda.synchronize()
    rc, ok, st = vb_dev(L, batch.vk, d_proofs, d_pub, batch.npub, k, rho)
    assert rc == 0 and ok == [1] * k and st == 1


@pytest.fixture(scope="module")
def other(L):
    b = Batch(L, n=N // 2, k=2, seed=5)   # another circuit size: another key
    yield b
    L.b200_pk_free(b.pk)


def corrupt(kind, batch, other, p):
    """(words, pubs) of the first 7 proofs with proof p corrupted."""
    words = batch.words[:7].copy()
    pubs = [list(ps) for ps in batch.pubs[:7]]
    if kind == "A + G":
        set_g1(words[p], 0, G1.add(get_g1(words[p], 0), G1.G))
    elif kind == "B of another proof":
        words[p, 24:48] = batch.words[(p + 1) % 7, 24:48]
    elif kind == "C changed":
        set_g1(words[p], 12, G1.double(get_g1(words[p], 12)))
    elif kind == "wrong public signal":
        pubs[p][0] = (pubs[p][0] + 1) % R
    else:   # a proof under another key
        words[p] = other.words[0]
        pubs[p] = list(other.pubs[0])
    return words, pubs


@pytest.mark.parametrize("kind", ["A + G", "B of another proof", "C changed", "wrong public signal", "another key"])
def test_one_corrupted_proof(L, batch, other, kind):
    for p in (0, 3, 6):
        words, pubs = corrupt(kind, batch, other, p)
        rc, ok, st = vb_host(L, batch.vk, words, pubs, rhos(7, seed=p))
        assert rc == 0
        assert ok == [0 if i == p else 1 for i in range(7)], (kind, p)
        assert ok == [single(L, batch.vk, words[i], pubs[i]) for i in range(7)], (kind, p)
        assert st & 2 and not st & 1, (kind, p, st)


def test_cancelling_pair_needs_random_rho(L, batch):
    d = G1.mul_scalar(G1.G, 0xC0FFEE)
    words = batch.words[:4].copy()
    set_g1(words[0], 12, G1.add(get_g1(words[0], 12), d))
    set_g1(words[2], 12, G1.add(get_g1(words[2], 12), G1.neg(d)))
    pubs = batch.pubs[:4]
    assert [single(L, batch.vk, words[i], pubs[i]) for i in range(4)] == [0, 1, 0, 1]
    rc, ok, st = vb_host(L, batch.vk, words, pubs, [1, 1, 1, 1])
    assert rc == 0 and ok == [1, 1, 1, 1] and st == 1           # rho = (1, 1): the errors cancel
    rc, ok, st = vb_host(L, batch.vk, words, pubs, rhos(4, seed=77))
    assert rc == 0 and ok == [0, 1, 0, 1] and st & 2 and not st & 1


def fq_sqrt(a):
    s = pow(a, (Q + 1) // 4, Q)
    return s if s * s % Q == a % Q else None


def twist_point(rng):
    """(x, y, 1) on the twist for a random x (F_q^2 square root): off the order-r subgroup."""
    F2 = o.BN.Fq2
    while True:
        x = (rng.randrange(Q), rng.randrange(Q))
        a0, a1 = F2.add(F2.mul(F2.square(x), x), o.BN.twist_coef_b)
        t = fq_sqrt((a0 * a0 + a1 * a1) % Q)
        if t is None:
            continue
        for tt in (t, Q - t):
            y0 = fq_sqrt((a0 + tt) * pow(2, -1, Q) % Q)
            if y0:
                y = (y0, a1 * pow(2 * y0, -1, Q) % Q)
                if F2.square(y) == (a0, a1):
                    return (x, y, (1, 0))


def test_irregular_proofs_get_the_single_verdict(L, batch):
    rng = random.Random(3)
    k_ic = batch.syn.k_ic
    s_inf = (-k_ic[0]) * pow(k_ic[1], -1, R) % R             # IC[0] + s IC[1] = O
    cases = {
        "A at infinity": lambda w, ps: set_g1(w, 0, (0, 0, 0)),
        "C at infinity": lambda w, ps: set_g1(w, 12, (1, 1, 0)),
        "A off the curve": lambda w, ps: set_g1(w, 0, (1, 3, 1)),
        "B off the subgroup": lambda w, ps: w.__setitem__(slice(24, 48), words_of([c for xy in twist_point(rng) for c in xy])),
        "icPubl at infinity": lambda w, ps: ps.__setitem__(0, s_inf),
    }
    for name, mk in cases.items():
        words = batch.words[:5].copy()
        pubs = [list(ps) for ps in batch.pubs[:5]]
        mk(words[2], pubs[2])
        want = [single(L, batch.vk, words[i], pubs[i]) for i in range(5)]
        rc, ok, st = vb_host(L, batch.vk, words, pubs, rhos(5))
        assert rc == 0 and ok == want and want[:2] == [1, 1], name
        assert st & 4 and st & 2 and st & 1, (name, st)
        rc, ok2, st2 = vb_dev(L, batch.vk, to_dev(words), to_dev(limbs([s for ps in pubs for s in ps])), batch.npub, 5, rhos(5))
        assert rc == 0 and ok2 == want and st2 == st, name


def test_errors(L, batch):
    import torch
    words = batch.words[:3].copy()
    pubs = batch.pubs[:3]
    rho = rhos(3)
    inf_b = words.copy()
    inf_b[1, 40:48] = 0
    big = words.copy()
    big[2, 0:4] = words_of([Q])
    assert vb_host(L, batch.vk, inf_b, pubs, rho)[0] == EINVAL
    assert vb_host(L, batch.vk, big, pubs, rho)[0] == ERANGE
    assert vb_host(L, batch.vk, words, [pubs[0], [R], pubs[2]], rho)[0] == ERANGE
    assert vb_host(L, batch.vk, words, pubs, [rho[0], 0, rho[2]])[0] == EINVAL
    ic, a1, b2, g2, d2 = batch.vk
    ok = np.zeros(1, np.int32)
    assert L.b200_groth16_verify_batch(_p(ic), 2, _p(a1), _p(b2), _p(g2), _p(d2), _p(words), _p(words), _p(words),
                                       _p(limbs([1])), 1, 0, _p(rho_limbs(rho)), _p(ok), None) == EINVAL
    assert vb_host(L, (ic[:1],) + batch.vk[1:], words, pubs, rho)[0] == EINVAL           # n_ic < n_public + 1
    # the device entry: per-proof zeros and status bit 3, no error code, and nothing leaks into the next call
    for bad_words, bad_pubs in ((big, pubs), (words, [pubs[0], pubs[1], [R]])):
        rc, ok, st = vb_dev(L, batch.vk, to_dev(bad_words), to_dev(limbs([s for ps in bad_pubs for s in ps])), 1, 3, rho)
        assert rc == 0 and ok == [1, 1, 0] and st & 8 and st & 4 and st & 1
    rc, ok, st = vb_dev(L, batch.vk, to_dev(inf_b), to_dev(limbs([s for ps in pubs for s in ps])), 1, 3, rho)
    assert rc == 0 and ok == [1, 0, 1] and not st & 8
    rc, ok, st = vb_host(L, batch.vk, words, pubs, rho)
    assert rc == 0 and ok == [1, 1, 1] and st == 1
    d = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert L.b200_groth16_verify_batch_device(_p(ic), 2, _p(a1), _p(b2), _p(g2), _p(d2), None, None, 1, 3,
                                              _p(rho_limbs(rho)), d.data_ptr(), None) == EINVAL


def _launches(L, fn):
    from gosnark_b200._lib import check
    out = (ctypes.c_double * 8)()
    check(L.b200_profile_read(out))
    fn()
    check(L.b200_profile_read(out))
    return int(out[6])


def test_launch_count_fixed(L, batch):
    bad = batch.words[:7].copy()
    set_g1(bad[3], 0, G1.add(get_g1(bad[3], 0), G1.G))
    counts = {k: _launches(L, lambda: vb_host(L, batch.vk, batch.words[:k], batch.pubs[:k], rhos(k))) for k in (1, 7, 64)}
    counts["failing"] = _launches(L, lambda: vb_host(L, batch.vk, bad, batch.pubs[:7], rhos(7)))
    counts["device"] = _launches(L, lambda: vb_dev(L, batch.vk, batch.d_out, batch.d_pub, batch.npub, 64, rhos(64)))
    assert len(set(counts.values())) == 1 and counts[1] == 9, counts


def test_reproducible(L, batch, other):
    words, pubs = corrupt("C changed", batch, other, 3)
    first = vb_host(L, batch.vk, words, pubs, rhos(7, seed=9))
    assert vb_host(L, batch.vk, words, pubs, rhos(7, seed=9)) == first


def test_python_entries(L, batch):
    from gosnark_b200 import groth16
    from gosnark_b200.bn128 import _unflatten_g1, _unflatten_g2
    ic, a1, b2, g2, d2 = batch.vk
    vk = {"IC": _unflatten_g1(ic), "G1": {"Alpha": _unflatten_g1(a1)[0]},
          "G2": {"Beta": _unflatten_g2(b2)[0], "Gamma": _unflatten_g2(g2)[0], "Delta": _unflatten_g2(d2)[0]}}
    proofs = []
    for w in batch.words[:5]:
        pa, pc = _unflatten_g1(w[:24])
        proofs.append({"PiA": pa, "PiB": _unflatten_g2(w[24:48])[0], "PiC": pc})
    proofs[1] = dict(proofs[1], PiC=proofs[2]["PiC"])
    assert groth16.VerifyProofBatch(vk, proofs, batch.pubs[:5]) == [True, False, True, True, True]
    d_ok = groth16.VerifyProofBatchDevice(vk, batch.d_out, batch.d_pub, 5, batch.npub)
    import torch
    torch.cuda.synchronize()
    assert d_ok.cpu().tolist() == [1] * 5 + [1]
