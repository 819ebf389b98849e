"""GPU: batched Pinocchio verification (include/b200snark.h: b200_pinocchio_verify_batch, b200_pinocchio_verify_batch_device)
on proofs made by the batch prover under a real key (synthetic.CircuitPinocchio) and on proofs with known discrete logs.
Every verdict that the contract ties to the per-proof path is compared with snark.VerifyProof on that proof."""
import ctypes
import random

import numpy as np
import pytest

from oracle import make_verify_golden as mvg
from oracle import ref_py as o
from test_gpu_pinocchio_batch import witnesses
from test_gpu_pinocchio_witness import EINVAL, ERANGE, ORDER, _launches, _p, limbs, split, to_dev

pytestmark = pytest.mark.gpu
G1, G2 = o.BN.G1, o.BN.G2
R, Q = o.R, o.Q
N = 1 << 10
W = 108                                   # u64 per proof: seven G1 points, then PiB
SLOT = {s: 12 * i for i, s in enumerate(ORDER)}


@pytest.fixture(scope="module")
def L():
    from gosnark_b200 import _lib
    _lib.init()
    return _lib.lib()


def vk_limbs(vk):
    """(ic, vk_g1, vk_g2) as b200_pinocchio_verify_batch takes them: one row of 12 (G1) or 24 (G2) words per point."""
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    return (_flatten_g1(vk["IC"]).reshape(-1, 12), _flatten_g1([vk["Vkb"], vk["G1Kbg"]]).reshape(-1, 12),
            _flatten_g2([vk["Vka"], vk["Vkc"], vk["G2Kbg"], vk["G2Kg"], vk["Vkz"]]).reshape(-1, 24))


class Batch:
    """k proofs of distinct satisfying witnesses of CircuitPinocchio(n), proved in one
    b200_pinocchio_prove_witness_batch_device call; ``d_out`` is the prover's output tensor, ``words`` its host copy."""

    def __init__(self, L, n=N, k=64, seed=0):
        from gosnark_b200.synthetic import CircuitPinocchio, SyntheticCircuit
        self.syn = CircuitPinocchio(n)
        self.pk = self.syn.load_pk()
        cs = [SyntheticCircuit(n, seed=0x91CC + 131 * seed + p) for p in range(k)]
        self.pubs = [c.public_signals for c in cs]
        self.d_out = self.prove(L, [c.witness for c in cs])
        self.words = self.d_out.cpu().numpy().view(np.uint64).reshape(k, W).copy()
        self.d_pub = to_dev(limbs([s for ps in self.pubs for s in ps]))
        self.vk = self.syn.vk
        self.vkl = vk_limbs(self.vk)
        self.npub = len(self.pubs[0])

    def prove(self, L, wits):
        import torch
        from gosnark_b200._lib import check
        k = len(wits)
        d_out = torch.zeros(W * k, dtype=torch.int64, device="cuda")
        check(L.b200_pinocchio_prove_witness_batch_device(self.pk, self.syn.r1cs.handle, to_dev(limbs([v for w in wits for v in w])).data_ptr(),
                                                          self.syn.m, k, d_out.data_ptr(), None))
        torch.cuda.synchronize()
        return d_out


@pytest.fixture(scope="module")
def batch(L):
    b = Batch(L)
    yield b
    L.b200_pk_free(b.pk)


@pytest.fixture(scope="module")
def other(L):
    b = Batch(L, n=N // 2, k=2, seed=5)   # another circuit size: another key
    yield b
    L.b200_pk_free(b.pk)


def rhos(k, seed=1):
    rng = random.Random(seed)
    return [rng.randrange(1, 1 << 128) for _ in range(5 * k)]


def rho_limbs(rho):
    return np.array([w for v in rho for w in (v & (2**64 - 1), v >> 64)], dtype=np.uint64)


def pvb_host(L, vkl, words, pubs, rho, npub=None):
    """b200_pinocchio_verify_batch -> (rc, verdicts, status)."""
    ic, g1, g2 = vkl
    words = np.ascontiguousarray(words, dtype=np.uint64).reshape(-1, W)
    k = len(words)
    npub = len(pubs[0]) if npub is None else npub
    out_g1, pb = np.ascontiguousarray(words[:, :84]), np.ascontiguousarray(words[:, 84:])
    pub = limbs([s for ps in pubs for s in ps]) if npub else np.zeros((1, 4), np.uint64)
    ok = np.full(k, -1, np.int32)
    st = ctypes.c_uint32(0)
    rc = L.b200_pinocchio_verify_batch(_p(ic), len(ic), _p(g1), _p(g2), _p(out_g1), _p(pb), _p(pub), npub, k,
                                       _p(rho_limbs(rho)), _p(ok), ctypes.byref(st))
    return rc, [int(v) for v in ok], st.value


def pvb_dev(L, vkl, d_proofs, d_pub, npub, k, rho):
    """b200_pinocchio_verify_batch_device on device tensors -> (rc, verdicts, status)."""
    import torch
    ic, g1, g2 = vkl
    d_ok = torch.full((k + 1,), -1, dtype=torch.int32, device="cuda")
    rc = L.b200_pinocchio_verify_batch_device(_p(ic), len(ic), _p(g1), _p(g2), d_proofs.data_ptr(), d_pub.data_ptr(), npub, k,
                                              _p(rho_limbs(rho)), d_ok.data_ptr(), None)
    torch.cuda.synchronize()
    out = d_ok.cpu().numpy()
    return rc, [int(v) for v in out[:k]], int(out[k].view(np.uint32))


def single(vk, words, pub):
    from gosnark_b200 import snark
    return int(snark.VerifyProof(vk, split(words), pub))


def ints(words):
    raw = np.ascontiguousarray(words, dtype=np.uint64).tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


def words_of(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy()


def set_g1(row, slot, p):
    row[SLOT[slot]:SLOT[slot] + 12] = words_of(list(p))


def get_g1(row, slot):
    return tuple(ints(row[SLOT[slot]:SLOT[slot] + 12]))


def get_b(row):
    v = ints(row[84:])
    return ((v[0], v[1]), (v[2], v[3]), (v[4], v[5]))


def set_b(row, q):
    row[84:] = words_of([c for xy in q for c in xy])


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
    rc, ok, st = pvb_host(L, batch.vkl, batch.words[:k], batch.pubs[:k], rho)
    assert rc == 0 and ok == [1] * k and st == 1
    # the prover's d_out, with no host copy in between
    rc, ok, st = pvb_dev(L, batch.vkl, batch.d_out, batch.d_pub, batch.npub, k, rho)
    assert rc == 0 and ok == [1] * k and st == 1


@pytest.mark.timeout(900)
def test_4096_tiled(L, batch):
    import torch
    k = 4096
    rho = rhos(k, seed=4096)
    rc, ok, st = pvb_host(L, batch.vkl, np.tile(batch.words, (k // 64, 1)), batch.pubs * (k // 64), rho)
    assert rc == 0 and ok == [1] * k and st == 1
    d_proofs = batch.d_out.view(64, W).repeat(k // 64, 1).reshape(-1).contiguous()
    d_pub = batch.d_pub.view(64, -1).repeat(k // 64, 1).reshape(-1).contiguous()
    torch.cuda.synchronize()
    rc, ok, st = pvb_dev(L, batch.vkl, d_proofs, d_pub, batch.npub, k, rho)
    assert rc == 0 and ok == [1] * k and st == 1


KINDS = [f"{s} + G" for s in ORDER] + ["PiB doubled", "PiB of another proof", "another key"]


def corrupt(kind, batch, other, p):
    """(words, pubs) of the first 7 proofs with proof p corrupted."""
    words = batch.words[:7].copy()
    pubs = [list(ps) for ps in batch.pubs[:7]]
    if kind.endswith(" + G"):
        s = kind.split()[0]
        set_g1(words[p], s, G1.add(get_g1(words[p], s), G1.G))
    elif kind == "PiB doubled":
        set_b(words[p], G2.double(get_b(words[p])))
    elif kind == "PiB of another proof":
        words[p, 84:] = batch.words[(p + 1) % 7, 84:]
    else:
        words[p] = other.words[0]
        pubs[p] = list(other.pubs[0])
    return words, pubs


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", KINDS)
def test_one_corrupted_proof(L, batch, other, kind):
    for p in (0, 3, 6):
        words, pubs = corrupt(kind, batch, other, p)
        rc, ok, st = pvb_host(L, batch.vkl, words, pubs, rhos(7, seed=p))
        assert rc == 0
        assert ok == [0 if i == p else 1 for i in range(7)], (kind, p)
        assert ok == [single(batch.vk, words[i], pubs[i]) for i in range(7)], (kind, p)
        assert st & 2 and not st & 1, (kind, p, st)
    rc, ok2, st2 = pvb_dev(L, batch.vkl, to_dev(words), to_dev(limbs([s for ps in pubs for s in ps])), 1, 7, rhos(7, seed=6))
    assert rc == 0 and ok2 == ok and st2 == st, kind


def test_unsatisfied_witnesses_rejected(L, batch):
    k = 12
    wits, sat = witnesses(batch.syn, k, seed=3)
    assert not all(sat)
    d_out = batch.prove(L, wits)
    words = d_out.cpu().numpy().view(np.uint64).reshape(k, W)
    pubs = [[w[1]] for w in wits]
    want = [single(batch.vk, words[i], pubs[i]) for i in range(k)]
    assert want == [int(s) for s in sat]
    rc, ok, st = pvb_host(L, batch.vkl, words, pubs, rhos(k))
    assert rc == 0 and ok == want and st & 2 and not st & 1
    rc, ok, st2 = pvb_dev(L, batch.vkl, d_out, to_dev(limbs([s for ps in pubs for s in ps])), 1, k, rhos(k))
    assert rc == 0 and ok == want and st2 == st


def test_wrong_public_signal_gets_the_reference_verdict(L, batch):
    """SyntheticCircuit's public signal has no A term, so IC[1] is infinity and the reference accepts a wrong signal: the
    batch must not be stricter."""
    words = batch.words[:4]
    pubs = [list(ps) for ps in batch.pubs[:4]]
    pubs[2][0] = (pubs[2][0] + 1) % R
    want = [single(batch.vk, words[i], pubs[i]) for i in range(4)]
    assert want == [1, 1, 1, 1]
    rc, ok, st = pvb_host(L, batch.vkl, words, pubs, rhos(4))
    assert rc == 0 and ok == want and st == 1


# ---- proofs with known discrete logs (oracle/make_verify_golden.py), minted on the GPU --------------------------------
def mint_logs(vk, pr):
    from gosnark_b200 import bn128
    g1, g2 = bn128.G1(), bn128.G2()
    m1 = lambda ks: g1.MulScalarBatch([g1.G], [int(x) % R for x in ks])
    m2 = lambda ks: g2.MulScalarBatch([g2.G], [int(x) % R for x in ks])
    g2k = [k for k in vk if k in mvg.G2_KEYS]
    g1k = [k for k in vk if k not in mvg.G2_KEYS and k != "IC"]
    pv = dict(zip(g2k, m2([vk[k] for k in g2k])))
    pv.update(zip(g1k, m1([vk[k] for k in g1k])))
    pv["IC"] = m1(vk["IC"])
    prk = [k for k in ORDER]
    pp = dict(zip(prk, m1([pr[k] for k in prk])))
    pp["PiB"] = m2([pr["PiB"]])[0]
    return pv, pp


def proof_words(proofs):
    from gosnark_b200.bn128 import _flatten_g1, _flatten_g2
    return np.stack([np.concatenate([_flatten_g1([p[s] for s in ORDER]).reshape(-1), _flatten_g2([p["PiB"]]).reshape(-1)])
                     for p in proofs])


KEY_SEED = 57


def logs_under_key(ic, pubs, a):
    """A proof's logs valid for the reference's sums, under the key KEY_SEED draws (pinocchio_logs draws the key's logs,
    and PiB, PiH, from the same seed each time, so proofs with different PiA share one key)."""
    return mvg.pinocchio_logs(random.Random(KEY_SEED), ic, a, mvg.ref_add(mvg.ic_sum(ic, pubs), a))


@pytest.mark.timeout(600)
def test_single_check_breakages_from_known_logs(L):
    from gosnark_b200 import snark
    rng = random.Random(58)
    r = lambda: rng.randrange(1, R)
    ic = [r(), r(), r()]
    proofs, pubs, want = [], [], []
    vk = None
    for c, key in enumerate(("PiAp", "PiBp", "PiCp", "PiH", "PiKp"), start=1):
        for broken in (False, True):
            ps = [r(), r()]
            vk, pr = logs_under_key(ic, ps, r())
            if broken:
                pr = dict(pr, **{key: (pr[key] + 1) % R})
            assert mvg.pinocchio_failed_check(vk, pr, ps) == (c if broken else 0)
            proofs.append(pr)
            pubs.append(ps)
            want.append(0 if broken else 1)
    pv = mint_logs(vk, proofs[0])[0]
    pts = [mint_logs(vk, pr)[1] for pr in proofs]
    assert [int(snark.VerifyProof(pv, p, ps)) for p, ps in zip(pts, pubs)] == want
    words = proof_words(pts)
    rc, ok, st = pvb_host(L, vk_limbs(pv), words, pubs, rhos(10))
    assert rc == 0 and ok == want and st & 2 and not st & 1
    assert snark.VerifyProofBatch(pv, pts, pubs) == [bool(v) for v in want]


def twist_point(rng):
    """(x, y, 1) on the twist for a random x (F_q^2 square root): off the order-r subgroup."""
    F2 = o.BN.Fq2
    sqrt = lambda a: (lambda s: s if s * s % Q == a % Q else None)(pow(a, (Q + 1) // 4, Q))
    while True:
        x = (rng.randrange(Q), rng.randrange(Q))
        a0, a1 = F2.add(F2.mul(F2.square(x), x), o.BN.twist_coef_b)
        t = sqrt((a0 * a0 + a1 * a1) % Q)
        if t is None:
            continue
        for tt in (t, Q - t):
            y0 = sqrt((a0 + tt) * pow(2, -1, Q) % Q)
            if y0:
                y = (y0, a1 * pow(2 * y0, -1, Q) % Q)
                if F2.square(y) == (a0, a1):
                    return (x, y, (1, 0))


@pytest.mark.timeout(600)
def test_irregular_proofs_get_the_reference_verdict(L, batch):
    rng = random.Random(3)
    cases = {
        "PiA at infinity": lambda w: set_g1(w, "PiA", (0, 0, 0)),
        "PiH at infinity": lambda w: set_g1(w, "PiH", (1, 1, 0)),
        "PiCp off the curve": lambda w: set_g1(w, "PiCp", (1, 3, 1)),
        "PiB off the subgroup": lambda w: set_b(w, twist_point(rng)),
    }
    for name, mk in cases.items():
        words = batch.words[:5].copy()
        pubs = batch.pubs[:5]
        mk(words[2])
        want = [single(batch.vk, words[i], pubs[i]) for i in range(5)]
        rc, ok, st = pvb_host(L, batch.vkl, words, pubs, rhos(5))
        assert rc == 0 and ok == want and want[:2] == [1, 1], name
        assert st & 4 and st & 2 and st & 1, (name, st)
        rc, ok2, st2 = pvb_dev(L, batch.vkl, to_dev(words), batch.d_pub, batch.npub, 5, rhos(5))
        assert rc == 0 and ok2 == want and st2 == st, name


@pytest.mark.timeout(600)
def test_reference_sums_vkx_equal_to_pia_and_signal_r_plus_2(L):
    """Vkx == PiA (S is infinity by the reference's Add) and a public signal of r + 2, each with a proof valid for the
    reference's sums and one valid for the mathematical sums, beside valid proofs: verdicts equal snark.VerifyProof's
    (through the Python entries, which reduce the signal as VerifyProof does), host and device agree."""
    import torch
    from gosnark_b200 import snark
    from gosnark_b200.bn128 import reduce_scalar
    rng = random.Random(59)
    r = lambda: rng.randrange(1, R)
    ic = [r(), r()]
    rows = []
    for name, pubs, equal in (("Vkx==PiA", [r()], True), ("r+2", [R + 2], False)):
        vkx, vkx_m = mvg.ic_sum(ic, pubs), mvg.ic_sum_math(ic, pubs)
        a = vkx if equal else r()
        for which, vkx_a in (("model", mvg.ref_add(vkx, a)), ("math", (vkx_m + a) % R)):
            vk, pr = mvg.pinocchio_logs(random.Random(KEY_SEED), ic, a, vkx_a)
            rows.append((pubs, pr, int(mvg.pinocchio_failed_check(vk, pr, pubs) == 0)))
        ps = [r()]
        rows.append((ps, logs_under_key(ic, ps, r())[1], 1))
    pv = mint_logs(vk, rows[0][1])[0]
    pts = [mint_logs(vk, pr)[1] for _, pr, _ in rows]
    pubs = [ps for ps, _, _ in rows]
    want = [int(snark.VerifyProof(pv, p, ps)) for p, ps in zip(pts, pubs)]
    assert want == [w for _, _, w in rows] == [1, 0, 1, 1, 0, 1]
    ok, st = snark.verify_batch_limbs(pv, pts, pubs, rho=rhos(6))
    assert [int(v) for v in ok] == want and st & 4 and st & 2 and not st & 1
    d_proofs = to_dev(proof_words(pts))
    d_pub = to_dev(limbs([reduce_scalar(s) for ps in pubs for s in ps]))
    d_ok = snark.VerifyProofBatchDevice(pv, d_proofs, d_pub, 6, 1, rho=rhos(6))
    torch.cuda.synchronize()
    out = d_ok.cpu().numpy()
    assert list(out[:6]) == want and int(out[6].view(np.uint32)) == st


def test_errors(L, batch):
    import torch
    words = batch.words[:3].copy()
    pubs = batch.pubs[:3]
    rho = rhos(3)
    ic, g1, g2 = batch.vkl
    inf_b = words.copy()
    inf_b[1, 100:108] = 0
    big = words.copy()
    big[2, SLOT["PiH"]:SLOT["PiH"] + 4] = words_of([Q])
    assert pvb_host(L, batch.vkl, inf_b, pubs, rho)[0] == EINVAL
    assert pvb_host(L, batch.vkl, big, pubs, rho)[0] == ERANGE
    assert pvb_host(L, batch.vkl, words, [pubs[0], [R], pubs[2]], rho)[0] == ERANGE
    for c in range(5):
        zero = list(rho)
        zero[5 + c] = 0
        assert pvb_host(L, batch.vkl, words, pubs, zero)[0] == EINVAL, c
    bad_ic = ic.copy()
    bad_ic[0, 4:8] = words_of([Q])
    assert pvb_host(L, (bad_ic, g1, g2), words, pubs, rho)[0] == ERANGE
    bad_g1 = g1.copy()
    bad_g1[1, 0:4] = words_of([Q + 5])
    assert pvb_host(L, (ic, bad_g1, g2), words, pubs, rho)[0] == ERANGE
    bad_g2 = g2.copy()
    bad_g2[3, 8:12] = words_of([Q])
    assert pvb_host(L, (ic, g1, bad_g2), words, pubs, rho)[0] == ERANGE
    for c in range(5):
        inf_vk = g2.copy()
        inf_vk[c, 16:24] = 0
        assert pvb_host(L, (ic, g1, inf_vk), words, pubs, rho)[0] == EINVAL, c
    assert pvb_host(L, (ic[:1], g1, g2), words, pubs, rho)[0] == EINVAL           # n_ic < n_public + 1
    ok = np.zeros(1, np.int32)
    for k in (0, 65537):
        assert L.b200_pinocchio_verify_batch(_p(ic), 2, _p(g1), _p(g2), _p(words), _p(words), _p(limbs([1])), 1, k,
                                             _p(rho_limbs(rhos(1))), _p(ok), None) == EINVAL, k
    assert L.b200_pinocchio_verify_batch(_p(ic), 2, _p(g1), _p(g2), None, _p(words), _p(limbs([1])), 1, 1,
                                         _p(rho_limbs(rhos(1))), _p(ok), None) == EINVAL
    assert L.b200_pinocchio_verify_batch(_p(ic), 2, _p(g1), None, _p(words), _p(words), _p(limbs([1])), 1, 1,
                                         _p(rho_limbs(rhos(1))), _p(ok), None) == EINVAL
    # the device entry: per-proof zeros and status bit 3, no error code, and nothing leaks into the next call
    for bad_words, bad_pubs in ((big, pubs), (words, [pubs[0], pubs[1], [R]])):
        rc, ok, st = pvb_dev(L, batch.vkl, to_dev(bad_words), to_dev(limbs([s for ps in bad_pubs for s in ps])), 1, 3, rho)
        assert rc == 0 and ok == [1, 1, 0] and st & 8 and st & 4 and st & 1
    rc, ok, st = pvb_dev(L, batch.vkl, to_dev(inf_b), to_dev(limbs([s for ps in pubs for s in ps])), 1, 3, rho)
    assert rc == 0 and ok == [1, 0, 1] and not st & 8
    rc, ok, st = pvb_host(L, batch.vkl, words, pubs, rho)
    assert rc == 0 and ok == [1, 1, 1] and st == 1
    rc, ok, st = pvb_dev(L, batch.vkl, to_dev(words), to_dev(limbs([s for ps in pubs for s in ps])), 1, 3, rho)
    assert rc == 0 and ok == [1, 1, 1] and st == 1
    d = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert L.b200_pinocchio_verify_batch_device(_p(ic), 2, _p(g1), _p(g2), None, None, 1, 3, _p(rho_limbs(rho)), d.data_ptr(),
                                                None) == EINVAL


def test_launch_count_fixed(L, batch):
    bad = batch.words[:7].copy()
    set_g1(bad[3], "PiA", G1.add(get_g1(bad[3], "PiA"), G1.G))
    counts = {k: _launches(L, lambda: pvb_host(L, batch.vkl, batch.words[:k], batch.pubs[:k], rhos(k))) for k in (1, 7, 64)}
    counts["failing"] = _launches(L, lambda: pvb_host(L, batch.vkl, bad, batch.pubs[:7], rhos(7)))
    counts["device"] = _launches(L, lambda: pvb_dev(L, batch.vkl, batch.d_out, batch.d_pub, batch.npub, 64, rhos(64)))
    assert len(set(counts.values())) == 1 and counts[1] == 9, counts


def test_reproducible(L, batch, other):
    words, pubs = corrupt("PiC + G", batch, other, 3)
    first = pvb_host(L, batch.vkl, words, pubs, rhos(7, seed=9))
    assert pvb_host(L, batch.vkl, words, pubs, rhos(7, seed=9)) == first


def test_python_entries(L, batch):
    import torch
    from gosnark_b200 import snark
    proofs = [split(w) for w in batch.words[:5]]
    proofs[1] = dict(proofs[1], PiC=proofs[2]["PiC"])
    assert snark.VerifyProofBatch(batch.vk, proofs, batch.pubs[:5]) == [True, False, True, True, True]
    d_ok = snark.VerifyProofBatchDevice(batch.vk, batch.d_out, batch.d_pub, 5, batch.npub)
    torch.cuda.synchronize()
    assert d_ok.cpu().tolist() == [1] * 5 + [1]
