"""CPU: the batched Pinocchio verifier's kernels (csrc/verify_batch_pinocchio.cuh) over emulated CTAs
(tests/host/pinocchio_verify_batch_test.cpp, csrc/host_stub), on keys and proofs with known discrete logs
(oracle/make_verify_golden.py) minted by the oracle.

- The aggregate, kernel by kernel in the library's order with fixed rho: a valid batch passes; a proof that breaks exactly
  one of the five checks fails it, for each check; two proofs breaking the same check by +d and -d pass only under rho = 1.
- S_i and T_i are the reference's sums (its order, its Add) as group elements; Vkx == PiA makes the proof irregular.
- k_pvb_classify: each G1 point at infinity or off the curve, PiB off the subgroup, a Vk point off its group, coordinates
  >= q, PiB at infinity."""
import ctypes
import random

import numpy as np
import pytest

import build as b200build
from oracle import make_verify_golden as mvg
from oracle import ref_py as o

G1, G2 = o.BN.G1, o.BN.G2
R, Q = o.R, o.Q
ORDER = ("PiA", "PiAp", "PiBp", "PiC", "PiCp", "PiH", "PiKp")
VK_G1, VK_G2 = ("Vkb", "G1Kbg"), ("Vka", "Vkc", "G2Kbg", "G2Kg", "Vkz")


@pytest.fixture(scope="module")
def lib():
    return ctypes.CDLL(b200build.build_host_pinocchio_verify_batch())


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def u64(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).copy()


def g1w(p):
    return [p[0], p[1], p[2]]


def g2w(p):
    return [p[0][0], p[0][1], p[1][0], p[1][1], p[2][0], p[2][1]]


_mint = {}


def mint(group, k):
    key = (group, k % R)
    if key not in _mint:
        G = G1 if group == 1 else G2
        _mint[key] = G.mul_scalar(G.G, k % R)
    return _mint[key]


KEY_SEED = 31


def proof_logs(ic, pubs, a):
    """A valid proof's logs under the key of KEY_SEED: pinocchio_logs draws the key's logs (and PiB, PiH) from the same
    seed every time, so proofs with different PiA share one key."""
    vk, pr = mvg.pinocchio_logs(random.Random(KEY_SEED), ic, a, mvg.ref_add(mvg.ic_sum(ic, pubs), a))
    assert mvg.pinocchio_failed_check(vk, pr, pubs) == 0
    return vk, pr


def points(vk, pr):
    """Oracle points of a proof's logs (0 = infinity is never drawn here)."""
    p = {k: mint(1, v) for k, v in pr.items() if k != "PiB"}
    p["PiB"] = mint(2, pr["PiB"])
    return p


def vk_words(vk, overrides=None):
    pts = {k: mint(1, vk[k]) for k in VK_G1}
    pts.update({k: mint(2, vk[k]) for k in VK_G2})
    pts.update(overrides or {})
    return u64([w for k in VK_G1 for w in g1w(pts[k])] + [w for k in VK_G2 for w in g2w(pts[k])] + g2w(G2.G))


def ic_words(vk):
    return u64([w for k in vk["IC"] for w in g1w(mint(1, k))])


def proof_words(proofs):
    return u64([w for p in proofs for w in [c for s in ORDER for c in g1w(p[s])] + g2w(p["PiB"])])


def rho_limbs(rho):
    return np.array([w for r in rho for w in (r & (2**64 - 1), r >> 64)], dtype=np.uint64)


def aggregate(lib, vk, proofs, pubs, rho, warp=False, vkw=None):
    k, npub = len(proofs), len(pubs[0])
    flags = np.zeros(k + 1, np.uint32)
    st = np.zeros(24 * k, np.uint64)
    agg, status = ctypes.c_uint32(0), ctypes.c_uint32(0)
    pub = u64([s for ps in pubs for s in ps]) if npub else np.zeros(4, np.uint64)
    k_reg = lib.t_pvb_aggregate(_p(ic_words(vk)), _p(vk_words(vk) if vkw is None else vkw), _p(proof_words(proofs)), _p(pub),
                                npub, k, _p(rho_limbs(rho)), int(warp), _p(flags), _p(st), ctypes.byref(agg),
                                ctypes.byref(status))
    return k_reg, agg.value, status.value, list(flags), st


def classify(lib, proofs, vkw):
    k = len(proofs)
    flags = np.zeros(k + 1, np.uint32)
    st = ctypes.c_uint32(0)
    assert lib.t_pvb_classify(_p(proof_words(proofs)), _p(vkw), k, _p(flags), ctypes.byref(st)) == 0
    return list(flags), st.value


def rhos(k, seed=1):
    rng = random.Random(seed)
    return [rng.randrange(1, 1 << 128) for _ in range(5 * k)]


@pytest.fixture(scope="module")
def batch():
    """Three valid proofs under one key with two public signals."""
    rng = random.Random(32)
    ic = [rng.randrange(1, R) for _ in range(3)]
    pubs = [[rng.randrange(R), rng.randrange(R)] for _ in range(3)]
    logs = [proof_logs(ic, ps, rng.randrange(1, R)) for ps in pubs]
    vk = logs[0][0]
    return vk, [pr for _, pr in logs], [points(vk, pr) for _, pr in logs], pubs


def test_valid_batch_passes(lib, batch):
    vk, _, proofs, pubs = batch
    k_reg, agg, status, flags, _ = aggregate(lib, vk, proofs, pubs, rhos(3))
    assert (k_reg, agg, status, flags) == (3, 1, 1, [0, 0, 0, 0])


def test_valid_batch_warp_miller(lib, batch):
    vk, _, proofs, pubs = batch
    assert aggregate(lib, vk, proofs[:1], pubs[:1], rhos(1), warp=True)[:3] == (1, 1, 1)


@pytest.mark.parametrize("check,key", list(enumerate(("PiAp", "PiBp", "PiCp", "PiH", "PiKp"), start=1)))
def test_each_broken_check_fails_the_aggregate(lib, batch, check, key):
    vk, logs, proofs, pubs = batch
    bad = dict(logs[1], **{key: (logs[1][key] + 1) % R})
    assert mvg.pinocchio_failed_check(vk, bad, pubs[1]) == check
    ps = list(proofs)
    ps[1] = points(vk, bad)
    assert aggregate(lib, vk, ps, pubs, rhos(3, seed=check))[:4] == (3, 0, 0, [0, 0, 0, 0])


@pytest.mark.parametrize("key", ["PiAp", "PiH"])
def test_cancelling_pair_needs_random_rho(lib, batch, key):
    vk, logs, proofs, pubs = batch
    d = 0xC0FFEE
    ps = list(proofs)
    ps[0] = points(vk, dict(logs[0], **{key: (logs[0][key] + d) % R}))
    ps[2] = points(vk, dict(logs[2], **{key: (logs[2][key] - d) % R}))
    assert aggregate(lib, vk, ps, pubs, [1] * 15)[:3] == (3, 1, 1)
    assert aggregate(lib, vk, ps, pubs, rhos(3))[:3] == (3, 0, 0)


def _affine_words(st, off):
    raw = st.tobytes()
    return G1.affine(tuple(int.from_bytes(raw[32 * (off + j):32 * (off + j + 1)], "little") for j in range(3)))


def test_s_and_t_are_the_reference_sums(lib, batch):
    vk, logs, proofs, pubs = batch
    st = aggregate(lib, vk, proofs, pubs, rhos(3))[4]
    for i, (pr, ps) in enumerate(zip(logs, pubs)):
        s = mvg.ref_add(mvg.ic_sum(vk["IC"], ps), pr["PiA"])
        t = mvg.ref_add(s, pr["PiC"])
        assert _affine_words(st, 6 * i) == G1.affine(mint(1, s)), i
        assert _affine_words(st, 6 * i + 3) == G1.affine(mint(1, t)), i


def test_vkx_equal_to_pia_is_irregular(lib, batch):
    """Vkx == PiA: the reference's Add gives S = infinity, paired as (0, 0); the proof stays out of the aggregate."""
    vk, logs, proofs, pubs = batch
    a = mvg.ic_sum(vk["IC"], pubs[1])
    v2, pr = proof_logs(vk["IC"], pubs[1], a)
    assert v2 == vk and mvg.ref_add(a, pr["PiA"]) == 0
    ps = list(proofs)
    ps[1] = points(vk, pr)
    k_reg, agg, status, flags, st = aggregate(lib, vk, ps, pubs, rhos(3))
    assert flags == [0, 1, 0, 0] and (k_reg, agg, status) == (2, 1, 1 | 4)
    assert np.all(st[24 + 8:24 + 12] == 0)          # S_1's Z


def twist_point(rng):
    """(x, y, 1) on the twist for a random x: almost never in G2."""
    F2 = o.BN.Fq2
    while True:
        x = (rng.randrange(Q), rng.randrange(Q))
        a0, a1 = F2.add(F2.mul(F2.square(x), x), o.BN.twist_coef_b)
        t = pow((a0 * a0 + a1 * a1) % Q, (Q + 1) // 4, Q)
        if t * t % Q != (a0 * a0 + a1 * a1) % Q:
            continue
        for tt in (t, Q - t):
            y0 = pow((a0 + tt) * pow(2, -1, Q) % Q, (Q + 1) // 4, Q)
            if y0 and y0 * y0 % Q == (a0 + tt) * pow(2, -1, Q) % Q:
                y = (y0, a1 * pow(2 * y0, -1, Q) % Q)
                if F2.square(y) == (a0, a1):
                    return (x, y, (1, 0))


def test_classification(lib, batch):
    vk, _, proofs, pubs = batch
    vkw = vk_words(vk)
    assert classify(lib, proofs, vkw) == ([0, 0, 0, 0], 0)
    for s in ORDER:
        for name, pt in (("infinity", (1, 1, 0)), ("off the curve", (1, 3, 1))):
            ps = list(proofs)
            ps[1] = dict(ps[1], **{s: pt})
            assert classify(lib, ps, vkw) == ([0, 1, 0, 0], 4), (s, name)
    rng = random.Random(33)
    ps = list(proofs)
    ps[2] = dict(ps[2], PiB=twist_point(rng))
    assert classify(lib, ps, vkw) == ([0, 0, 1, 0], 4)
    assert aggregate(lib, vk, ps, pubs, rhos(3))[:4] == (2, 1, 1 | 4, [0, 0, 1, 0])
    # a coordinate >= q and PiB at infinity: bad (verdict 0 without a pairing)
    ps = list(proofs)
    ps[0] = dict(ps[0], PiH=(Q, 1, 1))
    ps[2] = dict(ps[2], PiB=((1, 0), (1, 0), (0, 0)))
    assert classify(lib, ps, vkw) == ([3, 0, 3, 0], 4 | 8)
    # a Vk point off its group: nothing aggregated
    for key in VK_G2:
        bad_vk = vk_words(vk, {key: twist_point(rng)})
        assert classify(lib, proofs, bad_vk) == ([0, 0, 0, 1], 4), key
    assert classify(lib, proofs, vk_words(vk, {"G1Kbg": (1, 3, 1)})) == ([0, 0, 0, 1], 4)
    assert aggregate(lib, vk, proofs, pubs, rhos(3), vkw=vk_words(vk, {"Vkz": twist_point(rng)}))[:3] == (0, 0, 4)
