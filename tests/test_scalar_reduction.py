"""CPU: bn128.reduce_scalar, the scalar every Python entry point sends in place of a *big.Int, is the reference's
MulScalar as a group element (bn128/g1.go:140-155, g2.go:142-181).

MulScalar runs its double-and-add over every bit of |e| with an Add that has no doubling branch (SURVEY H6).  For
|e| >= r the accumulator can equal P just before an addition, and Add(P, P) is infinity.  So r + 2 is not 2: the
reference computes infinity there.  A public signal of r + 2 makes the reference accept a different proof than one
reduced mod r would.  The oracle's mul_scalar is the reference's own walk, so each value below is checked against it in
both groups, at a fixed point that is not the generator."""
import random

import pytest

from oracle import ref_py as o

R = o.R

CRAFTED = [R + 2, 2 * R + 5, 3 * R + 2, (R + 2) << 7, ((R + 2) << 7) + 93, (3 * R + 2) * 8 + 5, -(R + 2)]
PLAIN = [0, 1, 2, R - 1, R, R + 1, R + 3, 2 * R, (1 << 256) - 1, -1, -(R - 1), -R, -(R + 1), -((1 << 256) - 1)]


def _random_wide(n, seed=17):
    rng = random.Random(seed)
    return [rng.randrange(R, 1 << 256) for _ in range(n)] + [rng.randrange(1 << 256, 1 << 300) for _ in range(2)]


@pytest.fixture(scope="module")
def rs():
    from gosnark_b200.bn128 import reduce_scalar
    return reduce_scalar


@pytest.fixture(scope="module", params=[1, 2], ids=["G1", "G2"])
def group(request):
    g = o.BN.G1 if request.param == 1 else o.BN.G2
    return g, g.mul_scalar(g.G, 0x5eed_1234_5678_9abc_def0)


@pytest.mark.parametrize("e", CRAFTED + PLAIN + _random_wide(4),
                         ids=[f"crafted{i}" for i in range(len(CRAFTED))] + [f"plain{i}" for i in range(len(PLAIN))]
                         + [f"wide{i}" for i in range(6)])
def test_reduce_scalar_is_reference_mul_scalar(rs, group, e):
    g, p = group
    m = rs(e)
    assert 0 <= m < R
    assert g.equal(g.mul_scalar(p, m), g.mul_scalar(p, e)), (e, m)


def test_crafted_scalars_are_not_abs_mod_r(rs):
    """Each crafted value is one where |e| mod r names a different point than the reference's walk: a body of
    ``abs(e) % R`` fails here, and through the group comparison above."""
    for e in CRAFTED:
        assert rs(e) != abs(e) % R, e
    assert rs(R + 2) == 0 and rs(-(R + 2)) == 0 and rs(((R + 2) << 7) + 93) == 93


def test_below_r_is_identity_and_sign_is_dropped(rs):
    rng = random.Random(3)
    for e in [0, 1, R - 1] + [rng.randrange(R) for _ in range(200)]:
        assert rs(e) == e and rs(-e) == e
