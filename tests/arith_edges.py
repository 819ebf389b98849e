"""The edge operands of the field arithmetic, shared by the CPU vehicle (tests/test_host_arith.py) and the device vehicle
(tests/test_gpu_arith.py) so that both run the same vectors.

The kernels work on Montgomery representatives x * 2^256 mod p, not on x: a value that is an edge in standard form is a
random-looking word pattern in the limbs the carry chains see.  So every edge value e comes twice: once as itself, and
once as e * 2^-256 mod p, whose Montgomery representative IS e.  The second set is what puts 0, p - 1, all-ones limbs and
2^(32k) +- 1 into the carry chains of add, sub, the CIOS product, the wide product and the wide reduction."""

MASK32 = 0xffffffff


def base_edges(p):
    """Edge values in [0, p) as standard-form integers."""
    v = [0, 1, 2, 3, p - 1, p - 2, p - 3, (p - 1) // 2, (p + 1) // 2, (1 << 253), (1 << 254) - 1, (1 << 255), (1 << 256) - 1]
    for k in range(8):
        v += [(1 << (32 * k)) + 1, (1 << (32 * k)) - 1, 1 << (32 * k), p - (1 << (32 * k))]
        v.append(MASK32 << (32 * k))                  # one all-ones limb
        v.append((1 << (32 * (k + 1))) - 1)           # the k + 1 lowest limbs all ones
        v.append(((1 << 256) - 1) ^ (MASK32 << (32 * k)))   # all limbs all ones but one
    return [x % p for x in v]


def montgomery_preimages(p, vals):
    """x * 2^-256 mod p for each x: the values whose Montgomery representatives are vals."""
    rinv = pow(1 << 256, -1, p)
    return [x * rinv % p for x in vals]


def edges(p):
    """Sorted, de-duplicated edge set of modulus p: the base edges and their Montgomery preimages."""
    b = base_edges(p)
    return sorted(set(b) | set(montgomery_preimages(p, b)))


def wide_edges():
    """Edge operands of the raw 256 x 256 -> 512-bit product (no modulus): carries through every limb boundary."""
    M = (1 << 256) - 1
    H = (1 << 128) - 1
    v = [0, 1, 2, M, M - 1, H, H << 128, 1 << 128, 1 << 255, (H << 128) | 1, MASK32, MASK32 << 96,
         sum(MASK32 << (64 * i) for i in range(4)), sum(MASK32 << (64 * i + 32) for i in range(4))]
    for k in range(8):
        v += [(1 << (32 * k)) - 1, 1 << (32 * k), M ^ (MASK32 << (32 * k)), M >> (32 * k), (M << (32 * k)) & M]
    return sorted(set(v))


def redc_edges(p):
    """Edge inputs t of the wide Montgomery reduction t -> t / 2^256 mod p, all < p * 2^256 (its stated bound)."""
    top = p * (1 << 256)
    v = [0, 1, top - 1, top - 2, top - (1 << 256), (1 << 256) - 1, (1 << 256), (p - 1) * (p - 1), ((1 << 256) - 1) * (p - 1),
         p << 255, 2 * p * p - 1, 2 * p * p, p * p, p * p - 1, (p - 1) << 256, ((p - 1) << 256) | ((1 << 256) - 1)]
    for k in range(16):
        v += [(1 << (32 * (k + 1))) - 1, top - (1 << (32 * k)), top - 1 - (MASK32 << (32 * k))]
    return sorted(set(x for x in v if 0 <= x < top))
