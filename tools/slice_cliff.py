#!/usr/bin/env python3
"""Stand-alone G1 MSM either side of the slice-size step of bases_create (development aid):
at c = 17 the mean bucket population crosses 192 at 838 861 terms — below it S = 16, above it S = 32."""
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from gosnark_b200 import _lib, bn128  # noqa: E402


def rand_scalars(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64) * 2 + rng.integers(0, 2, size=(n, 4), dtype=np.uint64)
    a[:, 3] &= np.uint64((1 << 61) - 1)       # < 2^253 < r
    return a


_lib.init(0)
L = _lib.lib()
sizes = [int(x) for x in sys.argv[1:]] or [700000, 832000, 838000, 845000, 891000]
nmax = max(sizes)
ks = rand_scalars(nmax, 4)
pts = np.zeros((nmax, 12), dtype=np.uint64)
_lib.check(L.b200_g1_mul_batch_bcast(_lib.ptr(bn128._flatten_g1([bn128.G1.G])), _lib.ptr(ks), nmax, _lib.ptr(pts)))
d_s = torch.from_numpy(rand_scalars(nmax, 5).view(np.int64)).cuda()
d_out = torch.zeros(64, dtype=torch.int64, device="cuda")
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
st = stream.cuda_stream
for n in sizes:
    h = _lib._h(0)
    _lib.check(L.b200_g1_bases_load(_lib.ptr(pts), n, 0, h))
    for _ in range(3):
        _lib.check(L.b200_msm_device(h.value, d_s.data_ptr(), n, 0, d_out.data_ptr(), st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        _lib.check(L.b200_msm_device(h.value, d_s.data_ptr(), n, 0, d_out.data_ptr(), st))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print(f"G1 MSM n={n}: {ms:.3f} ms  ({ms / n * 1e6:.3f} ns/term)")
    _lib.check(L.b200_bases_free(h.value))
