// Trusted setup for a sparse R1CS of any size (b200_groth16_setup, b200_pinocchio_setup): groth16.GenerateTrustedSetup
// (groth16/groth16.go:94-222) and snark.GenerateTrustedSetup (snark.go:98-251) without the dense m x n polynomials.
//   1. at | bt | ct = A^T l(T) etc. on the device (qap_eval_at_enqueue), zt = Z(T) with Z = prod_{i=1..m-2}(x - i).
//   2. Every CRS scalar from them by one element-wise F_r kernel per protocol; the few Vk scalars are appended on the host,
//      so each group needs ONE fixed-base launch (fixed_base.cuh).
//   3. The points come back affine (x, y, 1), standard form, infinity all zero: the same group elements as the
//      reference's, not its Jacobian representatives.
// Included inside capi.cu's anonymous namespace (after qap_sparse_host.cuh and zero_poly_host).

// T^e by square and multiply (e < 2^32): every thread raises T to its own index, no serial chain over the powers.
__device__ __forceinline__ Fr fr_pow_u32(Fr b, uint32_t e) {
  Fr r = Fr::one();
  while (e) {
    if (e & 1) r = r * b;
    b = b.sqr();
    e >>= 1;
  }
  return r;
}

// ev = at | bt | ct (Montgomery, m each); all other arguments Montgomery.  Standard-form scalars:
//   g1 = At (m) | BACGamma (m) | BACDelta (m) | PowersTauDelta (m-1) | IC (npublic+1) | [Alpha, Beta, Delta: host]
//   g2 = BACGamma (m) | [Beta, Gamma, Delta: host]
__global__ void k_groth16_setup_scalars(const Fr* __restrict__ ev, uint32_t m, uint32_t npublic, Fr ka, Fr kb, Fr inv_d,
                                        Fr inv_g, Fr zt_d, Fr t, Fr* __restrict__ g1, Fr* __restrict__ g2) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  Fr at = ev[i], bt = ev[m + i], ct = ev[2 * m + i];
  Fr v = kb * at + ka * bt + ct;                                    // groth16.go:181-219
  g1[i] = at.from_mont();
  g1[m + i] = g2[i] = bt.from_mont();
  g1[2 * m + i] = i <= npublic ? Fr::zero() : (v * inv_d).from_mont();   // BACDelta[0..NPublic] = infinity, :177-180
  if (i <= npublic) g1[4 * m - 1 + i] = (v * inv_g).from_mont();
  if (i + 1 < m) g1[3 * m + i] = (zt_d * fr_pow_u32(t, i)).from_mont();    // (zt/delta) T^i, :139-149
}

// Pinocchio (snark.go:150-248), a = rhoA at, b = rhoB bt, c = rhoC ct.  Standard-form scalars:
//   g1 = A | Ap | Bp | C | Cp | Kp (m each) | G1T (m-1) | [Vkb, G1Kbg: host]
//   g2 = B (m) | [Vka, Vkc, G2Kbg, G2Kg, Vkz: host]
__global__ void k_pinocchio_setup_scalars(const Fr* __restrict__ ev, uint32_t m, Fr rho_a, Fr rho_b, Fr rho_c, Fr ka,
                                          Fr kb, Fr kc, Fr kbeta, Fr t, Fr* __restrict__ g1, Fr* __restrict__ g2) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  Fr a = rho_a * ev[i], b = rho_b * ev[m + i], c = rho_c * ev[2 * m + i];
  g1[i] = a.from_mont();
  g1[m + i] = (ka * a).from_mont();
  g1[2 * m + i] = (kb * b).from_mont();
  g1[3 * m + i] = c.from_mont();
  g1[4 * m + i] = (kc * c).from_mont();
  g1[5 * m + i] = (kbeta * (a + b + c)).from_mont();              // k = a + b + c by construction (snark.go:194-199)
  if (i + 1 < m) g1[6 * m + i] = fr_pow_u32(t, i).from_mont();    // G1T[j] = T^j, :230-237
  g2[i] = b.from_mont();
}

// The toxic values as Montgomery elements; B200_ERANGE when one is >= r.
int load_toxic(const uint64_t* toxic, int count, Fr* out, const char* what) {
  for (int k = 0; k < count; k++) {
    Fr v = fr_load_std(toxic + 4 * k);
    if (v.geq_modulus()) return fail(B200_ERANGE, "%s: toxic value %d >= r", what, k);
    out[k] = v.to_mont();
  }
  return B200_OK;
}

// Argument checks shared by both setups: the R1CS, m >= 3, npublic < m, T not one of the interpolation points 1..n.
int setup_check(b200_r1cs_t h, size_t npublic, const uint64_t* toxic, R1cs** out, const char* what) {
  R1cs* r = find_r1cs(h);
  if (!r) return fail(B200_EINVAL, "%s: bad R1CS handle", what);
  if (!toxic) return fail(B200_EINVAL, "%s: null pointer", what);
  if (r->m < 3 || npublic >= r->m) return fail(B200_EINVAL, "%s: needs m >= 3 signals and npublic < m (m = %zu, npublic = %zu)", what, r->m, npublic);
  *out = r;
  return B200_OK;
}
int setup_check_tau(const R1cs* r, const uint64_t* tau, const char* what) {
  if (tau[1] == 0 && tau[2] == 0 && tau[3] == 0 && tau[0] >= 1 && tau[0] <= r->n)
    return fail(B200_EINVAL, "%s: tau is one of the interpolation points 1..n", what);
  return B200_OK;
}

// Copies points [first, first + count) of d_pts (standard-form Jacobian) to host `dst`.
template <class F>
int copy_points(uint64_t* dst, const F* d_pts, size_t first, size_t count, cudaStream_t st) {
  if (count) CU(cudaMemcpyAsync(dst, d_pts + 3 * first, count * 3 * sizeof(F), cudaMemcpyDeviceToHost, st));
  return B200_OK;
}

int groth16_setup_host(b200_r1cs_t h, size_t npublic, const uint64_t* toxic, uint64_t* at, uint64_t* b1, uint64_t* b2,
                       uint64_t* bacdelta, uint64_t* ptd, uint64_t* z, uint64_t* alpha1, uint64_t* beta1, uint64_t* delta1,
                       uint64_t* beta2, uint64_t* gamma2, uint64_t* delta2, uint64_t* ic) {
  const char* what = "groth16_setup";
  R1cs* r;
  int rc = setup_check(h, npublic, toxic, &r, what);
  if (rc) return rc;
  if (!at || !b1 || !b2 || !bacdelta || !ptd || !z || !alpha1 || !beta1 || !delta1 || !beta2 || !gamma2 || !delta2 || !ic)
    return fail(B200_EINVAL, "%s: null pointer", what);
  Fr tx[5];   // T, Kalpha, Kbeta, Kgamma, Kdelta
  if ((rc = load_toxic(toxic, 5, tx, what))) return rc;
  if (tx[3].is_zero() || tx[4].is_zero()) return fail(B200_EINVAL, "%s: Kgamma and Kdelta must be non-zero (groth16.go:151,201)", what);
  if ((rc = setup_check_tau(r, toxic, what))) return rc;
  const size_t m = r->m, l1 = npublic + 1;
  if ((rc = zero_poly_host(m - 2, z))) return rc;                  // Z = prod_{i=1..m-2}(x - i), groth16.go:122-132
  cudaStream_t st = g_ctx[0].main;
  const size_t n1 = 4 * m - 1 + l1 + 3, n2 = m + 3;
  DevBuf ev, s1, s2, p1, p2;
  CU(ev.alloc(3 * m * sizeof(Fr)));
  CU(s1.alloc(n1 * sizeof(Fr)));
  CU(s2.alloc(n2 * sizeof(Fr)));
  CU(p1.alloc(n1 * 3 * sizeof(Fq)));
  CU(p2.alloc(n2 * 3 * sizeof(Fq2)));
  Fr zt;
  if ((rc = qap_eval_at_enqueue(r, tx[0], m - 2, ev.as<Fr>(), &zt, st))) return rc;
  const Fr inv_d = tx[4].inverse(), inv_g = tx[3].inverse();
  k_groth16_setup_scalars<<<nblk(m, 128), 128, 0, st>>>(ev.as<Fr>(), (uint32_t)m, (uint32_t)npublic, tx[1], tx[2], inv_d, inv_g,
                                                         zt * inv_d, tx[0], s1.as<Fr>(), s2.as<Fr>());
  const Fr v1[3] = {tx[1].from_mont(), tx[2].from_mont(), tx[4].from_mont()};   // Alpha, Beta, Delta in G1
  const Fr v2[3] = {tx[2].from_mont(), tx[3].from_mont(), tx[4].from_mont()};   // Beta, Gamma, Delta in G2
  CU(cudaMemcpyAsync(s1.as<Fr>() + n1 - 3, v1, sizeof v1, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s2.as<Fr>() + m, v2, sizeof v2, cudaMemcpyHostToDevice, st));
  CU(cudaGetLastError());
  CU(fixed_base_mul<Fq>(s1.as<Fr>(), n1, p1.as<Fq>(), g_d_err, st));
  CU(fixed_base_mul<Fq2>(s2.as<Fr>(), n2, p2.as<Fq2>(), g_d_err, st));
  const Fq* g1 = p1.as<Fq>();
  const Fq2* g2 = p2.as<Fq2>();
  uint64_t* outs1[5] = {at, b1, bacdelta, ptd, ic};
  const size_t first1[5] = {0, m, 2 * m, 3 * m, 4 * m - 1}, count1[5] = {m, m, m, m - 1, l1};
  for (int k = 0; k < 5; k++)
    if ((rc = copy_points(outs1[k], g1, first1[k], count1[k], st))) return rc;
  uint64_t* vk1[3] = {alpha1, beta1, delta1};
  uint64_t* vk2[3] = {beta2, gamma2, delta2};
  for (int k = 0; k < 3; k++) {
    if ((rc = copy_points(vk1[k], g1, n1 - 3 + k, 1, st))) return rc;
    if ((rc = copy_points(vk2[k], g2, m + k, 1, st))) return rc;
  }
  if ((rc = copy_points(b2, g2, 0, m, st))) return rc;
  return check_err_flag(what, g_d_err);
}

int pinocchio_setup_host(b200_r1cs_t h, size_t npublic, const uint64_t* toxic, uint64_t* a, uint64_t* ap, uint64_t* b2,
                         uint64_t* bp, uint64_t* c, uint64_t* cp, uint64_t* kp, uint64_t* g1t, uint64_t* z, uint64_t* vk_g1,
                         uint64_t* vk_g2) {
  const char* what = "pinocchio_setup";
  R1cs* r;
  int rc = setup_check(h, npublic, toxic, &r, what);
  if (rc) return rc;
  if (!a || !ap || !b2 || !bp || !c || !cp || !kp || !g1t || !z || !vk_g1 || !vk_g2) return fail(B200_EINVAL, "%s: null pointer", what);
  Fr tx[8];   // T, Ka, Kb, Kc, Kbeta, Kgamma, RhoA, RhoB
  if ((rc = load_toxic(toxic, 8, tx, what))) return rc;
  if ((rc = setup_check_tau(r, toxic, what))) return rc;
  const size_t m = r->m;
  if ((rc = zero_poly_host(m - 2, z))) return rc;                  // snark.go:210-221
  cudaStream_t st = g_ctx[0].main;
  const size_t n1 = 7 * m - 1 + 2, n2 = m + 5;
  DevBuf ev, s1, s2, p1, p2;
  CU(ev.alloc(3 * m * sizeof(Fr)));
  CU(s1.alloc(n1 * sizeof(Fr)));
  CU(s2.alloc(n2 * sizeof(Fr)));
  CU(p1.alloc(n1 * 3 * sizeof(Fq)));
  CU(p2.alloc(n2 * 3 * sizeof(Fq2)));
  Fr zt;
  if ((rc = qap_eval_at_enqueue(r, tx[0], m - 2, ev.as<Fr>(), &zt, st))) return rc;
  const Fr rho_c = tx[6] * tx[7], kbg = tx[4] * tx[5];             // snark.go:150, :223-228
  k_pinocchio_setup_scalars<<<nblk(m, 128), 128, 0, st>>>(ev.as<Fr>(), (uint32_t)m, tx[6], tx[7], rho_c, tx[1], tx[2], tx[3],
                                                           tx[4], tx[0], s1.as<Fr>(), s2.as<Fr>());
  const Fr v1[2] = {tx[2].from_mont(), kbg.from_mont()};                                   // Vkb, G1Kbg
  const Fr v2[5] = {tx[1].from_mont(), tx[3].from_mont(), kbg.from_mont(), tx[5].from_mont(),
                    (rho_c * zt).from_mont()};                                             // Vka, Vkc, G2Kbg, G2Kg, Vkz
  CU(cudaMemcpyAsync(s1.as<Fr>() + n1 - 2, v1, sizeof v1, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s2.as<Fr>() + m, v2, sizeof v2, cudaMemcpyHostToDevice, st));
  CU(cudaGetLastError());
  CU(fixed_base_mul<Fq>(s1.as<Fr>(), n1, p1.as<Fq>(), g_d_err, st));
  CU(fixed_base_mul<Fq2>(s2.as<Fr>(), n2, p2.as<Fq2>(), g_d_err, st));
  const Fq* g1 = p1.as<Fq>();
  const Fq2* g2 = p2.as<Fq2>();
  uint64_t* outs1[7] = {a, ap, bp, c, cp, kp, g1t};
  for (int k = 0; k < 7; k++)
    if ((rc = copy_points(outs1[k], g1, k * m, k == 6 ? m - 1 : m, st))) return rc;
  if ((rc = copy_points(vk_g1, g1, n1 - 2, 2, st))) return rc;
  if ((rc = copy_points(b2, g2, 0, m, st))) return rc;
  if ((rc = copy_points(vk_g2, g2, m, 5, st))) return rc;
  return check_err_flag(what, g_d_err);
}
