// Host orchestration of the sparse QAP front end (qap_sparse.cuh): resident sparse R1CS handles, witness -> px,
// interpolation over {1..n}, Lagrange evaluation at tau for the trusted setup, and the witness -> proof entry.
// Included inside capi.cu's anonymous namespace (after prove_host.cuh).

std::map<uint64_t, std::unique_ptr<R1cs>> g_r1cs;
uint64_t g_next_r1cs = 1;
std::map<size_t, std::unique_ptr<QapDomain>> g_domains;   // by N (power of two)

int get_domain(size_t N, QapDomain** out) {
  auto it = g_domains.find(N);
  if (it == g_domains.end()) {
    auto d = std::make_unique<QapDomain>();
    CU(qap_domain_build(*g_ctx[0].poly, *d, N, g_ctx[0].main));
    it = g_domains.emplace(N, std::move(d)).first;
  }
  *out = it->second.get();
  return B200_OK;
}
inline size_t pow2_at_least(size_t n) {
  size_t N = 1;
  while (N < n) N <<= 1;
  return N;
}

R1cs* find_r1cs(b200_r1cs_t h) {
  auto it = g_r1cs.find(h);
  return it == g_r1cs.end() ? nullptr : it->second.get();
}

int sparse_upload(SparseMat& M, size_t n, size_t m, const uint32_t* rowptr, const uint32_t* col, const uint64_t* val,
                  const char* name) {
  if (!rowptr) return fail(B200_EINVAL, "r1cs_load: %s: null row pointer array", name);
  if (rowptr[0] != 0) return fail(B200_EINVAL, "r1cs_load: %s: rowptr[0] != 0", name);
  for (size_t j = 0; j < n; j++)
    if (rowptr[j + 1] < rowptr[j]) return fail(B200_EINVAL, "r1cs_load: %s: rowptr not monotone at row %zu", name, j);
  size_t nnz = rowptr[n];
  if (nnz && (!col || !val)) return fail(B200_EINVAL, "r1cs_load: %s: null col/val", name);
  std::vector<Fr> vm(nnz ? nnz : 1);
  std::vector<uint32_t> cptr(m + 1, 0), crow(nnz ? nnz : 1);
  std::vector<Fr> cval(nnz ? nnz : 1);
  for (size_t k = 0; k < nnz; k++) {
    if (col[k] >= m) return fail(B200_EINVAL, "r1cs_load: %s: column index %u >= m", name, col[k]);
    Fr v = fr_load_std(val + 4 * k);
    if (v.geq_modulus()) return fail(B200_ERANGE, "r1cs_load: %s: coefficient >= r (send values mod r)", name);
    vm[k] = v.to_mont();
    cptr[col[k] + 1]++;
  }
  for (size_t i = 0; i < m; i++) cptr[i + 1] += cptr[i];
  {
    std::vector<uint32_t> fill(cptr.begin(), cptr.end() - 1);
    for (size_t j = 0; j < n; j++)
      for (uint32_t k = rowptr[j]; k < rowptr[j + 1]; k++) {
        uint32_t dst = fill[col[k]]++;
        crow[dst] = (uint32_t)j;
        cval[dst] = vm[k];
      }
  }
  M.nnz = nnz;
  CU(M.rowptr.alloc((n + 1) * 4));
  CU(M.col.alloc((nnz ? nnz : 1) * 4));
  CU(M.val.alloc((nnz ? nnz : 1) * sizeof(Fr)));
  CU(M.cptr.alloc((m + 1) * 4));
  CU(M.crow.alloc((nnz ? nnz : 1) * 4));
  CU(M.cval.alloc((nnz ? nnz : 1) * sizeof(Fr)));
  CU(cudaMemcpy(M.rowptr.p, rowptr, (n + 1) * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(M.cptr.p, cptr.data(), (m + 1) * 4, cudaMemcpyHostToDevice));
  if (nnz) {
    CU(cudaMemcpy(M.col.p, col, nnz * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(M.val.p, vm.data(), nnz * sizeof(Fr), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(M.crow.p, crow.data(), nnz * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(M.cval.p, cval.data(), nnz * sizeof(Fr), cudaMemcpyHostToDevice));
  }
  return B200_OK;
}

int r1cs_load(size_t n, size_t m, const uint32_t* const rowptr[3], const uint32_t* const col[3],
              const uint64_t* const val[3], b200_r1cs_t* out) {
  if (!out) return fail(B200_EINVAL, "r1cs_load: null handle pointer");
  if (n == 0 || m == 0 || n > ((size_t)1 << 26) || m > ((size_t)1 << 27)) return fail(B200_EINVAL, "r1cs_load: bad sizes");
  auto r = std::make_unique<R1cs>();
  r->n = n;
  r->m = m;
  static const char* names[3] = {"A", "B", "C"};
  for (int k = 0; k < 3; k++) {
    int rc = sparse_upload(r->M[k], n, m, rowptr[k], col[k], val[k], names[k]);
    if (rc) return rc;
  }
  uint64_t h = g_next_r1cs++;
  g_r1cs[h] = std::move(r);
  *out = h;
  return B200_OK;
}

// The scratch of prove context `ctx` on this R1CS, allocated on first use (which may synchronise the device).
int r1cs_work(R1cs* r, int ctx, R1csWork** out) {
  auto& ws = r->ws[ctx];
  if (!ws) {
    const size_t n = r->n, m = r->m, N = pow2_at_least(n);
    auto w = std::make_unique<R1csWork>();
    CU(w->w_mont.alloc(m * sizeof(Fr)));
    CU(w->vals.alloc(3 * n * sizeof(Fr)));
    CU(w->coef.alloc(3 * N * sizeof(Fr)));
    CU(w->px_mont.alloc((2 * n) * sizeof(Fr)));
    CU(w->h_std.alloc(n * sizeof(Fr)));
    ws = std::move(w);
  }
  *out = ws.get();
  return B200_OK;
}

// d_w: m witness values in device memory, standard form (an entry >= r is read as 0 and sets bit 1 of *err).  Leaves
// ax | bx | cx (N-strided, Montgomery) in ws.coef and px (2n-1, Montgomery) in ws.px_mont; optional standard-form copies
// to device buffers.  The interpolation domain is shared by every context: built (and waited for) on the first call.
int qap_px_enqueue(R1cs* r, R1csWork& ws, PolyCtx& pc, const Fr* d_w_std, Fr* d_abc_std /* 3 x n or null */,
                   Fr* d_px_std /* 2n-1 or null */, int* err, cudaStream_t st) {
  const size_t n = r->n, m = r->m, N = pow2_at_least(n);
  QapDomain* dom;
  int rc = get_domain(N, &dom);
  if (rc) return rc;
  Fr* w = ws.w_mont.as<Fr>();
  k_poly_load<<<nblk(m, 256), 256, 0, st>>>(d_w_std, (uint32_t)m, (uint32_t)m, 0, 0, w, (uint32_t)m, err);
  Fr* vals = ws.vals.as<Fr>();
  for (int k = 0; k < 3; k++)
    k_spmv_csr<<<nblk(n, 128), 128, 0, st>>>(r->M[k].rowptr.as<uint32_t>(), r->M[k].col.as<uint32_t>(), r->M[k].val.as<Fr>(), w,
                                              (uint32_t)n, vals + k * n);
  g_launches += 4;
  Fr* coef = ws.coef.as<Fr>();
  CU(interpolate_ap(pc, *dom, ws.work, vals, n, n, 3, coef, st));
  if (d_abc_std)
    for (int k = 0; k < 3; k++)
      k_poly_store<<<nblk(n, 256), 256, 0, st>>>(coef + k * N, (uint32_t)n, 0, 1, d_abc_std + k * n);
  // px = ax * bx - cx: one size-2N cyclic product (2n - 1 <= 2N)
  const size_t N2 = 2 * N;
  const int l2 = dom->logN + 1;
  Fr* U = ws.work.U.as<Fr>();   // >= 3 * 2N elements (interpolate_ap sized it)
  k_take<<<nblk(N2, 256), 256, 0, st>>>(coef, (uint32_t)n, (uint32_t)N2, U);
  k_take<<<nblk(N2, 256), 256, 0, st>>>(coef + N, (uint32_t)n, (uint32_t)N2, U + N2);
  CU(ntt_batched(pc, U, l2, 2 * N2, 0, st));
  CU(pc.pointwise(U, U + N2, l2, true, st));
  CU(ntt_batched(pc, U, l2, N2, 1, st));
  k_px_finish<<<nblk(2 * n - 1, 256), 256, 0, st>>>(U, coef + 2 * N, (uint32_t)n, ws.px_mont.as<Fr>(), d_px_std);
  g_launches += 4;
  CU(cudaGetLastError());
  return B200_OK;
}

// d_w: m witness values (device, standard form; an entry >= r is read as 0 and sets bit 1 of *err) -> the n - 1
// coefficients of h = DivisorPolynomial(ax*bx - cx, Z) in ws.h_std (standard form), without forming px (qap_sparse.cuh:
// QapHDomain).  The quotient does not depend on cx, so C w is not computed.  Requires n >= 2.  The domains are shared by
// every context: built on g_ctx[0].main and waited for on the first call.
int qap_h_enqueue(R1cs* r, R1csWork& ws, PolyCtx& pc, const Fr* d_w_std, int* err, cudaStream_t st) {
  const size_t n = r->n, m = r->m, N = pow2_at_least(n);
  if (n < 2) return fail(B200_EINVAL, "qap_h: needs at least 2 constraints");
  QapDomain* dom;
  int rc = get_domain(N, &dom);
  if (rc) return rc;
  if (!r->hd) {
    auto hd = std::make_unique<QapHDomain>();
    CU(qap_hdomain_build(*g_ctx[0].poly, *hd, n, g_ctx[0].main));   // synchronises g_ctx[0].main
    r->hd = std::move(hd);
  }
  Fr* w = ws.w_mont.as<Fr>();
  k_poly_load<<<nblk(m, 256), 256, 0, st>>>(d_w_std, (uint32_t)m, (uint32_t)m, 0, 0, w, (uint32_t)m, err);
  Fr* vals = ws.vals.as<Fr>();
  for (int k = 0; k < 2; k++)
    k_spmv_csr<<<nblk(n, 128), 128, 0, st>>>(r->M[k].rowptr.as<uint32_t>(), r->M[k].col.as<uint32_t>(), r->M[k].val.as<Fr>(), w,
                                              (uint32_t)n, vals + k * n);
  g_launches += 3;
  Fr* coef = ws.coef.as<Fr>();   // here: the Newton coefficients of a | b | a*b (N-strided)
  CU(qap_h_from_values(pc, *dom, ws.work, *r->hd, vals, coef, st, &ws.hw));
  k_poly_store<<<nblk(n - 1, 256), 256, 0, st>>>(ws.hw.coef.as<Fr>(), (uint32_t)(n - 1), 0, 1, ws.h_std.as<Fr>());
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}

int qap_px_host(b200_r1cs_t h, const uint64_t* w, size_t nw, uint64_t* ax, uint64_t* bx, uint64_t* cx, uint64_t* px) {
  R1cs* r = find_r1cs(h);
  if (!r) return fail(B200_EINVAL, "qap_px: bad R1CS handle");
  if (!w || nw != r->m) return fail(B200_EINVAL, "qap_px: witness length %zu != m %zu", nw, r->m);
  const size_t n = r->n;
  cudaStream_t st = g_ctx[0].main;
  R1csWork* ws;
  int rc = r1cs_work(r, 0, &ws);
  if (rc) return rc;
  DevBuf dw, dabc, dpx;
  CU(dw.alloc(nw * sizeof(Fr)));
  CU(dabc.alloc(3 * n * sizeof(Fr)));
  CU(dpx.alloc((2 * n - 1) * sizeof(Fr)));
  CU(cudaMemcpyAsync(dw.p, w, nw * sizeof(Fr), cudaMemcpyHostToDevice, st));
  rc = qap_px_enqueue(r, *ws, *g_ctx[0].poly, dw.as<Fr>(), dabc.as<Fr>(), dpx.as<Fr>(), g_d_err, st);
  if (rc) return rc;
  uint64_t* outs[3] = {ax, bx, cx};
  for (int k = 0; k < 3; k++)
    if (outs[k]) CU(cudaMemcpyAsync(outs[k], dabc.as<Fr>() + k * n, n * sizeof(Fr), cudaMemcpyDeviceToHost, st));
  if (px) CU(cudaMemcpyAsync(px, dpx.p, (2 * n - 1) * sizeof(Fr), cudaMemcpyDeviceToHost, st));
  return check_err_flag("qap_px", g_d_err);
}

// LagrangeInterpolation over x = 1..n (r1csqap.go:150-158) at any n: values -> n coefficients
int interpolate_host(const uint64_t* values, size_t n, uint64_t* coeffs) {
  if (!values || !coeffs || n == 0 || n > ((size_t)1 << 26)) return fail(B200_EINVAL, "interpolate: bad arguments");
  const size_t N = pow2_at_least(n);
  QapDomain* dom;
  int rc = get_domain(N, &dom);
  if (rc) return rc;
  cudaStream_t st = g_ctx[0].main;
  DevBuf dv, dm, dc, ds;
  QapWork wk;
  CU(dv.alloc(n * sizeof(Fr)));
  CU(dm.alloc(n * sizeof(Fr)));
  CU(dc.alloc(N * sizeof(Fr)));
  CU(ds.alloc(n * sizeof(Fr)));
  CU(cudaMemcpyAsync(dv.p, values, n * sizeof(Fr), cudaMemcpyHostToDevice, st));
  k_poly_load<<<nblk(n, 256), 256, 0, st>>>(dv.as<Fr>(), (uint32_t)n, (uint32_t)n, 0, 0, dm.as<Fr>(), (uint32_t)n, g_d_err);
  CU(interpolate_ap(*g_ctx[0].poly, *dom, wk, dm.as<Fr>(), n, n, 1, dc.as<Fr>(), st));
  k_poly_store<<<nblk(n, 256), 256, 0, st>>>(dc.as<Fr>(), (uint32_t)n, 0, 1, ds.as<Fr>());
  CU(cudaMemcpyAsync(coeffs, ds.p, n * sizeof(Fr), cudaMemcpyDeviceToHost, st));
  return check_err_flag("interpolate", g_d_err);
}

// prod_{i=1..n}(x - i) at any n: the Newton basis element of index n, converted by the same divide and conquer
// (for n a power of two it is the tree's root).  Montgomery coefficients left in d_out[0..n].
int zero_poly_device(size_t n, DevBuf& d_out, cudaStream_t st) {
  CU(d_out.alloc((n + 1) * sizeof(Fr)));
  Fr* o = d_out.as<Fr>();
  if (n == 0) {
    Fr one = Fr::one();
    CU(cudaMemcpyAsync(o, &one, sizeof(Fr), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    return B200_OK;
  }
  const size_t N = pow2_at_least(n + 1);
  QapDomain* dom;
  int rc = get_domain(N, &dom);
  if (rc) return rc;
  DevBuf P, X;
  CU(P.alloc(N * sizeof(Fr)));
  CU(X.alloc(N * sizeof(Fr)));
  CU(cudaMemsetAsync(P.p, 0, N * sizeof(Fr), st));
  Fr one = Fr::one();
  CU(cudaMemcpyAsync(P.as<Fr>() + n, &one, sizeof(Fr), cudaMemcpyHostToDevice, st));
  CU(newton_to_monomial(*g_ctx[0].poly, *dom, P.as<Fr>(), X.as<Fr>(), 1, st));
  CU(cudaMemcpyAsync(o, P.p, (n + 1) * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
  CU(cudaStreamSynchronize(st));
  return B200_OK;
}

// alpha_i(tau), beta_i(tau), gamma_i(tau) for every signal i (the Eval(alphas[i], t) loops of GenerateTrustedSetup,
// groth16/groth16.go:164-205, snark.go:171-189) without the dense polynomials: A^T l(tau) with l = Lagrange basis of
// {1..n} at tau; and zt = prod_{i=1..nz}(tau - i).
__global__ void k_spmv_t(const uint32_t* __restrict__ cptr, const uint32_t* __restrict__ crow, const Fr* __restrict__ cval,
                         const Fr* __restrict__ l, uint32_t m, Fr* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  Fr acc = Fr::zero();
  for (uint32_t k = cptr[i], e = cptr[i + 1]; k < e; k++) acc = acc + cval[k] * l[crow[k]];
  out[i] = acc;
}
// Enqueues at | bt | ct (Montgomery, m each) into d_out on `st`; *zt = prod_{i=1..nz}(tau - i) (Montgomery).  t: tau in
// Montgomery form.  tau in 1..n sets bit 4 of g_d_err.
int qap_eval_at_enqueue(R1cs* r, Fr t, size_t nz, Fr* d_out, Fr* zt, cudaStream_t st) {
  const size_t n = r->n, m = r->m, N = pow2_at_least(n);
  QapDomain* dom;
  int rc = get_domain(N, &dom);
  if (rc) return rc;
  Fr zn = Fr::one(), znz = Fr::one();   // prod_{i=1..n}(tau - i) and prod_{i=1..nz}(tau - i), on the host (O(n))
  size_t top = n > nz ? n : nz;
  Fr acc = Fr::one();
  for (size_t i = 1; i <= top; i++) {
    acc = acc * (t - fr_from_u64(i));
    if (i == n) zn = acc;
    if (i == nz) znz = acc;
  }
  CU(r->lag.ensure(n * sizeof(Fr)));
  k_lagrange_at<<<nblk(n, 128), 128, 0, st>>>(dom->invfact.as<Fr>(), (uint32_t)n, t, zn, r->lag.as<Fr>(), g_d_err);
  for (int k = 0; k < 3; k++)
    k_spmv_t<<<nblk(m, 128), 128, 0, st>>>(r->M[k].cptr.as<uint32_t>(), r->M[k].crow.as<uint32_t>(), r->M[k].cval.as<Fr>(),
                                            r->lag.as<Fr>(), (uint32_t)m, d_out + k * m);
  CU(cudaGetLastError());
  *zt = znz;
  return B200_OK;
}
int qap_eval_at_host(b200_r1cs_t h, const uint64_t* tau, size_t nz, uint64_t* at, uint64_t* bt, uint64_t* ct, uint64_t* zt_out) {
  R1cs* r = find_r1cs(h);
  if (!r) return fail(B200_EINVAL, "qap_eval_at: bad R1CS handle");
  if (!tau || !at || !bt || !ct) return fail(B200_EINVAL, "qap_eval_at: null pointer");
  Fr t_std = fr_load_std(tau);
  if (t_std.geq_modulus()) return fail(B200_ERANGE, "qap_eval_at: tau >= r");
  const size_t m = r->m;
  cudaStream_t st = g_ctx[0].main;
  DevBuf o, os;
  CU(o.alloc(3 * m * sizeof(Fr)));
  CU(os.alloc(3 * m * sizeof(Fr)));
  Fr znz;
  int rc = qap_eval_at_enqueue(r, t_std.to_mont(), nz, o.as<Fr>(), &znz, st);
  if (rc) return rc;
  k_poly_store<<<nblk(3 * m, 256), 256, 0, st>>>(o.as<Fr>(), (uint32_t)(3 * m), 0, 1, os.as<Fr>());
  uint64_t* outs[3] = {at, bt, ct};
  for (int k = 0; k < 3; k++) CU(cudaMemcpyAsync(outs[k], os.as<Fr>() + k * m, m * sizeof(Fr), cudaMemcpyDeviceToHost, st));
  if (zt_out) {
    Fr z = znz.from_mont();
    memcpy(zt_out, &z, sizeof(Fr));
  }
  rc = check_err_flag("qap_eval_at", g_d_err);
  if (rc == B200_OK) return rc;
  return rc;
}
