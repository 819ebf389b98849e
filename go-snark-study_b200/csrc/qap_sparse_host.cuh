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
    CU(w->part.alloc(kShortZDotBlocks * sizeof(Fr)));
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

// The h-direct domains of r (the QAP domain and QapHDomain), built on g_ctx[0].main and waited for on first use.
int r1cs_hdomain(R1cs* r, QapDomain** dom) {
  int rc = get_domain(pow2_at_least(r->n), dom);
  if (rc) return rc;
  if (!r->hd) {
    auto hd = std::make_unique<QapHDomain>();
    CU(qap_hdomain_build(*g_ctx[0].poly, *hd, r->n, g_ctx[0].main));   // synchronises g_ctx[0].main
    r->hd = std::move(hd);
  }
  return B200_OK;
}

// d_w: m witness values (device, standard form; an entry >= r is read as 0 and sets bit 1 of *err) -> the n - 1
// coefficients of h = DivisorPolynomial(ax*bx - cx, Z) in ws.h_std (standard form), without forming px (qap_sparse.cuh:
// QapHDomain).  The quotient does not depend on cx, so C w is not computed.  Requires n >= 2.  The domains are shared by
// every context: built on g_ctx[0].main and waited for on the first call.
// The witness load and the quotient q by Z_{n+1} (Montgomery, ws.hw.coef), from the Newton coefficients of a | b | a*b that
// it leaves in ws.coef (N-strided) and the witness (Montgomery) in ws.w_mont.  Requires n >= 2.
int qap_q_enqueue(R1cs* r, R1csWork& ws, PolyCtx& pc, const Fr* d_w_std, int* err, cudaStream_t st) {
  const size_t n = r->n, m = r->m;
  QapDomain* dom;
  int rc = r1cs_hdomain(r, &dom);
  if (rc) return rc;
  Fr* w = ws.w_mont.as<Fr>();
  k_poly_load<<<nblk(m, 256), 256, 0, st>>>(d_w_std, (uint32_t)m, (uint32_t)m, 0, 0, w, (uint32_t)m, err);
  Fr* vals = ws.vals.as<Fr>();
  for (int k = 0; k < 2; k++)
    k_spmv_csr<<<nblk(n, 128), 128, 0, st>>>(r->M[k].rowptr.as<uint32_t>(), r->M[k].col.as<uint32_t>(), r->M[k].val.as<Fr>(), w,
                                              (uint32_t)n, vals + k * n);
  g_launches += 3;
  Fr* coef = ws.coef.as<Fr>();   // here: the Newton coefficients of a | b | a*b (N-strided)
  CU(qap_h_from_values(pc, *dom, ws.work, *r->hd, vals, coef, st, &ws.hw));
  return B200_OK;
}

int qap_h_enqueue(R1cs* r, R1csWork& ws, PolyCtx& pc, const Fr* d_w_std, int* err, cudaStream_t st) {
  const size_t n = r->n;
  if (n < 2) return fail(B200_EINVAL, "qap_h: needs at least 2 constraints");
  int rc = qap_q_enqueue(r, ws, pc, d_w_std, err, st);
  if (rc) return rc;
  k_poly_store<<<nblk(n - 1, 256), 256, 0, st>>>(ws.hw.coef.as<Fr>(), (uint32_t)(n - 1), 0, 1, ws.h_std.as<Fr>());
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}

// The batch scratch of a prove context's workspace; `done` is recorded behind the last batch that used it.
struct R1csBatch : R1csBatchWork {
  cudaEvent_t done = nullptr;
  ~R1csBatch() override { if (done) cudaEventDestroy(done); }
};

// Before a batch of k witnesses on the h-direct branch or the len(Z) = n one: builds the domains (first use) and grows the workspace's batch
// scratch to k witnesses, every buffer the batch touches included, so that enqueueing it allocates nothing.  A regrowth
// first waits for the last batch that used the scratch, not for the device.
int qap_batch_prepare(R1cs* r, R1csWork& ws, size_t k, R1csBatch** out) {
  QapDomain* dom;
  int rc = r1cs_hdomain(r, &dom);
  if (rc) return rc;
  if (!ws.batch) {
    auto b = std::make_unique<R1csBatch>();
    CU(cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming));
    ws.batch = std::move(b);
  }
  auto* b = static_cast<R1csBatch*>(ws.batch.get());
  if (b->k < k) {
    CU(cudaEventSynchronize(b->done));
    const size_t n = r->n, m = r->m, N = dom->N, M = r->hd->M, Nt = r->hd->tree.N, F = sizeof(Fr);
    CU(b->wt.alloc(m * k * F));
    CU(b->vals.alloc(3 * k * n * F));
    CU(b->coef.alloc(3 * k * N * F));
    CU(b->part.alloc(k * kShortZDotBlocks * F));
    CU(b->work.U.alloc(3 * k * 2 * N * F));
    CU(b->hw.V.alloc(3 * k * M * F));
    CU(b->hw.hv.alloc(k * n * F));
    CU(b->hw.coef.alloc(k * Nt * F));
    CU(b->hw.work.U.alloc(k * 2 * Nt * F));
    CU(b->hw.work.X.alloc(k * Nt * F));
    b->k = k;
  }
  CU(b->work.E.ensure(2 * dom->N * sizeof(Fr)));   // the cached e^-x series: allocated once
  CU(b->hw.work.E.ensure(2 * r->hd->tree.N * sizeof(Fr)));
  *out = b;
  return B200_OK;
}

// d_w: k witnesses of m standard-form scalars (witness p at d_w + p*m; an entry >= r is read as 0 and sets bit 1 of
// *err) -> quotient p (n - 1 coefficients, Montgomery) at b.hw.coef + p * tree.N.  After qap_batch_prepare for >= k.
int qap_h_batch_enqueue(R1cs* r, R1csBatch& b, PolyCtx& pc, const Fr* d_w, size_t k, int* err, cudaStream_t st) {
  const size_t n = r->n, m = r->m;
  QapDomain* dom;
  int rc = get_domain(pow2_at_least(n), &dom);
  if (rc) return rc;
  k_witness_load_batch<<<nblk(m * k, 256), 256, 0, st>>>(d_w, (uint32_t)m, (uint32_t)k, b.wt.as<Fr>(), err);
  const size_t tiles = (k + kSpmmTile - 1) / kSpmmTile;
  k_spmm_ab<<<nblk(n * tiles, 128), 128, 0, st>>>(r->M[0].rowptr.as<uint32_t>(), r->M[0].col.as<uint32_t>(), r->M[0].val.as<Fr>(),
                                                  r->M[1].rowptr.as<uint32_t>(), r->M[1].col.as<uint32_t>(), r->M[1].val.as<Fr>(),
                                                  b.wt.as<Fr>(), (uint32_t)n, (uint32_t)k, b.vals.as<Fr>());
  g_launches += 2;
  CU(qap_h_batch(pc, *dom, b.work, *r->hd, b.vals.as<Fr>(), b.coef.as<Fr>(), (int)k, st, &b.hw));
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
  if ((rc = scratch_acquire(g_ctx[0], st))) return rc;   // ws: context 0's, which its proofs' front ends share
  rc = qap_px_enqueue(r, *ws, *g_ctx[0].poly, dw.as<Fr>(), dabc.as<Fr>(), dpx.as<Fr>(), g_d_err, st);
  if (rc) return rc;
  if ((rc = scratch_release(g_ctx[0], st))) return rc;
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
  if ((rc = scratch_acquire(g_ctx[0], st))) return rc;
  CU(interpolate_ap(*g_ctx[0].poly, *dom, wk, dm.as<Fr>(), n, n, 1, dc.as<Fr>(), st));
  if ((rc = scratch_release(g_ctx[0], st))) return rc;
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
  if ((rc = scratch_acquire(g_ctx[0], st))) return rc;
  CU(newton_to_monomial(*g_ctx[0].poly, *dom, P.as<Fr>(), X.as<Fr>(), 1, st));
  if ((rc = scratch_release(g_ctx[0], st))) return rc;
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

// ---- the quotient by len(Z) = n (m = n + 1 signals): h = (x - n) q + kappa (qap_sparse.cuh) -----------------------------
// u = C^T lambda of r, built on g_ctx[0].main and waited for on first use; shared by both prove contexts.
int r1cs_short_u(R1cs* r) {
  if (r->short_u) return B200_OK;
  const size_t n = r->n, m = r->m;
  QapDomain* dom;
  int rc = get_domain(pow2_at_least(n), &dom);
  if (rc) return rc;
  cudaStream_t st = g_ctx[0].main;
  auto u = std::make_unique<DevBuf>();
  DevBuf lam;
  CU(lam.alloc(n * sizeof(Fr)));
  CU(u->alloc(m * sizeof(Fr)));
  k_short_z_lambda<<<nblk(n, 256), 256, 0, st>>>(dom->invfact.as<Fr>(), (uint32_t)n, lam.as<Fr>());
  k_spmv_t<<<nblk(m, 128), 128, 0, st>>>(r->M[2].cptr.as<uint32_t>(), r->M[2].crow.as<uint32_t>(), r->M[2].cval.as<Fr>(),
                                          lam.as<Fr>(), (uint32_t)m, u->as<Fr>());
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(st));   // lam is freed on return
  r->short_u = std::move(u);
  return B200_OK;
}

// h_p[off + i] (i < n_ptd) of k quotients into the vectors at vec + p * stride, standard form, zeros beyond len(h) = n,
// then tail[4p] when given (k_quotient_store_shifted).  q: quotient p at q + p * qstride; d: the Newton coefficients of
// a | b | a*b of witness p at d + 3p * N; part: the k_short_z_dot partials.
int qap_short_store(R1cs* r, const Fr* q, size_t qstride, const Fr* d, const Fr* part, size_t k, Fr* vec, size_t stride,
                    size_t n_ptd, size_t off, const Fr* tail, cudaStream_t st) {
  const size_t n = r->n, N = pow2_at_least(n);
  const uint32_t total = (uint32_t)(k * (n_ptd + 1));
  k_quotient_store_shifted<<<nblk(total, 256), 256, 0, st>>>(q, (uint32_t)qstride, (uint32_t)n, fr_from_u64(n), d + 2 * N + (n - 1),
                                                             (uint32_t)(3 * N), part, short_z_dot_blocks(r->m), (uint32_t)n_ptd, tail, 4,
                                                             total, vec, (uint32_t)stride, (uint32_t)off);
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}

// qap_h_enqueue for len(Z) = n: the n coefficients of h = DivisorPolynomial(ax*bx - cx, Z_n) in ws.h_std (standard form),
// from the same front end plus one dot product; C w is not computed.  Requires n >= 2.
int qap_h_short_enqueue(R1cs* r, R1csWork& ws, PolyCtx& pc, const Fr* d_w_std, int* err, cudaStream_t st) {
  const size_t n = r->n;
  if (n < 2) return fail(B200_EINVAL, "qap_h: needs at least 2 constraints");
  int rc = r1cs_short_u(r);
  if (rc) return rc;
  if ((rc = qap_q_enqueue(r, ws, pc, d_w_std, err, st))) return rc;
  CU(short_z_dot(pc, r->short_u->as<Fr>(), ws.w_mont.as<Fr>(), r->m, 1, ws.part.as<Fr>(), st));
  return qap_short_store(r, ws.hw.coef.as<Fr>(), 0, ws.coef.as<Fr>(), ws.part.as<Fr>(), 1, ws.h_std.as<Fr>(), n, n, 0, nullptr, st);
}

// qap_h_batch_enqueue for len(Z) = n, quotients included: h_p[off + i] (i < n_ptd) into vec + p * stride (standard form,
// zeros beyond len(h) = n), then tail[4p] when given.  After qap_batch_prepare for >= k.  The launches of
// qap_h_batch_enqueue plus k_short_z_dot, whatever k; the store takes the place of k_quotient_store.
int qap_h_short_batch_enqueue(R1cs* r, R1csBatch& b, PolyCtx& pc, const Fr* d_w, size_t k, int* err, cudaStream_t st, Fr* vec,
                              size_t stride, size_t n_ptd, size_t off, const Fr* tail) {
  int rc = r1cs_short_u(r);
  if (rc) return rc;
  if ((rc = qap_h_batch_enqueue(r, b, pc, d_w, k, err, st))) return rc;
  CU(short_z_dot(pc, r->short_u->as<Fr>(), b.wt.as<Fr>(), r->m, (int)k, b.part.as<Fr>(), st));
  return qap_short_store(r, b.hw.coef.as<Fr>(), r->hd->tree.N, b.coef.as<Fr>(), b.part.as<Fr>(), k, vec, stride, n_ptd, off, tail, st);
}

// ---- the witness-fed quotient h = (ax*bx - cx) / Z, whichever Z the key has ------------------------------------------
// The shapes whose proofs can verify have Z = prod_{i<=n}(x - i) (m = n + 2, SURVEY H5: h straight from the rows' values)
// or Z = prod_{i<n}(x - i) (m = n + 1: the same front end, h = (x - n) q + kappa); both need n >= 2.  Any other Z goes
// through px and the key's division, one witness at a time.  The only place that compares len(Z) with n.
enum class QapForm { HDirect, ShortZ, PxDivision };
QapForm qap_form(const R1cs* r, size_t nz) {
  if (r->n >= 2 && nz == r->n + 1) return QapForm::HDirect;
  if (r->n >= 2 && nz == r->n) return QapForm::ShortZ;
  return QapForm::PxDivision;
}

// One witness's quotient on `st`, in the workspace of prove context ctx: either *h_std (the standard-form h) or *px_mont
// (the Montgomery px, for the caller's division by Z) is set, the other null.
int qap_quotient_enqueue(R1cs* r, size_t nz, int ctx, PolyCtx& pc, const Fr* d_w, int* err, cudaStream_t st,
                         const Fr** h_std, const Fr** px_mont) {
  *h_std = *px_mont = nullptr;
  R1csWork* ws;
  int rc = r1cs_work(r, ctx, &ws);
  if (rc) return rc;
  switch (qap_form(r, nz)) {
    case QapForm::HDirect: rc = qap_h_enqueue(r, *ws, pc, d_w, err, st); break;
    case QapForm::ShortZ: rc = qap_h_short_enqueue(r, *ws, pc, d_w, err, st); break;
    case QapForm::PxDivision:
      if ((rc = qap_px_enqueue(r, *ws, pc, d_w, nullptr, nullptr, err, st))) return rc;
      *px_mont = ws->px_mont.as<Fr>();
      return B200_OK;
  }
  if (rc) return rc;
  *h_std = ws->h_std.as<Fr>();
  return B200_OK;
}

// Before a batch of k witnesses: every scratch of its quotients (the workspace of prove context ctx; the batch scratch
// of the batched forms; u for len(Z) = n), so that enqueueing the batch allocates nothing.  *fb: the batch scratch, or
// null (px-division), whose `done` the caller records behind the batch.
int qap_quotient_batch_prepare(R1cs* r, size_t nz, int ctx, size_t k, R1csWork** ws, R1csBatch** fb) {
  *fb = nullptr;
  int rc = r1cs_work(r, ctx, ws);
  if (rc) return rc;
  const QapForm f = qap_form(r, nz);
  if (f != QapForm::PxDivision && (rc = qap_batch_prepare(r, **ws, k, fb))) return rc;
  return f == QapForm::ShortZ ? r1cs_short_u(r) : B200_OK;
}

// A batch of k witnesses stays inside 32-bit transform indexing: 3k * 2N < 2^32 (N = the power of two >= n).
int qap_batch_check(const R1cs* r, size_t k, const char* what) {
  const uint64_t N = pow2_at_least(r->n);
  if (6 * (uint64_t)k * N >= (1ull << 32)) return fail(B200_EINVAL, "%s: 3k * 2N = 3 * %zu * %llu transform elements exceed 2^32", what, k, (unsigned long long)(2 * N));
  return B200_OK;
}

// d_w: k witnesses (standard form, witness p at d_w + p*m) -> coefficients [off, off + n_ptd) of each quotient h_p by Z
// into the vectors at vec + p * stride, standard form, zeros beyond len(h), then tail[4p] when given.  After
// qap_quotient_batch_prepare for >= k with the same ws and fb.  px-division: each witness's px is divided straight into
// its vector when the slice is all of h from h[0], else into `scratch` (>= len(h) coefficients) and the slice copied out.
int qap_quotient_batch_enqueue(R1cs* r, R1csWork* ws, R1csBatch* fb, PolyCtx& pc, Divisor& Z, Fr* scratch,
                               const Fr* d_w, size_t k, Fr* vec, size_t stride, size_t n_ptd, size_t off, const Fr* tail,
                               cudaStream_t st, int* err) {
  const size_t npx = 2 * r->n - 1, nq = npx - Z.nb + 1;
  const QapForm f = qap_form(r, Z.nb);
  int rc;
  if (f == QapForm::ShortZ)   // the store is part of it
    return qap_h_short_batch_enqueue(r, *fb, pc, d_w, k, err, st, vec, stride, n_ptd, off, tail);
  const Fr* q = nullptr;   // px-division: the quotients are already in place, the store only zero-fills and adds the tail
  if (f == QapForm::HDirect) {
    if ((rc = qap_h_batch_enqueue(r, *fb, pc, d_w, k, err, st))) return rc;
    q = fb->hw.coef.as<Fr>();
  } else {
    const bool direct = off == 0 && nq <= n_ptd;
    const size_t have = nq > off ? std::min(nq - off, n_ptd) : 0;   // quotient coefficients inside the slice
    for (size_t p = 0; p < k; p++) {
      if ((rc = qap_px_enqueue(r, *ws, pc, d_w + p * r->m, nullptr, nullptr, err, st))) return rc;
      CU(poly_div_device(pc, Z, ws->px_mont.as<Fr>(), npx, 1, direct ? vec + p * stride : scratch, nullptr, err, st));
      if (!direct && have) CU(cudaMemcpyAsync(vec + p * stride, scratch + off, have * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    }
  }
  const uint32_t qtotal = (uint32_t)(k * (n_ptd + 1));
  k_quotient_store<<<nblk(qtotal, 256), 256, 0, st>>>(q, q ? (uint32_t)r->hd->tree.N : 0, (uint32_t)nq, (uint32_t)n_ptd, tail, 4,
                                                      qtotal, vec, (uint32_t)stride, (uint32_t)off);
  g_launches += 1;
  return B200_OK;
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
