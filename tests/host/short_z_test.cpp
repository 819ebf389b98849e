// CPU test vehicle for the quotient by len(Z) = n of witness-fed proving on circuits with m = n + 1 signals (g++,
// csrc/host_stub): the kernels the branch adds (k_short_z_lambda, k_short_z_dot, k_quotient_store_shifted, qap_sparse.cuh)
// after the batched front end it shares with the h-direct branch (k_witness_load_batch, k_spmm_ab, qap_h_batch), in the
// order and with the arguments of qap_h_short_batch_enqueue / qap_short_store (qap_sparse_host.cuh).  u = C^T lambda is
// restated here as a plain loop (k_spmv_t's sum).
// Test infrastructure only: never linked into libb200snark.
#include "host_kernel_test.cpp"

namespace {
struct Csr {
  const uint32_t *rowptr, *col;
  std::vector<Fr> val;   // Montgomery
};
Csr load_csr(const uint32_t* rowptr, const uint32_t* col, const uint32_t* val_std, uint32_t n) {
  Csr c{rowptr, col, {}};
  c.val.resize(rowptr[n] ? rowptr[n] : 1);
  for (uint32_t i = 0; i < rowptr[n]; i++) c.val[i] = load_std<Fr>(val_std + 8 * (size_t)i);
  return c;
}
}  // namespace

extern "C" {
// k witnesses (standard form, k x m) of the R1CS A, B, C (CSR, standard-form values) -> the vectors the batch writes:
// vec (k x stride scalars, standard form, in place) gets h_p[off + i] for i < n_ptd, zeros beyond len(h) = n, and tail[p]
// after them (tail: k scalars, standard form).  lambda_out: the n weights of k_short_z_lambda (standard form).
// launches: what the library counts for the branch on a call after the first (the first also fills the e^-x caches):
// the witness load and the sparse product, qap_h_batch's steps, the dot product and the store.  err: the load's word.
int t_short_z_batch(uint32_t n, uint32_t m, const uint32_t* a_rowptr, const uint32_t* a_col, const uint32_t* a_val,
                    const uint32_t* b_rowptr, const uint32_t* b_col, const uint32_t* b_val, const uint32_t* c_rowptr,
                    const uint32_t* c_col, const uint32_t* c_val, const uint32_t* w_std, uint32_t k, uint32_t n_ptd, uint32_t off,
                    const uint32_t* tail_std, uint32_t* vec_std, uint32_t stride, uint32_t* lambda_out,
                    unsigned long long* launches, int* err) {
  Csr A = load_csr(a_rowptr, a_col, a_val, n), B = load_csr(b_rowptr, b_col, b_val, n), C = load_csr(c_rowptr, c_col, c_val, n);
  size_t N = 1;
  while (N < n) N <<= 1;
  QapDomain dom;
  if (qap_domain_build(poly_ctx(), dom, N, nullptr)) return 1;
  QapHDomain hd;
  if (qap_hdomain_build(poly_ctx(), hd, n, nullptr)) return 2;
  // u = C^T lambda (r1cs_short_u)
  std::vector<Fr> lam(n), u(m, Fr::zero());
  run_threads(cdiv(n, 256), 256, [&] { k_short_z_lambda(dom.invfact.as<Fr>(), n, lam.data()); });
  for (uint32_t j = 0; j < n; j++) {
    for (uint32_t x = c_rowptr[j]; x < c_rowptr[j + 1]; x++) u[c_col[x]] = u[c_col[x]] + C.val[x] * lam[j];
    store_std(lambda_out + 8 * (size_t)j, lam[j]);
  }
  std::vector<Fr> w((size_t)k * m), wt((size_t)k * m), vals(3 * (size_t)k * n), d(3 * (size_t)k * N);
  std::vector<Fr> part((size_t)k * kShortZDotBlocks), tail(k), vec((size_t)k * stride);
  std::memcpy(w.data(), w_std, w.size() * sizeof(Fr));
  std::memcpy(tail.data(), tail_std, tail.size() * sizeof(Fr));
  std::memcpy(vec.data(), vec_std, vec.size() * sizeof(Fr));
  QapWork wk;
  QapHWork hw;
  unsigned long long counted = 0;
  poly_ctx().launch_counter = &counted;
  for (int run = 0; run < 2; run++) {
    counted = 0;
    *err = 0;
    // qap_h_batch_enqueue
    run_threads(cdiv((size_t)m * k, 256), 256, [&] { k_witness_load_batch(w.data(), m, k, wt.data(), err); });
    const uint32_t tiles = (k + kSpmmTile - 1) / kSpmmTile;
    run_threads(cdiv((size_t)n * tiles, 128), 128, [&] {
      k_spmm_ab(A.rowptr, A.col, A.val.data(), B.rowptr, B.col, B.val.data(), wt.data(), n, k, vals.data());
    });
    counted += 2;
    if (qap_h_batch(poly_ctx(), dom, wk, hd, vals.data(), d.data(), (int)k, nullptr, &hw)) return 3;
    // qap_h_short_batch_enqueue: the dot product, then qap_short_store
    if (short_z_dot(poly_ctx(), u.data(), wt.data(), m, (int)k, part.data(), nullptr)) return 4;
    const uint32_t total = k * (n_ptd + 1);
    run_threads(cdiv(total, 256), 256, [&] {
      k_quotient_store_shifted(hw.coef.as<Fr>(), (uint32_t)hd.tree.N, n, fr_from_u64(n), d.data() + 2 * N + (n - 1), (uint32_t)(3 * N),
                               part.data(), short_z_dot_blocks(m), n_ptd, tail.data(), 1, total, vec.data(), stride, off);
    });
    counted += 1;
  }
  poly_ctx().launch_counter = nullptr;
  *launches = counted;
  std::memcpy(vec_std, vec.data(), vec.size() * sizeof(Fr));
  return 0;
}
}
