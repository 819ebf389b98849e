// CPU test vehicle for the batched QAP front end of b200_groth16_prove_witness_batch (g++, csrc/host_stub): k witnesses
// through k_witness_load_batch, k_spmm_ab and qap_h_batch (qap_sparse.cuh), the library's own host orchestration on the
// emulated kernels, next to k runs of the single-witness path (k_poly_load, k_spmv_csr, qap_h_from_values), and the
// quotient store into the C||PTD scalar vectors (k_quotient_store).
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
void store_block(uint32_t* out, const Fr* v, size_t cnt) {
  for (size_t i = 0; i < cnt; i++) store_std(out + 8 * i, v[i]);
}
}  // namespace

extern "C" {
// k witnesses (standard form, k x m) -> out: (A w_p)_j | (B w_p)_j | products, blocks 3p .. 3p+2 of n (standard form), by
// k_spmm_ab; ref: the same from k_spmv_csr per witness and matrix.  err: the witness-load error word.
int t_spmm_ab(uint32_t n, uint32_t m, const uint32_t* a_rowptr, const uint32_t* a_col, const uint32_t* a_val,
              const uint32_t* b_rowptr, const uint32_t* b_col, const uint32_t* b_val, const uint32_t* w_std, uint32_t k,
              uint32_t* out, uint32_t* ref, int* err) {
  Csr A = load_csr(a_rowptr, a_col, a_val, n), B = load_csr(b_rowptr, b_col, b_val, n);
  std::vector<Fr> w(w_std ? (size_t)k * m : 0), wt((size_t)k * m), vals(3 * (size_t)k * n);
  std::memcpy(w.data(), w_std, w.size() * sizeof(Fr));
  *err = 0;
  run_threads(cdiv((size_t)m * k, 256), 256, [&] { k_witness_load_batch(w.data(), m, k, wt.data(), err); });
  const uint32_t tiles = (k + kSpmmTile - 1) / kSpmmTile;
  run_threads(cdiv((size_t)n * tiles, 128), 128, [&] {
    k_spmm_ab(A.rowptr, A.col, A.val.data(), B.rowptr, B.col, B.val.data(), wt.data(), n, k, vals.data());
  });
  store_block(out, vals.data(), vals.size());
  int err1 = 0;
  std::vector<Fr> wm(m), ab(2 * (size_t)n);
  for (uint32_t p = 0; p < k; p++) {
    run_threads(cdiv(m, 256), 256, [&] { k_poly_load(w.data() + (size_t)p * m, m, m, 0, 0, wm.data(), m, &err1); });
    run_threads(cdiv(n, 128), 128, [&] { k_spmv_csr(A.rowptr, A.col, A.val.data(), wm.data(), n, ab.data()); });
    run_threads(cdiv(n, 128), 128, [&] { k_spmv_csr(B.rowptr, B.col, B.val.data(), wm.data(), n, ab.data() + n); });
    uint32_t* o = ref + 24 * (size_t)p * n;
    store_block(o, ab.data(), 2 * (size_t)n);
    for (uint32_t j = 0; j < n; j++) store_std(o + 8 * (2 * (size_t)n + j), ab[j] * ab[n + j]);
  }
  return err1 == *err ? 0 : 100 + err1;
}

// The quotients of k value sets a_p | b_p | c_p (standard form, blocks 3p .. 3p+2 of n): h_batch by qap_h_batch (the
// values of c replaced by the products a_j b_j first, as k_spmm_ab writes them), h_single by qap_h_from_values once per
// set; n - 1 coefficients each, standard form.  Returns nonzero if a coefficient at or beyond n - 1 is not zero.
int t_qap_h_batch(const uint32_t* abc_std, uint32_t n, uint32_t k, uint32_t* h_batch, uint32_t* h_single) {
  size_t N = 1;
  while (N < n) N <<= 1;
  QapDomain dom;
  if (qap_domain_build(poly_ctx(), dom, N, nullptr)) return 1;
  QapHDomain hd;
  if (qap_hdomain_build(poly_ctx(), hd, n, nullptr)) return 2;
  std::vector<Fr> v(3 * (size_t)k * n);
  for (size_t i = 0; i < v.size(); i++) v[i] = load_std<Fr>(abc_std + 8 * i);
  std::vector<Fr> vb = v, d(3 * (size_t)k * N);
  for (uint32_t p = 0; p < k; p++)
    for (uint32_t j = 0; j < n; j++) vb[(3 * (size_t)p + 2) * n + j] = vb[3 * (size_t)p * n + j] * vb[(3 * (size_t)p + 1) * n + j];
  QapWork wk;
  QapHWork hw;
  if (qap_h_batch(poly_ctx(), dom, wk, hd, vb.data(), d.data(), (int)k, nullptr, &hw)) return 3;
  const Fr* c = hw.coef.as<Fr>();
  for (uint32_t p = 0; p < k; p++) {
    store_block(h_batch + 8 * (size_t)p * (n - 1), c + (size_t)p * hd.tree.N, n - 1);
    for (size_t i = n - 1; i < hd.tree.N; i++)
      if (!c[(size_t)p * hd.tree.N + i].is_zero()) return 4;
  }
  for (uint32_t p = 0; p < k; p++) {
    std::vector<Fr> vs(v.begin() + 3 * (size_t)p * n, v.begin() + 3 * (size_t)(p + 1) * n), ds(3 * N);
    QapWork wk1;
    QapHWork hw1;
    if (qap_h_from_values(poly_ctx(), dom, wk1, hd, vs.data(), ds.data(), nullptr, &hw1)) return 5;
    store_block(h_single + 8 * (size_t)p * (n - 1), hw1.coef.as<Fr>(), n - 1);
  }
  return 0;
}

// k_quotient_store over k vectors of `stride` scalars (standard form, in place), from offset `off`: coef (k blocks of
// cstride, standard form on input: converted to Montgomery here, so the kernel's conversion gives them back) or, with
// coef null, the vectors' own entries below nh; tail: k x tstride scalars (standard form).
int t_quotient_store(const uint32_t* coef_std, uint32_t cstride, uint32_t nh, uint32_t n_ptd, const uint32_t* tail_std,
                     uint32_t tstride, uint32_t k, uint32_t* vec_std, uint32_t stride, uint32_t off) {
  std::vector<Fr> coef(coef_std ? (size_t)k * cstride : 0), tail((size_t)k * tstride), vec((size_t)k * stride);
  for (size_t i = 0; i < coef.size(); i++) coef[i] = load_std<Fr>(coef_std + 8 * i);
  std::memcpy(tail.data(), tail_std, tail.size() * sizeof(Fr));
  std::memcpy(vec.data(), vec_std, vec.size() * sizeof(Fr));
  const uint32_t total = k * (n_ptd + 1);
  run_threads(cdiv(total, 256), 256, [&] {
    k_quotient_store(coef_std ? coef.data() : nullptr, cstride, nh, n_ptd, tail.data(), tstride, total, vec.data() + off, stride);
  });
  std::memcpy(vec_std, vec.data(), vec.size() * sizeof(Fr));
  return 0;
}
}
