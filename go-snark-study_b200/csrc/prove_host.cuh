// Prove-path orchestration: groth16.GenerateProofs (groth16/groth16.go:225-278)
// and snark.GenerateProofs (snark.go:254-289) as a fixed sequence of MSM launches,
// one exact polynomial division and a tiny finalisation kernel — all enqueued on
// one stream, one host synchronisation per proof.
//
// Included inside capi.cu's anonymous namespace (uses its context globals).
//
// Groth16 algebra (DESIGN.md §4).  With pk base sets extended by the blinding
// points, the reference's
//     PiA  = sum w_i At_i + Alpha + r*Delta                       (:243,253-255)
//     piB1 = sum w_i B1_i + Beta1 + s*Delta                       (:244,259-262)
//     PiB  = sum w_i B2_i + Beta2 + s*Delta2                      (:245,260-264)
//     PiC  = sum_{i>l} w_i C_i + sum h_i PTD_i + s*PiA + r*piB1 - rs*Delta   (:248-275)
// become four MSMs, the first three over ONE scalar vector W = w ++ [1, r, s] (O = infinity):
//     A-set  = At ++ [Alpha, Delta,  O     ]
//     B1-set = B1 ++ [Beta1, O,      Delta ]
//     B2-set = B2 ++ [Beta2, O,      Delta2]
//     CH-set = C[l+1..m) ++ PTD ++ [Delta]   scalars  w[l+1..m) ++ h ++ 0.. ++ [-rs]
// so the digit recode + counting sort of W is done once and shared by A, B1 and B2
// (the sorted entry list depends only on the scalars).  The two variable-base
// products s*PiA and r*piB1 run on a side stream while B2 / CH are still accumulating.
//
// Streams: the four bucket phases are independent, so they are issued on four streams
// (caller's + 3 side streams): the latency-bound tails (bucket reduction, tree sum) of
// one MSM overlap the throughput-bound accumulation of the others.

// A key's scratch for batches of up to k proofs (b200_groth16_prove_witness_batch, b200_pinocchio_prove_witness_batch):
// allocated on the first batch, grown (never shrunk) by a larger one after waiting for `done`, which is recorded behind
// the key's last batch.  A Pinocchio key has no blinding, so it holds only the quotient vectors, the records and the host
// entry's buffers: its other seven scalar vectors are the caller's witnesses themselves.
struct ProveBatch {
  size_t k = 0;
  DevBuf W;          // k scalar vectors w_p ++ [1, r_p, s_p] of A, B1, B2 (stride m + 3)
  DevBuf CH;         // k scalar vectors of C||PTD: w_p[l+1..m) ++ h_p ++ 0.. ++ [-r_p s_p]; Pinocchio: of G1T, h_p ++ 0..
  DevBuf rec;        // k records per set: A, B1 (G1), B2 (G2), CH (G1), then 2k products (G1); Pinocchio: 7k G1, then k G2
  DevBuf rs;         // per proof {1, r_p, s_p, -r_p s_p}, standard form
  DevBuf glv;        // per proof GlvScalars of (s_p, r_p)
  DevBuf w_stage;    // the host entry's witnesses
  DevBuf out;        // the host entry's k proofs (48 u64 each; Pinocchio: 108)
  DevBuf parts;      // a sharded key's k partial records (1 KB each), the input of the all-gather
  uint64_t* h_out = nullptr;   // pinned landing area of the host entry: the k proofs + the error word
  cudaEvent_t ev[9] = {};
  cudaEvent_t done = nullptr;
  ProveBatch() = default;
  ProveBatch(const ProveBatch&) = delete;
  ProveBatch& operator=(const ProveBatch&) = delete;
  ~ProveBatch() {
    for (auto e : ev) if (e) cudaEventDestroy(e);
    if (done) cudaEventDestroy(done);
    if (h_out) cudaFreeHost(h_out);
  }
};
constexpr size_t kBatchProofWords = 48;

struct ProvingKey {
  int kind = 0;  // 1 Groth16, 2 Pinocchio
  size_t m = 0, npublic = 0, n_h_bases = 0;
  // Work shard of this rank (world == 1: everything).  The four MSMs are laid end to end on a line weighted
  // by cost (a G2 term ~2.8 G1 terms) and rank g takes the g-th of `world` equal pieces, so a rank holds
  // whole MSMs where it can and index ranges where it must: fewer sorts / reduction tails per rank than
  // slicing every MSM `world` ways.  set k: 0 A, 1 B1, 2 B2, 3 C||PTD.
  int rank = 0, world = 1;
  int ctx = 0;  // prove context (B200_CFG_PK_CONTEXT at load): streams, polynomial workspace and communicator of its proofs
  ProveCtx& pctx() const { return g_ctx[ctx]; }
  size_t lo[4] = {0, 0, 0, 0}, hi[4] = {0, 0, 0, 0};  // index range inside set k
  bool tail[4] = {false, false, false, false};        // this rank also holds set k's blinding points
  size_t n_c_full = 0;                                // length of the C part of the C||PTD set (m - npublic - 1)
  int sort_src[3] = {0, 1, 2};                        // set k reuses the digit sort of set sort_src[k] (same scalars)
  // every rank's cut, the set lengths, and the window bits and table rows the sets were built with: what a batch's
  // refusals are decided on, so that every rank of the shard decides them alike
  std::vector<ShardCut> cuts;
  size_t len[4] = {0, 0, 0, 0};
  int window_bits = 0, table_windows = 0;
  DevBuf s4;                                          // extra scalar vector (non-shared case)
  DevBuf h_full;              // full quotient (sharded mode)
  DevBuf gather;              // all-gathered partial records (world x 1 KB), when a communicator is active
  cudaEvent_t ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // pinned landing area of the host-pointer entry points: up to kHostProofWords words of proof + the error flags.  Pinned,
  // so the D2H copies are truly asynchronous and the call can wait for them with the library mutex released (a pageable
  // destination makes cudaMemcpyAsync block until the proof is done — under the mutex).
  uint64_t* h_out = nullptr;
  ~ProvingKey() {
    for (auto e : ev) if (e) cudaEventDestroy(e);
    if (h_out) cudaFreeHost(h_out);
  }
  std::unique_ptr<Bases> g[8];  // Groth16: A, B1, B2(G2), CH   Pinocchio: A, Ap, B(G2), Bp, C, Cp, Kp, H
  Divisor Z;
  DevBuf s1, s2, s3;   // scalar vectors
  DevBuf px, w_stage;  // px coefficients / witness staging (host-pointer entry points)
  DevBuf res;          // XYZZ results (8 x 256 B)
  DevBuf out_std;      // standard-form Jacobian outputs
  DevBuf rs;           // r, s on device (standard form)
  // error word of b200_groth16_prove_device on this key: written by the kernels, never read (see b200snark.h), so an
  // out-of-range input of one device-resident proof is reported by no later call and never by a proof on another key
  DevBuf d_err;
  // error word of the host-pointer proofs on this key: written by the proof's kernels and read back by the same call on
  // the key's main stream.  Its own word, because those calls wait with the library mutex released: a word shared with
  // a proof on another key would report one proof's error to the other.
  DevBuf d_err_sync;
  std::unique_ptr<ProveBatch> batch;   // scratch of the key's batches of proofs (null until the first batch)
};

size_t pk_device_bytes(const ProvingKey& pk) {
  size_t s = dev_bytes({&pk.Z.b_mont, &pk.Z.inv_ntt, &pk.s1, &pk.s2, &pk.s3, &pk.s4, &pk.h_full, &pk.gather, &pk.px,
                        &pk.w_stage, &pk.res, &pk.out_std, &pk.rs, &pk.d_err, &pk.d_err_sync});
  for (const auto& g : pk.g)
    if (g) s += bases_device_bytes(*g);
  if (const ProveBatch* b = pk.batch.get())
    s += dev_bytes({&b->W, &b->CH, &b->rec, &b->rs, &b->glv, &b->w_stage, &b->out, &b->parts});
  return s;
}

// Largest proof a host-pointer entry point copies out: Pinocchio's 7 G1 + 1 G2 Jacobian points.
constexpr size_t kHostProofWords = 7 * 12 + 24;

std::map<uint64_t, std::unique_ptr<ProvingKey>> g_pks;
uint64_t g_next_pk = 1;

// p <- k * p for a 256-bit standard-form scalar (MSB-first double-and-add)
template <class F>
__device__ XYZZ<F> xyzz_mul_scalar(const XYZZ<F>& p, const Fr& k) {
  XYZZ<F> r = XYZZ<F>::inf();
  bool started = false;
  for (int w = 7; w >= 0; w--) {
    uint32_t limb = k.l[w];
    for (int b = 31; b >= 0; b--) {
      uint32_t bit = (limb >> b) & 1;
      if (!started && !bit) continue;
      started = true;
      r = xyzz_dbl(r);
      if (bit) xyzz_add(r, p);
    }
  }
  return r;
}

// Partial-result record of one rank: kPartialBytes (shard_batch.cuh); `parts` holds nparts consecutive records (1 on a
// single GPU, world_size after the NCCL all-gather), summed by k_groth16_finalize_batch with k = 1.  Sharded mode: each
// rank has already folded s*A_part + r*B1_part into its C part (linear in the partial sums, so this is done per rank,
// overlapped with its other MSMs); what remains after the all-gather is three point sums: A (slot @+0), B2 (@+512),
// C (@+768).
// in place: CH part (@+768) += prod[0] + prod[1]
__global__ void k_groth16_fold_products(uint8_t* res, const XYZZ<Fq>* prod) {
  if (threadIdx.x | blockIdx.x) return;
  XYZZ<Fq> c = *reinterpret_cast<const XYZZ<Fq>*>(res + 768);
  xyzz_add(c, prod[0]);
  xyzz_add(c, prod[1]);
  *reinterpret_cast<XYZZ<Fq>*>(res + 768) = c;
}

// out[k] = Jacobian(res[k]) for the 7 G1 results and the G2 result of Pinocchio
__global__ void k_pinocchio_finalize(const uint8_t* res, Fq* out_g1, Fq2* out_b) {
  uint32_t t = threadIdx.x;
  if (t < 7) store_jacobian_std(*reinterpret_cast<const XYZZ<Fq>*>(res + 256 * t), out_g1 + 3 * t);
  if (t == 32) store_jacobian_std(*reinterpret_cast<const XYZZ<Fq2>*>(res + 256 * 7), out_b);
}

// host: concatenate Jacobian point arrays (words per point = 12 or 24)
struct PointCat {
  std::vector<uint64_t> v;
  size_t words;
  explicit PointCat(size_t w) : words(w) {}
  void add(const uint64_t* p, size_t n) { v.insert(v.end(), p, p + n * words); }
  size_t count() const { return v.size() / words; }
};

// Where the points of a key's base sets come from when they are minted on the device (setup into a resident key) instead
// of read from the host arrays of b200_*_pk_load: the standard-form scalars of k_groth16_setup_scalars /
// k_pinocchio_setup_scalars in their layouts (setup_host.cuh), each set's slice being a contiguous range there, the
// generator tables (built once per call), the Groth16 tail scalars Kalpha, Kbeta, Kdelta (standard form), and Z.
struct MintSource {
  const Fr* g1 = nullptr;
  const Fr* g2 = nullptr;
  const FixedBaseTable<Fq>* gen1 = nullptr;
  const FixedBaseTable<Fq2>* gen2 = nullptr;
  Fr alpha{}, beta{}, delta{};
  const Fr* d_z = nullptr;   // standard-form coefficients on the device
};

// A base set of cnt scalars src[0..cnt) (device) ++ `tail` (host; only when with_tail) minted into its table's row 0.
// Transient device memory: the n scalars here and bases_create's XYZZ state, freed before the next set.
template <class F>
int mint_set(const FixedBaseTable<F>& gen, const Fr* src, size_t cnt, bool with_tail, std::initializer_list<Fr> tail, int c,
             int group, std::unique_ptr<Bases>& out, bool prefer_affine) {
  const size_t nt = with_tail ? tail.size() : 0, n = cnt + nt;
  if (n == 0) return fail(B200_EINVAL, "bases_load: bad arguments");
  DevBuf sc;
  CU(sc.alloc(n * sizeof(Fr)));
  if (cnt) CU(cudaMemcpyAsync(sc.p, src, cnt * sizeof(Fr), cudaMemcpyDeviceToDevice, g_ctx[0].main));
  if (nt) CU(cudaMemcpyAsync(sc.as<Fr>() + cnt, tail.begin(), nt * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  return bases_create<F>(nullptr, n, c, group, out, prefer_affine, &gen, sc.as<Fr>());
}

int pk_common_init(ProvingKey& pk, const uint64_t* z, size_t nz, size_t m, const Fr* d_z = nullptr) {
  if ((!z && !d_z) || nz == 0) return fail(B200_EINVAL, "pk_load: missing Z");
  pk.ctx = g_pk_ctx;
  int rc = divisor_init(pk.Z, z, nz, d_z);
  if (rc) return rc;
  CU(pk.s1.alloc((m + 4) * sizeof(Fr)));
  CU(pk.s2.alloc((m + 4) * sizeof(Fr)));
  CU(pk.res.alloc(8 * 256));
  CU(pk.out_std.alloc(64 * sizeof(Fq)));
  CU(pk.rs.alloc(8 * sizeof(Fr)));
  for (DevBuf* e : {&pk.d_err, &pk.d_err_sync}) {
    CU(e->alloc(sizeof(int)));
    CU(cudaMemset(e->p, 0, sizeof(int)));
  }
  for (auto& e : pk.ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  CU(cudaHostAlloc(reinterpret_cast<void**>(&pk.h_out), (kHostProofWords + 1) * sizeof(uint64_t), cudaHostAllocDefault));
  return check_err_flag("pk_load(Z)", g_d_err);
}

int groth16_pk_load(const uint64_t* at, const uint64_t* b1, const uint64_t* b2, const uint64_t* bacdelta, size_t m,
                    const uint64_t* ptd, size_t n_ptd, const uint64_t* z, size_t nz, const uint64_t* alpha1,
                    const uint64_t* beta1, const uint64_t* delta1, const uint64_t* beta2, const uint64_t* delta2,
                    size_t npublic, int c, int rank, int world, b200_pk_t* out, const MintSource* mint = nullptr) {
  if ((!mint && (!at || !b1 || !b2 || !bacdelta || !ptd || !alpha1 || !beta1 || !delta1 || !beta2 || !delta2)) || !out)
    return fail(B200_EINVAL, "groth16_pk_load: null pointer");
  if (m == 0 || npublic + 1 > m || n_ptd == 0) return fail(B200_EINVAL, "groth16_pk_load: bad sizes");
  if (world < 1 || rank < 0 || rank >= world) return fail(B200_EINVAL, "groth16_pk_load: bad shard %d/%d", rank, world);
  auto pk = std::make_unique<ProvingKey>();
  pk->kind = 1;
  pk->m = m;
  pk->npublic = npublic;
  pk->n_h_bases = n_ptd;
  int rc = pk_common_init(*pk, z, nz, m, mint ? mint->d_z : nullptr);
  if (rc) return rc;
  pk->rank = rank;
  pk->world = world;
  const size_t l1 = npublic + 1;
  const size_t n_c_full = pk->n_c_full = m - l1;
  // Cost weights of the line partition, in G1 terms of the C||PTD set: a G2 term (B2), and a term of A / B1 — whose ranks
  // also pay the two GLV products s*A_part + r*B1_part (single-warp latency) on their critical path when sharded.
  const double w_ab = world > 1 ? g_w_ab / 100.0 : 1.0;
  const double wgt[4] = {w_ab, w_ab, g_w_g2 / 100.0, 1.0};
  G16Plan plan = groth16_set_plan(m, npublic, n_ptd, wgt, rank, world);   // equal pieces of the weighted line
  pk->window_bits = c;
  pk->table_windows = g_table_windows;
  for (int k = 0; k < 4; k++) {
    pk->len[k] = plan.len[k];
    pk->lo[k] = plan.cuts[(size_t)rank].lo[k];
    pk->hi[k] = plan.cuts[(size_t)rank].hi[k];
    pk->tail[k] = plan.tail[k];
  }
  // a set whose end falls exactly on a cut: the rank holding its last element owns the tail (shard_holds_tail);
  // if no rank holds elements of it (len == 0) the last rank does.
  // Accumulation kernel per SET of this rank.  The batched-affine tree pays off once a set is large enough to amortise its
  // per-round launches (G2 sets earlier than G1 sets); below g_aff_min_g1 / g_aff_min_g2 terms a shard takes the XYZZ
  // kernel, whose single launch has the shorter latency chain.  A single-GPU key always takes the affine tree: its four
  // MSMs cover each other's gaps.
  auto set_terms = [&](int k) { return (double)(pk->hi[k] - pk->lo[k]); };
  auto affine_for = [&](int k) { return world == 1 || set_terms(k) >= (double)(k == 2 ? g_aff_min_g2 : g_aff_min_g1); };
  // Each set from the host arrays, or minted: its slice of the setup's scalars (C||PTD: BACDelta[l1..m) ++ PTD is one
  // range there), then the scalars of its tail (0 for an infinity).
  static const uint64_t inf1[12] = {0}, inf2[24] = {0};
  auto has = [&](int k) { return pk->lo[k] < pk->hi[k] || pk->tail[k]; };
  const Fr o = Fr::zero();
  auto cnt = [&](int k) { return pk->hi[k] - pk->lo[k]; };
  if (has(0)) {
    if (mint) {
      rc = mint_set<Fq>(*mint->gen1, mint->g1 + pk->lo[0], cnt(0), pk->tail[0], {mint->alpha, mint->delta, o}, c, 1, pk->g[0], affine_for(0));
    } else {
      PointCat cat(12);
      cat.add(at + 12 * pk->lo[0], cnt(0));
      if (pk->tail[0]) { cat.add(alpha1, 1); cat.add(delta1, 1); cat.add(inf1, 1); }
      rc = bases_create<Fq>(cat.v.data(), cat.count(), c, 1, pk->g[0], affine_for(0));
    }
    if (rc) return rc;
  }
  if (has(1)) {
    if (mint) {
      rc = mint_set<Fq>(*mint->gen1, mint->g1 + m + pk->lo[1], cnt(1), pk->tail[1], {mint->beta, o, mint->delta}, c, 1, pk->g[1], affine_for(1));
    } else {
      PointCat cat(12);
      cat.add(b1 + 12 * pk->lo[1], cnt(1));
      if (pk->tail[1]) { cat.add(beta1, 1); cat.add(inf1, 1); cat.add(delta1, 1); }
      rc = bases_create<Fq>(cat.v.data(), cat.count(), c, 1, pk->g[1], affine_for(1));
    }
    if (rc) return rc;
  }
  if (has(2)) {
    if (mint) {
      rc = mint_set<Fq2>(*mint->gen2, mint->g2 + pk->lo[2], cnt(2), pk->tail[2], {mint->beta, o, mint->delta}, c, 2, pk->g[2], affine_for(2));
    } else {
      PointCat cat(24);
      cat.add(b2 + 24 * pk->lo[2], cnt(2));
      if (pk->tail[2]) { cat.add(beta2, 1); cat.add(inf2, 1); cat.add(delta2, 1); }
      rc = bases_create<Fq2>(cat.v.data(), cat.count(), c, 2, pk->g[2], affine_for(2));
    }
    if (rc) return rc;
  }
  if (has(3)) {
    if (mint) {
      rc = mint_set<Fq>(*mint->gen1, mint->g1 + 2 * m + l1 + pk->lo[3], cnt(3), pk->tail[3], {mint->delta}, c, 1, pk->g[3], affine_for(3));
    } else {
      PointCat cat(12);
      size_t lo3 = pk->lo[3], hi3 = pk->hi[3];
      size_t c_lo = lo3 < n_c_full ? lo3 : n_c_full, c_hi = hi3 < n_c_full ? hi3 : n_c_full;
      size_t p_lo = lo3 > n_c_full ? lo3 - n_c_full : 0, p_hi = hi3 > n_c_full ? hi3 - n_c_full : 0;
      cat.add(bacdelta + 12 * (l1 + c_lo), c_hi - c_lo);
      cat.add(ptd + 12 * p_lo, p_hi - p_lo);
      if (pk->tail[3]) cat.add(delta1, 1);
      rc = bases_create<Fq>(cat.v.data(), cat.count(), c, 1, pk->g[3], affine_for(3));
    }
    if (rc) return rc;
  }
  // sets that consume identical scalar slices into the same table rows share one digit sort
  for (int k = 1; k < 3; k++)
    for (int j = 0; j < k; j++)
      if (pk->sort_src[k] == k && pk->lo[k] == pk->lo[j] && pk->hi[k] == pk->hi[j] && pk->tail[k] == pk->tail[j] && affine_for(k) == affine_for(j) &&
          (pk->lo[k] < pk->hi[k] || pk->tail[k]) && pk->g[k]->sh.rows == pk->g[j]->sh.rows)
        pk->sort_src[k] = pk->sort_src[j];
  CU(pk->s3.alloc((m + n_ptd + 4) * sizeof(Fr)));
  CU(pk->s4.alloc((m + 4) * sizeof(Fr)));
  if (world > 1) CU(pk->h_full.alloc((m + n_ptd + 4) * sizeof(Fr)));
  pk->cuts = std::move(plan.cuts);
  uint64_t h = g_next_pk++;
  g_pks[h] = std::move(pk);
  *out = h;
  return B200_OK;
}

ProvingKey* find_pk(b200_pk_t h, int kind) {
  auto it = g_pks.find(h);
  if (it == g_pks.end() || it->second->kind != kind) return nullptr;
  return it->second.get();
}

// One rank's part of a Groth16 proof: set j in {A, B1, B2} reads w[lo_j, hi_j), ++ [1, r, s] when the rank holds the
// set's tail; C||PTD reads w[l1 + c_lo, l1 + c_lo + n_c) ++ h[p_lo, p_lo + n_p), ++ [-r s] with the tail.  terms[j]: the
// length of set j's scalar vector, 0 if the rank holds none of it (one GPU: m + 3, and n_c_full + len(PTD) + 1).
// Computed from the cuts of any rank, so every rank can size every rank's part.
struct G16Slices {
  size_t lo[4], hi[4], terms[4];
  bool tail[4];
  size_t c_lo, n_c, p_lo, n_p;
};
G16Slices g16_slices(const ProvingKey* pk, int rank) {
  G16Slices sl{};
  const ShardCut& ct = pk->cuts[(size_t)rank];
  for (int j = 0; j < 4; j++) {
    sl.lo[j] = ct.lo[j];
    sl.hi[j] = ct.hi[j];
    sl.tail[j] = shard_holds_tail(sl.lo[j], sl.hi[j], pk->len[j], rank, pk->world);
    sl.terms[j] = sl.hi[j] - sl.lo[j] + (sl.tail[j] ? (j < 3 ? 3 : 1) : 0);
  }
  const size_t ncf = pk->n_c_full;
  sl.c_lo = std::min(sl.lo[3], ncf);
  sl.n_c = std::min(sl.hi[3], ncf) - sl.c_lo;
  sl.p_lo = sl.lo[3] > ncf ? sl.lo[3] - ncf : 0;
  sl.n_p = (sl.hi[3] > ncf ? sl.hi[3] - ncf : 0) - sl.p_lo;
  return sl;
}
// Where the A / B1 / B2 vectors of a batch live in its W: per proof, one vector per digit sort (sets that share a sort
// share its vector), vector j of proof p at W + k*woff[j] + p*terms[j].  Returns the scalars per proof (one GPU: m + 3).
size_t g16_w_layout(const ProvingKey* pk, const G16Slices& sl, size_t woff[3]) {
  size_t total = 0;
  for (int j = 0; j < 3; j++) {
    woff[j] = 0;
    if (!pk->g[j]) continue;
    if (pk->sort_src[j] == j) {
      woff[j] = total;
      total += sl.terms[j];
    } else {
      woff[j] = woff[pk->sort_src[j]];
    }
  }
  return total;
}

// Grows the key's batch scratch to k proofs (host: also the host entry's witness staging, proof buffer and pinned landing
// area).  A regrowth first waits for the key's last batch (its `done` event), not for the device.  A sharded key's
// vectors are those of its own part (G16Slices), and it keeps k partial records for the all-gather.
int groth16_batch_scratch(ProvingKey* pk, size_t k, bool host) {
  if (!pk->batch) {
    auto b = std::make_unique<ProveBatch>();
    for (auto& e : b->ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming));
    pk->batch = std::move(b);
  }
  ProveBatch& b = *pk->batch;
  const size_t m = pk->m;
  const G16Slices sl = g16_slices(pk, pk->rank);
  size_t woff[3];
  const size_t nw = g16_w_layout(pk, sl, woff), nch = pk->g[3] ? sl.terms[3] : 0;
  const bool grow_host = host && b.out.bytes < k * kBatchProofWords * sizeof(uint64_t);
  if (b.k < k || grow_host) CU(cudaEventSynchronize(b.done));
  if (b.k < k) {
    CU(b.W.alloc(k * nw * sizeof(Fr)));
    CU(b.CH.alloc(k * nch * sizeof(Fr)));
    CU(b.rec.alloc(k * (5 * sizeof(XYZZ<Fq>) + sizeof(XYZZ<Fq2>))));
    CU(b.rs.alloc(k * 4 * sizeof(Fr)));
    CU(b.glv.alloc(k * sizeof(GlvScalars)));
    if (pk->world > 1) CU(b.parts.alloc(k * kPartialBytes));
    b.k = k;
  }
  if (grow_host) {
    CU(b.w_stage.alloc(k * m * sizeof(Fr)));
    CU(b.out.alloc(k * kBatchProofWords * sizeof(uint64_t)));
    if (b.h_out) CU(cudaFreeHost(b.h_out));
    b.h_out = nullptr;
    CU(cudaHostAlloc(reinterpret_cast<void**>(&b.h_out), (k * kBatchProofWords + 1) * sizeof(uint64_t), cudaHostAllocDefault));
  }
  return B200_OK;
}

// host F_r helpers for the blinding scalars (the reference does this with big.Int, groth16.go:274)
Fr fr_load_std(const uint64_t* v) {
  Fr r;
  memcpy(&r, v, sizeof(Fr));
  return r;
}

// ---- blinding products s*A and r*B1 (groth16.go:272-273): GLV half-warps (glv.cuh) -----------------------------
// One warp, all 32 lanes: lanes 0..15 -> prod[0] = s*A, lanes 16..31 -> prod[1] = r*B1 (the partial record layout, shard_batch.cuh).
__global__ void k_groth16_products(const uint8_t* res, GlvScalars g, XYZZ<Fq>* prod) {
  const uint32_t t = threadIdx.x & 31u;
  const uint32_t grp = t >> 4;
  Jacobian<Fq> p = xyzz_to_jacobian(*reinterpret_cast<const XYZZ<Fq>*>(res + (grp ? 256 : 0)));
  Jacobian<Fq> r = glv_mul_halfwarp(p, g.k[grp], g.neg[grp], t);
  if ((t & 15u) == 0) prod[grp] = jacobian_to_xyzz(r);
}
__global__ void k_groth16_combine(const uint8_t* res, const XYZZ<Fq>* prod, Fq* out_a, Fq* out_c, Fq2* out_b) {
  uint32_t t = threadIdx.x;
  if (t == 0) {
    XYZZ<Fq> c = *reinterpret_cast<const XYZZ<Fq>*>(res + 768);
    xyzz_add(c, prod[0]);
    xyzz_add(c, prod[1]);
    store_jacobian_std(c, out_c);
  }
  if (t == 32) store_jacobian_std(*reinterpret_cast<const XYZZ<Fq>*>(res), out_a);
  if (t == 64) store_jacobian_std(*reinterpret_cast<const XYZZ<Fq2>*>(res + 512), out_b);
}

// ---- batches of k proofs under one key (b200_groth16_prove_witness_batch) ----------------------------------------------
// The batched MSMs leave k records per set: rA[p], rB1[p], rB2[p], rCH[p].  Block p: the warp of k_groth16_products for
// proof p, prod[2p] = s_p * A_p and prod[2p+1] = r_p * B1_p.
__global__ void k_groth16_products_batch(const XYZZ<Fq>* rA, const XYZZ<Fq>* rB1, const GlvScalars* g, XYZZ<Fq>* prod) {
  const uint32_t t = threadIdx.x & 31u, p = blockIdx.x;
  const uint32_t grp = t >> 4;
  Jacobian<Fq> pt = xyzz_to_jacobian(grp ? rB1[p] : rA[p]);
  Jacobian<Fq> r = glv_mul_halfwarp(pt, g[p].k[grp], g[p].neg[grp], t);
  if ((t & 15u) == 0) prod[2 * p + grp] = jacobian_to_xyzz(r);
}
// Thread 3p + j of k proofs: j = 0 PiC_p = CH_p + prod[2p] + prod[2p+1], j = 1 PiA_p, j = 2 PiB_p; proof p at out + 48p
// (u64), PiA | PiC | PiB as in k_groth16_combine.
__global__ void k_groth16_combine_batch(const XYZZ<Fq>* rA, const XYZZ<Fq2>* rB2, const XYZZ<Fq>* rCH, const XYZZ<Fq>* prod,
                                        uint32_t k, Fq* out) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 3 * k) return;
  const uint32_t p = e / 3, j = e - 3 * p;
  Fq* o = out + 12 * (size_t)p;   // 48 u64 = 12 Fq per proof
  if (j == 0) {
    XYZZ<Fq> c = rCH[p];
    xyzz_add(c, prod[2 * p]);
    xyzz_add(c, prod[2 * p + 1]);
    store_jacobian_std(c, o + 3);
  } else if (j == 1) {
    store_jacobian_std(rA[p], o);
  } else {
    store_jacobian_std(rB2[p], reinterpret_cast<Fq2*>(o + 6));
  }
}


#define EV_REC(e, stream) CU(cudaEventRecord((e), (stream)))
#define EV_WAIT(stream, e) CU(cudaStreamWaitEvent((stream), (e), 0))

// Enqueue one Groth16 proof on `st` from DEVICE-resident witness / px (standard
// form).  d_out receives PiA (3 Fq) | PiC (3 Fq) | PiB (3 Fq2) in standard form
// (or, for a sharded key, the 1 KB partial record).  No host synchronisation.  A witness entry or px coefficient >= r
// is read as 0 and sets bit 1 of *err.
int groth16_enqueue(ProvingKey* pk, const Fr* d_w, size_t nw, const Fr* d_px, size_t npx, const uint64_t* r,
                    const uint64_t* s, Fq* d_out, cudaStream_t st, int* err, int px_mont = 0, const Fr* d_h_std = nullptr) {
  // d_h_std != nullptr: the quotient h (npx - len(Z) + 1 coefficients, standard form, device) is supplied by the caller
  // (witness path: qap_h_enqueue on side stream 3) and the division is skipped; d_px is then unused.
  size_t m = pk->m;
  if (nw != m) return fail(B200_EINVAL, "groth16_prove: witness length %zu != NVars %zu", nw, m);
  if (npx < pk->Z.nb) return fail(B200_EINVAL, "groth16_prove: len(px) < len(Z)");
  size_t nq = npx - pk->Z.nb + 1;
  // groth16.go:269-270 indexes PowersTauDelta[i] for i < len(hx): out of range panics in the reference
  if (nq > pk->n_h_bases)
    return fail(B200_EINVAL, "groth16_prove: len(hx)=%zu exceeds len(PowersTauDelta)=%zu", nq, pk->n_h_bases);
  Fr fr_r = fr_load_std(r), fr_s = fr_load_std(s);
  if (fr_r.geq_modulus() || fr_s.geq_modulus()) return fail(B200_ERANGE, "groth16_prove: r or s >= field order");
  Fr neg_rs = (fr_r.to_mont() * fr_s.to_mont()).neg().from_mont();  // -(r*s) mod r  (groth16.go:274)
  Fr one = Fr::zero();
  one.l[0] = 1;
  cudaStream_t s1 = pk->pctx().side[0], s2 = pk->pctx().side[1], s3 = pk->pctx().side[2];
  if (g_serial) s1 = s2 = s3 = st;  // measurement mode (b200_profile bit 1): no overlap, exclusive kernel timings
  cudaEvent_t e_in = pk->ev[0], e_w = pk->ev[1], e_a = pk->ev[2], e_b1 = pk->ev[3], e_b2 = pk->ev[4],
              e_ch = pk->ev[5], e_prod = pk->ev[6];
  const size_t l1 = pk->npublic + 1, n_c_full = pk->n_c_full;
  uint8_t* res = pk->res.as<uint8_t>();
  int rc;
  Fr small[6] = {one, fr_r, fr_s, neg_rs, fr_r, fr_s};
  CU(cudaMemcpyAsync(pk->rs.p, small, sizeof small, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(res, 0, kPartialBytes, st));      // sets this rank does not hold contribute infinity
  // scalar vectors: set k in {A, B1, B2} uses w[lo_k, hi_k) (+ [1, r, s] when it owns the blinding points)
  Fr* sv[3] = {pk->s1.as<Fr>(), pk->s2.as<Fr>(), pk->s4.as<Fr>()};
  size_t nterm[4] = {0, 0, 0, 0};
  for (int k = 0; k < 3; k++) {
    if (!pk->g[k]) continue;
    if (pk->sort_src[k] != k) { nterm[k] = nterm[pk->sort_src[k]]; continue; }   // shares the sort of an identical slice
    size_t cnt = pk->hi[k] - pk->lo[k];
    if (cnt) CU(cudaMemcpyAsync(sv[k], d_w + pk->lo[k], cnt * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    if (pk->tail[k]) CU(cudaMemcpyAsync(sv[k] + cnt, pk->rs.as<Fr>(), 3 * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    nterm[k] = cnt + (pk->tail[k] ? 3 : 0);
  }
  // C || PTD set
  Fr* sCH = pk->s3.as<Fr>();
  size_t lo3 = pk->lo[3], hi3 = pk->hi[3];
  size_t c_lo = lo3 < n_c_full ? lo3 : n_c_full, c_hi = hi3 < n_c_full ? hi3 : n_c_full;
  size_t p_lo = lo3 > n_c_full ? lo3 - n_c_full : 0, p_hi = hi3 > n_c_full ? hi3 - n_c_full : 0;
  size_t n_c = c_hi - c_lo, n_p = p_hi - p_lo;
  if (pk->g[3]) {
    if (n_c) CU(cudaMemcpyAsync(sCH, d_w + l1 + c_lo, n_c * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    if (pk->tail[3]) CU(cudaMemcpyAsync(sCH + n_c + n_p, pk->rs.as<Fr>() + 3, sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    nterm[3] = n_c + n_p + (pk->tail[3] ? 1 : 0);
  }
  EV_REC(e_in, st);
  // --- side stream 3: hx = px / Z (groth16.go:266) when this rank holds PowersTauDelta points, then C||PTD.
  // Single GPU: h is written straight into the scalar vector.  Sharded: the rank(s) holding PTD indices repeat
  // the (cheap) division and keep h[p_lo, p_hi) — no inter-GPU traffic (SURVEY §8e).
  EV_WAIT(s3, e_in);
  if (pk->g[3]) {
    if (n_p) {
      bool direct = p_lo == 0 && nq <= n_p;
      Fr* h_dst = direct ? sCH + n_c : pk->h_full.as<Fr>();
      if (!direct && !pk->h_full.p) CU(pk->h_full.alloc((pk->m + pk->n_h_bases + 4) * sizeof(Fr)));
      if (d_h_std) CU(cudaMemcpyAsync(h_dst, d_h_std, nq * sizeof(Fr), cudaMemcpyDeviceToDevice, s3));
      else CU(poly_div_device(*pk->pctx().poly, pk->Z, d_px, npx, px_mont, h_dst, nullptr, err, s3));
      size_t have = nq > p_lo ? (nq < p_hi ? nq - p_lo : n_p) : 0;   // valid h coefficients inside [p_lo, p_hi)
      if (!direct && have)
        CU(cudaMemcpyAsync(sCH + n_c, pk->h_full.as<Fr>() + p_lo, have * sizeof(Fr), cudaMemcpyDeviceToDevice, s3));
      if (n_p > have) CU(cudaMemsetAsync(sCH + n_c + have, 0, (n_p - have) * sizeof(Fr), s3));
    }
    if ((rc = msm_enqueue<Fq>(pk->g[3].get(), sCH, nterm[3], 0, reinterpret_cast<XYZZ<Fq>*>(res + 768), err, s3))) return rc;
  }
  EV_REC(e_ch, s3);
  // --- A, B1, B2.  Sets that consume identical scalar slices (all three on one GPU; A and B1 on a rank that
  // holds both whole) share ONE digit sort; the sort runs on the main stream, the bucket phases fan out.
  XYZZ<Fq>* rA = reinterpret_cast<XYZZ<Fq>*>(res);
  XYZZ<Fq>* rB1 = reinterpret_cast<XYZZ<Fq>*>(res + 256);
  XYZZ<Fq2>* rB2 = reinterpret_cast<XYZZ<Fq2>*>(res + 512);
  cudaStream_t sk[3] = {st, s1, s2};
  cudaEvent_t e_sorted[3] = {e_w, pk->ev[7], e_prod};   // e_prod is re-recorded later; safe: waits are enqueued first
  for (int k = 0; k < 3; k++) {
    if (!pk->g[k] || pk->sort_src[k] != k) continue;
    if ((rc = msm_sort(pk->g[k]->sort, pk->g[k]->sh, sv[k], nterm[k], 0, err, st))) return rc;
    EV_REC(e_sorted[k], st);
  }
  for (int k = 2; k >= 0; k--) {   // B2 first: it is the longest
    if (!pk->g[k]) continue;
    int src = pk->sort_src[k];
    if (sk[k] != st) EV_WAIT(sk[k], e_sorted[src]);
    size_t nt = nterm[src];
    if (k == 0) rc = msm_buckets<Fq>(pk->g[0].get(), pk->g[src]->sort, nt, rA, sk[0]);
    else if (k == 1) rc = msm_buckets<Fq>(pk->g[1].get(), pk->g[src]->sort, nt, rB1, sk[1]);
    else rc = msm_buckets<Fq2>(pk->g[2].get(), pk->g[src]->sort, nt, rB2, sk[2]);
    if (rc) return rc;
  }
  EV_REC(e_a, st);
  EV_REC(e_b1, s1);
  EV_REC(e_b2, s2);
  // s*A_part and r*B1_part (groth16.go:272-273; linear, so each rank does its own parts) on side stream 1
  // while B2 / C||PTD are still running
  XYZZ<Fq>* prod = reinterpret_cast<XYZZ<Fq>*>(res + 1024);
  EV_WAIT(s1, e_a);
  GlvScalars glv;
  if (glv_decompose(fr_s, glv.k[0], glv.neg[0]) || glv_decompose(fr_r, glv.k[1], glv.neg[1]))
    return fail(B200_EINVAL, "groth16_prove: GLV decomposition out of range");
  if (pk->g[0] || pk->g[1]) {
    k_groth16_products<<<1, 32, 0, s1>>>(res, glv, prod);
  } else {   // a rank that holds no part of A or B1: both products are the point at infinity (all-zero XYZZ) — skip the
    // single-warp chain (it would sit on the critical path of most ranks of an 8-way proof)
    CU(cudaMemsetAsync(prod, 0, 2 * sizeof(XYZZ<Fq>), s1));
  }
  EV_REC(e_prod, s1);
  EV_WAIT(st, e_prod);
  EV_WAIT(st, e_b2);
  EV_WAIT(st, e_ch);
  if (pk->world == 1) {
    k_groth16_combine<<<1, 96, 0, st>>>(res, prod, d_out, d_out + 3, reinterpret_cast<Fq2*>(d_out + 6));
  } else {  // fold the products into this rank's C part; the 1 KB partial record goes to the all-gather
    k_groth16_fold_products<<<1, 32, 0, st>>>(res, prod);
    if (comm_active() && g_comm.world == pk->world) {
      if (g_comm.rank != pk->rank) return fail(B200_EINVAL, "groth16_prove: key shard %d on communicator rank %d", pk->rank, g_comm.rank);
      CU(pk->gather.ensure(kPartialBytes * (size_t)pk->world));
      ncclResult_t nrc = g_comm.api.AllGather(res, pk->gather.p, kPartialBytes, ncclUint8, pk->pctx().comm, st);
      if (nrc != ncclSuccess) return fail(B200_ECOMM, "ncclAllGather: %s", g_comm.api.GetErrorString(nrc));
      k_groth16_finalize_batch<<<groth16_finalize_blocks(1), kG16FinalizeBlock, 0, st>>>(pk->gather.as<uint8_t>(), pk->world, 1, d_out);
      g_launches += 2;
    } else {
      CU(cudaMemcpyAsync(d_out, res, kPartialBytes, cudaMemcpyDeviceToDevice, st));
    }
  }
  g_launches += 3;
  CU(cudaGetLastError());
  return B200_OK;
}

// Sharded mode, after the all-gather: sum the `world` partial records and finish the proof.
int groth16_finalize_enqueue(ProvingKey* pk, const uint8_t* d_parts, int nparts, const uint64_t* r, const uint64_t* s,
                             Fq* d_out, cudaStream_t st) {
  (void)pk; (void)r; (void)s;  // r, s were consumed per rank (their products are already inside the C parts)
  k_groth16_finalize_batch<<<groth16_finalize_blocks(1), kG16FinalizeBlock, 0, st>>>(d_parts, nparts, 1, d_out);
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}

// This rank's C||PTD slice reaches into PowersTauDelta, so its proof needs the quotient h (always, on one GPU).
bool pk_needs_px(const ProvingKey* pk) { return pk->hi[3] > pk->n_c_full; }

// Host-pointer entry points: refuse a sharded key unless the proof can be finished inside the call.
int check_sharded_host_call(const ProvingKey* pk, const char* what, const char* device_entry) {
  if (pk->world != 1 && !(comm_active() && g_comm.world == pk->world))
    return fail(B200_EINVAL, "%s: sharded key (rank %d/%d) without a matching communicator: call b200_comm_init, "
                             "or use %s + b200_groth16_finalize_device around your own all-gather",
                what, pk->rank, pk->world, device_entry);
  return B200_OK;
}

// Upload the host witness into pk->w_stage on `st`: all of it, or only the index ranges this rank's MSMs read.  dst:
// nwit witnesses (row-major, m scalars each) into dst instead, each staged alike (a batch's).
int stage_witness(ProvingKey* pk, const uint64_t* w, bool all, cudaStream_t st, Fr* dst = nullptr, size_t nwit = 1) {
  if (!dst) {
    CU(pk->w_stage.ensure(pk->m * sizeof(Fr)));
    dst = pk->w_stage.as<Fr>();
  }
  const Fr* src = reinterpret_cast<const Fr*>(w);
  const size_t pitch = pk->m * sizeof(Fr);
  auto upload = [&](size_t lo, size_t cnt) {
    return nwit == 1 ? cudaMemcpyAsync(dst + lo, src + lo, cnt * sizeof(Fr), cudaMemcpyHostToDevice, st)
                     : cudaMemcpy2DAsync(dst + lo, pitch, src + lo, pitch, cnt * sizeof(Fr), nwit, cudaMemcpyHostToDevice, st);
  };
  if (all) {
    CU(upload(0, pk->m));
    return B200_OK;
  }
  const size_t l1 = pk->npublic + 1, ncf = pk->n_c_full;
  size_t lo[4], hi[4];
  for (int k = 0; k < 3; k++) { lo[k] = pk->lo[k]; hi[k] = pk->hi[k]; }
  size_t c_lo = pk->lo[3] < ncf ? pk->lo[3] : ncf, c_hi = pk->hi[3] < ncf ? pk->hi[3] : ncf;
  lo[3] = l1 + c_lo;
  hi[3] = l1 + c_hi;
  for (int k = 0; k < 4; k++) {
    if (lo[k] >= hi[k]) continue;
    bool dup = false;
    for (int j = 0; j < k; j++) dup = dup || (lo[j] <= lo[k] && hi[k] <= hi[j] && lo[j] < hi[j]);
    if (dup) continue;
    CU(upload(lo[k], hi[k] - lo[k]));
  }
  return B200_OK;
}

// Copy the proof out to the key's pinned landing area, read the key's d_err_sync behind it and wait (with `lk`: the wait
// runs with the library mutex released), then split the proof into the caller's arrays: `outs` lists each array and its
// word count, in the order of the device layout.
int finish_host_proof(ProvingKey* pk, const Fq* d_proof, const char* what, cudaStream_t st, std::unique_lock<std::mutex>* lk,
                      std::initializer_list<std::pair<uint64_t*, size_t>> outs) {
  size_t words = 0;
  for (const auto& o : outs) words += o.second;
  uint64_t* host_out = pk->h_out;
  CU(cudaMemcpyAsync(host_out, d_proof, words * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  int rc = check_err_flag(what, pk->d_err_sync.as<int>(), st, lk, reinterpret_cast<int*>(host_out + kHostProofWords));
  if (rc) return rc;
  for (const auto& o : outs) {
    memcpy(o.first, host_out, o.second * sizeof(uint64_t));
    host_out += o.second;
  }
  return B200_OK;
}

int groth16_prove(b200_pk_t h, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx, const uint64_t* r,
                  const uint64_t* s, uint64_t* pi_a, uint64_t* pi_b, uint64_t* pi_c, std::unique_lock<std::mutex>* lk = nullptr) {
  ProvingKey* pk = find_pk(h, 1);
  if (!pk) return fail(B200_EINVAL, "groth16_prove: bad proving-key handle");
  if (!w || !px || !r || !s || !pi_a || !pi_b || !pi_c) return fail(B200_EINVAL, "groth16_prove: null pointer");
  if (nw != pk->m) return fail(B200_EINVAL, "groth16_prove: witness length %zu != NVars %zu", nw, pk->m);
  int rc = check_sharded_host_call(pk, "groth16_prove", "b200_groth16_prove_device");
  if (rc) return rc;
  if (npx < pk->Z.nb) return fail(B200_EINVAL, "groth16_prove: len(px) < len(Z)");
  cudaStream_t st = pk->pctx().main;   // context 1 keys: their own main stream (a second host thread's proof in flight)
  CU(pk->px.ensure(npx * sizeof(Fr)));
  // sharded: stage only what this rank reads, its witness index ranges, and px only if it holds PowersTauDelta points
  if ((rc = stage_witness(pk, w, pk->world == 1, st))) return rc;
  const bool need_px = pk_needs_px(pk);
  // px is only needed by the division on side stream 3: copy it there so the transfer overlaps the sort of w
  // (same-stream order makes the division see it; the previous proof's use of pk->px finished before its combine)
  // (measurement mode runs the division on `st`, so the copy goes there too)
  // Only the TOP len(px) - len(Z) + 1 coefficients are staged: the quotient of the division depends on nothing else
  // (poly_div_device reads rev(px) mod x^nq; the remainder is never formed on the prove path) — at 2^20 constraints that
  // is 32 MB over PCIe instead of 64 MB.  They land at their own offset, so the device layout of px is unchanged.
  if (need_px) {
    const size_t px_off = pk->Z.nb - 1;
    CU(cudaMemcpyAsync(pk->px.as<Fr>() + px_off, reinterpret_cast<const Fr*>(px) + px_off, (npx - px_off) * sizeof(Fr),
                       cudaMemcpyHostToDevice, g_serial ? st : pk->pctx().side[2]));
  }
  Fq* o = pk->out_std.as<Fq>();
  rc = groth16_enqueue(pk, pk->w_stage.as<Fr>(), nw, pk->px.as<Fr>(), npx, r, s, o, st, pk->d_err_sync.as<int>());
  if (rc) return rc;
  return finish_host_proof(pk, o, "groth16_prove", st, lk, {{pi_a, 12}, {pi_c, 12}, {pi_b, 24}});
}

// Pinocchio result slots (XYZZ, 256 B each): 0 PiA, 1 PiAp, 2 PiBp, 3 PiC, 4 PiCp, 5 PiH, 6 PiKp, 7 PiB (G2).
// Base sets g[k]: 0 A, 1 Ap, 2 B (G2), 3 Bp, 4 C, 5 Cp, 6 Kp, 7 G1T.
constexpr int kPinSlot[8] = {0, 1, 7, 2, 3, 4, 6, 5};

// Sharded mode (world > 1): whole MSMs are dealt to the ranks by pinocchio_owners (shard_partition.h).

// The world records of one proof are summed slot by slot by k_pinocchio_gather_finalize_batch (pinocchio_batch.cuh) with
// k = 1: every slot is non-infinity on exactly one rank.

int pinocchio_pk_load(const uint64_t* a, const uint64_t* ap, const uint64_t* b2, const uint64_t* bp,
                      const uint64_t* c, const uint64_t* cp, const uint64_t* kp, size_t m, const uint64_t* g1t,
                      size_t n_g1t, const uint64_t* z, size_t nz, size_t npublic, int wb, int rank, int world, b200_pk_t* out,
                      const MintSource* mint = nullptr) {
  if ((!mint && (!a || !ap || !b2 || !bp || !c || !cp || !kp || !g1t)) || !out)
    return fail(B200_EINVAL, "pinocchio_pk_load: null pointer");
  if (m == 0 || npublic + 1 > m || n_g1t == 0) return fail(B200_EINVAL, "pinocchio_pk_load: bad sizes");
  if (world < 1 || rank < 0 || rank >= world) return fail(B200_EINVAL, "pinocchio_pk_load: bad shard %d/%d", rank, world);
  auto pk = std::make_unique<ProvingKey>();
  pk->kind = 2;
  pk->m = m;
  pk->npublic = npublic;
  pk->n_h_bases = n_g1t;
  int rc = pk_common_init(*pk, z, nz, m, mint ? mint->d_z : nullptr);
  if (rc) return rc;
  size_t l1 = npublic + 1;
  pk->rank = rank;
  pk->world = world;
  pk->window_bits = wb;
  pk->table_windows = g_table_windows;
  int owner[8];
  pinocchio_owners(m, l1, n_g1t, world, owner);
  auto mine = [&](int k) { return owner[k] == rank; };
  // Set k: `cnt` points from index `first` of its host array, or minted from offset `off` of the setup's G1 / G2 scalars
  // (layout of k_pinocchio_setup_scalars).
  auto set = [&](int k, const uint64_t* pts, size_t first, size_t off, size_t cnt) {
    if (!mine(k)) return (int)B200_OK;
    if (k == 2)
      return mint ? mint_set<Fq2>(*mint->gen2, mint->g2 + off, cnt, false, {}, wb, 2, pk->g[k], true)
                  : bases_create<Fq2>(pts + 24 * first, cnt, wb, 2, pk->g[k], true);
    return mint ? mint_set<Fq>(*mint->gen1, mint->g1 + off, cnt, false, {}, wb, 1, pk->g[k], true)
                : bases_create<Fq>(pts + 12 * first, cnt, wb, 1, pk->g[k], true);
  };
  // snark.go:265-268: PiA, PiAp run over i in [NPublic+1, NVars)
  if (m > l1) {
    if ((rc = set(0, a, l1, l1, m - l1))) return rc;
    if ((rc = set(1, ap, l1, m + l1, m - l1))) return rc;
  }
  if ((rc = set(2, b2, 0, 0, m))) return rc;
  if ((rc = set(3, bp, 0, 2 * m, m))) return rc;
  if ((rc = set(4, c, 0, 3 * m, m))) return rc;
  if ((rc = set(5, cp, 0, 4 * m, m))) return rc;
  if ((rc = set(6, kp, 0, 5 * m, m))) return rc;
  if ((rc = set(7, g1t, 0, 6 * m, n_g1t))) return rc;
  CU(pk->s3.alloc((n_g1t + 4) * sizeof(Fr)));
  uint64_t h = g_next_pk++;
  g_pks[h] = std::move(pk);
  *out = h;
  return B200_OK;
}

// len(px) against the key, as snark.GenerateProofs would index G1T (snark.go:284-286)
int pinocchio_check_px(const ProvingKey* pk, size_t npx, const char* what) {
  if (npx < pk->Z.nb) return fail(B200_EINVAL, "%s: len(px) < len(Z)", what);
  size_t nq = npx - pk->Z.nb + 1;
  if (nq > pk->n_h_bases) return fail(B200_EINVAL, "%s: len(hx)=%zu exceeds len(G1T)=%zu", what, nq, pk->n_h_bases);
  return B200_OK;
}
// A proof on this key ends in the all-gather of the ranks' records (sharded, with a matching communicator).
bool pinocchio_gathers(const ProvingKey* pk) {
  return pk->world > 1 && comm_active() && g_comm.world == pk->world && g_comm.rank == pk->rank;
}

// Enqueue one Pinocchio proof on `st` from the DEVICE-resident witness d_w (m standard-form scalars).  The quotient, read
// only by the rank that holds G1T: d_h_std (npx - len(Z) + 1 coefficients, standard form, ready on the key's side stream
// 3) when given, else px / Z from d_px (npx coefficients, Montgomery form when px_mont) on that stream.  d_out receives
// the proof (7 G1 Jacobian points and PiB, 108 u64, standard form) or, with `record`, this rank's 2 KB record of XYZZ
// results.  After pinocchio_check_px.  No host synchronisation.  A scalar >= r is read as 0 and sets bit 1 of *err.
int pinocchio_enqueue(ProvingKey* pk, const Fr* d_w, const Fr* d_px, size_t npx, int px_mont, const Fr* d_h_std, Fq* d_out,
                      bool record, cudaStream_t st, int* err) {
  const size_t m = pk->m, l1 = pk->npublic + 1, nq = npx - pk->Z.nb + 1;
  const cudaStream_t* side = pk->pctx().side;
  cudaEvent_t e_in = pk->ev[0], e_sorted[2] = {pk->ev[1], pk->ev[2]}, e_done[3] = {pk->ev[3], pk->ev[4], pk->ev[5]};
  uint8_t* res = pk->res.as<uint8_t>();
  CU(cudaMemsetAsync(res, 0, kPinRecordBytes, st));        // slots this rank does not own stay at infinity
  EV_REC(e_in, st);
  int rc;
  int next_side = 0;
  auto slot_g1 = [&](int k) { return reinterpret_cast<XYZZ<Fq>*>(res + 256 * kPinSlot[k]); };
  // side stream: hx = px / Z (snark.go:280) and PiH (snark.go:284-286)
  bool used[3] = {false, false, false};
  if (pk->g[7]) {
    cudaStream_t s3 = side[2];
    used[2] = true;
    EV_WAIT(s3, e_in);
    const Fr* dh = d_h_std;
    if (!dh) {
      CU(poly_div_device(*pk->pctx().poly, pk->Z, d_px, npx, px_mont, pk->s3.as<Fr>(), nullptr, err, s3));
      dh = pk->s3.as<Fr>();
    }
    if ((rc = msm_enqueue<Fq>(pk->g[7].get(), dh, nq, 0, slot_g1(7), err, s3))) return rc;
  }
  // two scalar vectors: w[l+1..m) feeds PiA, PiAp (snark.go:265-268); w feeds PiB, PiBp, PiC, PiCp, PiKp (:270-278).
  // Per vector ONE digit sort (held by the first owned set of the group), the bucket phases fan out over the streams.
  const int groups[2][5] = {{0, 1, -1, -1, -1}, {2, 3, 4, 5, 6}};
  int holder[2] = {-1, -1};
  for (int gi = 0; gi < 2; gi++) {   // both sorts first (main stream), then the bucket phases fan out
    for (int q = 0; q < 5; q++)
      if (groups[gi][q] >= 0 && pk->g[groups[gi][q]]) { holder[gi] = groups[gi][q]; break; }
    if (holder[gi] < 0) continue;
    const Fr* sc = gi == 0 ? d_w + l1 : d_w;
    const size_t cnt = gi == 0 ? m - l1 : m;
    if ((rc = msm_sort(pk->g[holder[gi]]->sort, pk->g[holder[gi]]->sh, sc, cnt, 0, err, st))) return rc;
    EV_REC(e_sorted[gi], st);
  }
  for (int gi = 1; gi >= 0; gi--) {   // the larger group first
    if (holder[gi] < 0) continue;
    const size_t cnt = gi == 0 ? m - l1 : m;
    SortScratch& ss = pk->g[holder[gi]]->sort;
    for (int q = 0; q < 5; q++) {
      int k = groups[gi][q];
      if (k < 0 || !pk->g[k]) continue;
      cudaStream_t sk = st;
      if (!(gi == 1 && k == holder[1])) {   // one bucket phase stays on the main stream, the others rotate over the side streams
        int si = next_side++ % 3;
        sk = side[si];
        used[si] = true;
        EV_WAIT(sk, e_sorted[gi]);
      }
      if (k == 2) rc = msm_buckets<Fq2>(pk->g[2].get(), ss, cnt, reinterpret_cast<XYZZ<Fq2>*>(res + 256 * 7), sk);
      else rc = msm_buckets<Fq>(pk->g[k].get(), ss, cnt, slot_g1(k), sk);
      if (rc) return rc;
    }
  }
  for (int si = 0; si < 3; si++)
    if (used[si]) {
      EV_REC(e_done[si], side[si]);
      EV_WAIT(st, e_done[si]);
    }
  if (record) {
    CU(cudaMemcpyAsync(d_out, res, kPinRecordBytes, cudaMemcpyDeviceToDevice, st));
  } else if (pk->world > 1) {
    CU(pk->gather.ensure(kPinRecordBytes * (size_t)pk->world));
    ncclResult_t nrc = g_comm.api.AllGather(res, pk->gather.p, kPinRecordBytes, ncclUint8, pk->pctx().comm, st);
    if (nrc != ncclSuccess) return fail(B200_ECOMM, "ncclAllGather: %s", g_comm.api.GetErrorString(nrc));
    k_pinocchio_gather_finalize_batch<<<pinocchio_finalize_blocks(1), kPinFinalizeBlock, 0, st>>>(pk->gather.as<uint8_t>(), pk->world, 1, d_out);
  } else {
    k_pinocchio_finalize<<<1, 64, 0, st>>>(res, d_out, reinterpret_cast<Fq2*>(d_out + 21));
  }
  CU(cudaGetLastError());
  return B200_OK;
}

// On the key's prove context; waits with the library mutex held.  d_rec_out != nullptr: leave this rank's 2 KB record of
// XYZZ results there (device) — the form the one-GPU tests use to emulate N ranks.
int pinocchio_prove(b200_pk_t h, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx, uint64_t* out_g1,
                    uint64_t* pi_b, uint8_t* d_rec_out = nullptr) {
  ProvingKey* pk = find_pk(h, 2);
  if (!pk) return fail(B200_EINVAL, "pinocchio_prove: bad proving-key handle");
  if (!w || !px || (!d_rec_out && (!out_g1 || !pi_b))) return fail(B200_EINVAL, "pinocchio_prove: null pointer");
  size_t m = pk->m;
  if (nw != m) return fail(B200_EINVAL, "pinocchio_prove: witness length %zu != NVars %zu", nw, m);
  int rc = pinocchio_check_px(pk, npx, "pinocchio_prove");
  if (rc) return rc;
  if (pk->world > 1 && !d_rec_out && !pinocchio_gathers(pk))
    return fail(B200_EINVAL, "pinocchio_prove: sharded key (rank %d/%d) without a matching communicator (b200_comm_init)",
                pk->rank, pk->world);
  cudaStream_t st = pk->pctx().main;
  int* err = pk->d_err_sync.as<int>();
  Fr* dw = pk->s1.as<Fr>();
  CU(cudaMemcpyAsync(dw, w, m * sizeof(Fr), cudaMemcpyHostToDevice, st));
  if (pk->g[7]) {
    CU(pk->px.ensure(npx * sizeof(Fr)));
    const size_t px_off = pk->Z.nb - 1;   // the top nq coefficients are all the division reads (see groth16_prove)
    CU(cudaMemcpyAsync(pk->px.as<Fr>() + px_off, reinterpret_cast<const Fr*>(px) + px_off, (npx - px_off) * sizeof(Fr),
                       cudaMemcpyHostToDevice, st));
  }
  if (d_rec_out) {
    if ((rc = pinocchio_enqueue(pk, dw, pk->px.as<Fr>(), npx, 0, nullptr, reinterpret_cast<Fq*>(d_rec_out), true, st, err))) return rc;
    return check_err_flag("pinocchio_prove_record", err, st);
  }
  Fq* o = pk->out_std.as<Fq>();
  if ((rc = pinocchio_enqueue(pk, dw, pk->px.as<Fr>(), npx, 0, nullptr, o, false, st, err))) return rc;
  return finish_host_proof(pk, o, "pinocchio_prove", st, nullptr, {{out_g1, 84}, {pi_b, 24}});
}

// Grows a Pinocchio key's batch scratch to k proofs (host: also the host entry's witness staging, proof buffer and pinned
// landing area), as groth16_batch_scratch does for a Groth16 key.
int pinocchio_batch_scratch(ProvingKey* pk, size_t k, bool host) {
  if (!pk->batch) {
    auto b = std::make_unique<ProveBatch>();
    for (auto& e : b->ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming));
    pk->batch = std::move(b);
  }
  ProveBatch& b = *pk->batch;
  const bool grow_host = host && b.out.bytes < k * kHostProofWords * sizeof(uint64_t);
  if (b.k < k || grow_host) CU(cudaEventSynchronize(b.done));
  if (b.k < k) {
    CU(b.CH.alloc(k * pk->n_h_bases * sizeof(Fr)));
    CU(b.rec.alloc(k * (7 * sizeof(XYZZ<Fq>) + sizeof(XYZZ<Fq2>))));
    if (pk->world > 1) CU(b.parts.alloc(k * kPinRecordBytes));
    b.k = k;
  }
  if (grow_host) {
    CU(b.w_stage.alloc(k * pk->m * sizeof(Fr)));
    CU(b.out.alloc(k * kHostProofWords * sizeof(uint64_t)));
    if (b.h_out) CU(cudaFreeHost(b.h_out));
    b.h_out = nullptr;
    CU(cudaHostAlloc(reinterpret_cast<void**>(&b.h_out), (k * kHostProofWords + 1) * sizeof(uint64_t), cudaHostAllocDefault));
  }
  return B200_OK;
}

// one-GPU emulation of the collective: sum `world` gathered records (device) -> the proof (host)
int pinocchio_finalize_records(const uint8_t* d_recs, int world, uint64_t* out_g1, uint64_t* pi_b) {
  if (!d_recs || world < 1 || !out_g1 || !pi_b) return fail(B200_EINVAL, "pinocchio_finalize: bad arguments");
  DevBuf o;
  CU(o.alloc(64 * sizeof(Fq)));
  k_pinocchio_gather_finalize_batch<<<pinocchio_finalize_blocks(1), kPinFinalizeBlock, 0, g_ctx[0].main>>>(d_recs, world, 1, o.as<Fq>());
  CU(cudaGetLastError());
  uint64_t host_out[(21 + 6) * 4];
  CU(cudaMemcpyAsync(host_out, o.p, sizeof host_out, cudaMemcpyDeviceToHost, g_ctx[0].main));
  int rc = check_err_flag("pinocchio_finalize", g_d_err);
  if (rc) return rc;
  memcpy(out_g1, host_out, 84 * 8);
  memcpy(pi_b, host_out + 84, 24 * 8);
  return B200_OK;
}
