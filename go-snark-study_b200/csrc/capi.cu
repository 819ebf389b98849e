// libb200snark: C-ABI entry points (include/b200snark.h) and the host-side
// orchestration of the CUDA kernels.  Device-only: there is no CPU fallback —
// every entry point fails with B200_ENODEVICE when no CUDA device is usable.
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include <algorithm>

#include "b200snark.h"
#include "msm.cuh"
#include "bucket_affine.cuh"
#include "poly_host.cuh"
#include "msm_host.cuh"
#include "qap.cuh"
#include "qap_sparse.cuh"
#include "fixed_base.cuh"
#include "comm.cuh"
#include "shard_partition.h"
#include "glv.cuh"
#include "pinocchio_batch.cuh"
#include "shard_batch.cuh"
#ifndef B200_NO_PAIRING
#include "pairing.cuh"
#include "pairing_warp.cuh"
#include "verify_batch.cuh"
#include "verify_batch_pinocchio.cuh"
#endif

using namespace b200;

namespace {

std::mutex g_mu;
std::string g_err;
bool g_init = false;
int g_device = -1;
// Prove context (B200_CFG_PK_CONTEXT): what a proof on a key loaded under it runs on.  A proof on a context-1 key can be in
// flight beside a proof on a context-0 key (two proofs pipelined on two caller streams: the latency-bound sort / tail /
// product chains of one overlap the accumulation of the other).  Every other library call runs on context 0's main stream
// and polynomial workspace.
// A context's shared scratch is its PolyCtx (buffers and transform plans) and its R1csWork on every R1CS.  Proofs on the
// context's keys use it on their side stream 3 while the caller's stream runs on; library calls use context 0's on its
// main stream.  Every enqueue that touches it first makes its stream wait on `scratch_free` and records `scratch_free`
// behind its last use (scratch_acquire / scratch_release), under the library mutex: the uses run in the host's order.
struct ProveCtx {
  cudaStream_t main = nullptr;   // host-pointer proofs on this context's keys
  cudaStream_t side[3] = {nullptr, nullptr, nullptr};   // side streams: independent MSMs of one proof overlap
  cudaEvent_t scratch_free = nullptr;   // behind the last enqueued use of the shared scratch
  std::unique_ptr<PolyCtx> poly;
  // NCCL communicator of the all-gathers (b200_comm_init).  Context 1 gathers on its own (ncclCommSplit of context 0's):
  // NCCL matches collectives by issue order per communicator, and two host threads proving on the two contexts reach
  // their all-gathers in an order that differs from rank to rank.  Without ncclCommSplit it is context 0's.
  ncclComm_t comm = nullptr;
};
ProveCtx g_ctx[2];
int g_pk_ctx = 0;
int g_pairing_kernel = 0;   // B200_CFG_PAIRING_KERNEL: 0 auto, 1 one thread per pairing, 2 one warp per pairing
// device error flags of the calls that hold the library mutex until they have waited (bit0: coordinate >= q, bit1: scalar
// >= r, bit2: zero leading coeff)
int* g_d_err = nullptr;

Comm g_comm;  // NCCL library, rank and world of this process (b200_comm_init); world 1 = none
bool comm_active() { return g_ctx[0].comm != nullptr; }

// Waits for the device, then destroys the communicators of both prove contexts (a shared one once).
void comm_destroy_locked() {
  if (!comm_active()) return;
  cudaSetDevice(g_device);
  cudaDeviceSynchronize();
  if (g_ctx[1].comm != g_ctx[0].comm) g_comm.api.CommDestroy(g_ctx[1].comm);
  g_comm.api.CommDestroy(g_ctx[0].comm);
  for (auto& c : g_ctx) c.comm = nullptr;
  g_comm.world = 1;
  g_comm.rank = 0;
}

// b200_config: bucket-accumulation kernel of base sets / proving keys created afterwards
// (0 auto: batched affine where the bucket population and the shard size amortise its rounds, else XYZZ; 1, 2 force)
int g_acc_mode = 0;
// partition tuning (b200_config keys 10..13; defaults = the measured best for one proof at a time)
int g_w_ab = 100, g_w_g2 = 280, g_aff_min_g1 = 700000, g_aff_min_g2 = 400000;
int g_tma_staging = 0;   // B200_CFG_TMA_STAGING: 1 staged backward pass in every round, 2 only in the contiguous rounds (>= 2)
int g_table_windows = 0;   // B200_CFG_TABLE_WINDOWS: stored window rows t of base sets created afterwards (0: all)

// ---- instrumentation (bench.py): kernel-launch counter and optional CUDA-event
// timing of the dominant kernel (k_accumulate), per group.
unsigned long long g_launches = 0;
bool g_prof = false;
bool g_serial = false;  // measurement mode: issue every MSM of a proof on the caller's stream (exclusive kernel timings)
struct ProfRec { cudaEvent_t e0, e1; int group; size_t terms; };
std::vector<ProfRec> g_prof_recs;
std::vector<cudaEvent_t> g_event_pool;
cudaEvent_t prof_event() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

// A failed allocation is not sticky, but the runtime keeps it as its last error: it is cleared here, so that the next
// call's cudaGetLastError() after a launch does not report it (a batch that did not fit would fail every later key load).
#define CU(call)                                                                             \
  do {                                                                                       \
    cudaError_t e_ = (call);                                                                 \
    if (e_ != cudaSuccess) {                                                                 \
      if (e_ == cudaErrorMemoryAllocation) cudaGetLastError();                               \
      return fail(e_ == cudaErrorMemoryAllocation ? B200_ENOMEM : B200_ECUDA, "%s:%d %s: %s", \
                  __FILE__, __LINE__, #call, cudaGetErrorString(e_));                        \
    }                                                                                        \
  } while (0)

#define NEED_INIT()                                                                      \
  do {                                                                                   \
    if (!g_init) {                                                                       \
      int rc_ = init_locked(-1);                                                         \
      if (rc_) return rc_;                                                               \
    } else {                                                                             \
      cudaSetDevice(g_device);                                                           \
    }                                                                                    \
  } while (0)

int init_locked(int device) {
  if (g_init) {
    if (device >= 0 && device != g_device) return fail(B200_EINVAL, "already initialised on device %d", g_device);
    return B200_OK;
  }
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(B200_ENODEVICE, "no CUDA device (%s); libb200snark has no CPU fallback",
                e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
  if (device < 0) {
    if (cudaGetDevice(&device) != cudaSuccess) device = 0;
  }
  if (device >= count) return fail(B200_EINVAL, "device %d out of range (%d devices)", device, count);
  CU(cudaSetDevice(device));
  for (auto& c : g_ctx) {
    CU(cudaStreamCreateWithFlags(&c.main, cudaStreamNonBlocking));
    for (auto& sd : c.side) CU(cudaStreamCreateWithFlags(&sd, cudaStreamNonBlocking));  // (stream priorities: no measurable effect)
    CU(cudaEventCreateWithFlags(&c.scratch_free, cudaEventDisableTiming));
    c.poly = std::make_unique<PolyCtx>();
    c.poly->launch_counter = &g_launches;
  }
  CU(cudaMalloc(&g_d_err, sizeof(int)));
  CU(cudaMemset(g_d_err, 0, sizeof(int)));
  g_device = device;
  g_init = true;
  return B200_OK;
}

// Order `st` behind the last enqueued use of context c's shared scratch / mark the end of this stream's use (ProveCtx).
int scratch_acquire(ProveCtx& c, cudaStream_t st) {
  CU(cudaStreamWaitEvent(st, c.scratch_free, 0));
  return B200_OK;
}
int scratch_release(ProveCtx& c, cudaStream_t st) {
  CU(cudaEventRecord(c.scratch_free, st));
  return B200_OK;
}

// ---- the MSM engine (msm_host.cuh) under the library's settings.  msm_env() is filled from the globals at every call,
// so that b200_config (B200_CFG_TMA_STAGING) and b200_profile take effect on the next MSM.  The wrappers below keep the
// argument checks and their messages, and map the engine's cudaError_t to B200 codes.
ProfRec g_prof_open{};   // the accumulation being timed (one at a time: the library mutex is held)
void prof_begin(int group, size_t terms, cudaStream_t st) {
  g_prof_open = ProfRec{prof_event(), prof_event(), group, terms};
  cudaEventRecord(g_prof_open.e0, st);
}
void prof_end(cudaStream_t st) {
  cudaEventRecord(g_prof_open.e1, st);
  g_prof_recs.push_back(g_prof_open);
}
MsmEnv msm_env() {
  MsmEnv env;
  env.launch_counter = &g_launches;
  env.tma_staging = g_tma_staging;
  if (g_prof) {
    env.prof_begin = prof_begin;
    env.prof_end = prof_end;
  }
  return env;
}

int msm_sort(SortScratch& ss, const MsmShape& shape, const Fr* d_scalars, size_t n, int mont, int* err, cudaStream_t st,
             unsigned long long* scan_totals = nullptr) {
  if (n > ss.sh.n || shape.c != ss.sh.c || shape.table_stride != ss.sh.table_stride || shape.rows != ss.sh.rows ||
      shape.vecs > ss.sh.vecs)
    return fail(B200_EINVAL, "msm_sort: shape mismatch");
  CU(b200::msm_sort(msm_env(), ss, shape, d_scalars, n, mont, err, st, scan_totals));
  return B200_OK;
}

template <class F>
int bucket_phase(Bases* b, const SortScratch& ss, BucketScratch& bk, uint32_t vecs, size_t n_terms, XYZZ<F>* d_out,
                 cudaStream_t st) {
  if (b->affine_S && ss.slice_S != b->affine_S) return fail(B200_EINVAL, "msm_buckets: slice size mismatch");
  CU(b200::bucket_phase<F>(msm_env(), b, ss, bk, vecs, n_terms, d_out, st));
  return B200_OK;
}

// One MSM's back end in the set's own bucket scratch, over `ss` (the set's own sort or that of a set sharing it).
template <class F>
int msm_buckets(Bases* b, const SortScratch& ss, size_t n_terms, XYZZ<F>* d_out, cudaStream_t st) {
  const MsmShape& sh = b->sh;
  if (ss.sh.c != sh.c || ss.sh.table_stride != sh.table_stride || ss.sh.rows != sh.rows || ss.max_slices != b->sort.max_slices ||
      ss.slice_S != b->sort.slice_S)
    return fail(B200_EINVAL, "msm_buckets: sort scratch does not match the base set");
  return bucket_phase<F>(b, ss, b->bk, 1, n_terms, d_out, st);
}

template <class F>
int msm_enqueue(Bases* b, const Fr* d_scalars, size_t n, int mont, XYZZ<F>* d_out, int* err, cudaStream_t st) {
  if (n > b->n) return fail(B200_EINVAL, "msm: n=%zu exceeds base set size %zu", n, b->n);
  CU(b200::msm_enqueue<F>(msm_env(), b, d_scalars, n, mont, d_out, err, st));
  return B200_OK;
}

std::map<uint64_t, std::unique_ptr<Bases>> g_bases;
uint64_t g_next_handle = 1;

// Reads the device error word `d_err` behind everything queued on `st` and waits for the stream.  With `lk` (the library
// mutex, held by the caller) the wait itself runs UNLOCKED, so a second host thread can enqueue a proof on the other prove
// context meanwhile (two host-pointer proofs in flight, B200_CFG_PK_CONTEXT).  A set word is cleared on `st`, behind the
// read, so the next call that uses the word on that stream starts from zero.
int check_err_flag(const char* what, int* d_err, cudaStream_t st = nullptr, std::unique_lock<std::mutex>* lk = nullptr,
                   int* pinned = nullptr) {
  if (!st) st = g_ctx[0].main;
  int h_local = 0;
  int* hp = pinned ? pinned : &h_local;   // `pinned`: a page-locked word, so the copy does not block the host under the mutex
  *hp = 0;
  CU(cudaMemcpyAsync(hp, d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (lk) lk->unlock();
  cudaError_t se = cudaStreamSynchronize(st);
  if (lk) lk->lock();
  CU(se);
  const int h = *hp;
  if (h) {
    CU(cudaMemsetAsync(d_err, 0, sizeof(int), st));
    if (h & 16) return fail(B200_EINVAL, "%s: tau is one of the interpolation points 1..n", what);
    if (h & 8) return fail(B200_EINVAL, "%s: q1[2] != Fq2.One() (G2 point at infinity; the reference panics, bn128.go:238-241)", what);
    // before the zero divisor: a leading coefficient >= r is read as 0 and also sets bit 2; the input is what is wrong
    if (h & 3) return fail(B200_ERANGE, "%s: %s", what, (h & 1) ? "point coordinate >= q" : "scalar / coefficient >= r");
    return fail(B200_EDIVZERO, "%s: divisor has a zero leading coefficient", what);
  }
  return B200_OK;
}

// The points: n standard-form Jacobian points `pts` on the host, or, with `gen`, d_scalars[i] * G minted on the device
// straight into the table's row 0 (n standard-form scalars < r, device memory): the same table words either way.
// prefer_affine: see affine_slice_size (msm_host.cuh).
template <class F>
int bases_create(const uint64_t* pts, size_t n, int c, int group, std::unique_ptr<Bases>& out_b, bool prefer_affine = true,
                 const FixedBaseTable<F>* gen = nullptr, const Fr* d_scalars = nullptr) {
  if ((!pts && !gen) || n == 0 || n > (1u << 26)) return fail(B200_EINVAL, "bases_load: bad arguments");
  if (c == 0) c = pick_window_bits(n);
  if (c < 2 || c > 24) return fail(B200_EINVAL, "window_bits must be in [2,24]");
  auto b = std::make_unique<Bases>();
  b->group = group;
  b->n = n;
  b->sh = msm_shape(n, c, g_table_windows);
  const MsmShape& sh = b->sh;
  if ((uint64_t)sh.nwin * n >= (1ull << 31)) return fail(B200_EINVAL, "nwin*n exceeds 2^31 entries");
  CU(b->table.alloc((size_t)sh.rows * n * sizeof(Affine<F>)));
  CU(b->scalars.alloc(n * sizeof(Fr)));
  b->affine_S = affine_slice_size(sh, g_acc_mode, prefer_affine);
  CU(bases_scratch<F>(*b));
  CU(b->result.alloc(sizeof(XYZZ<F>)));
  CU(b->out_std.alloc(3 * sizeof(F)));
  CU(b->d_err.alloc(sizeof(int)));
  CU(cudaMemset(b->d_err.p, 0, sizeof(int)));

  // upload + normalise (or mint row 0) + window precompute
  DevBuf staging, state;
  CU(state.alloc(n * sizeof(XYZZ<F>)));
  if (gen) {
    fixed_base_row_enqueue<F>(*gen, d_scalars, n, b->table.as<Affine<F>>(), state.as<XYZZ<F>>(), g_ctx[0].main);
  } else {
    CU(staging.alloc(n * 3 * sizeof(F)));
    CU(cudaMemcpyAsync(staging.p, pts, n * 3 * sizeof(F), cudaMemcpyHostToDevice, g_ctx[0].main));
  }
  window_table_enqueue<F>(staging.as<F>(), n, sh.rows, c, b->table.as<Affine<F>>(), state.as<XYZZ<F>>(), g_d_err, g_ctx[0].main);
  CU(cudaGetLastError());
  int rc = check_err_flag("bases_load", g_d_err);
  if (rc) return rc;
  out_b = std::move(b);
  return B200_OK;
}

template <class F>
int bases_load(const uint64_t* pts, size_t n, int c, int group, b200_bases_t* out) {
  if (!out) return fail(B200_EINVAL, "bases_load: null handle pointer");
  std::unique_ptr<Bases> b;
  int rc = bases_create<F>(pts, n, c, group, b);
  if (rc) return rc;
  uint64_t h = g_next_handle++;
  g_bases[h] = std::move(b);
  *out = h;
  return B200_OK;
}

Bases* find_bases(b200_bases_t h, int group) {
  auto it = g_bases.find(h);
  if (it == g_bases.end()) return nullptr;
  if (group && it->second->group != group) return nullptr;
  return it->second.get();
}

template <class F>
int msm_host(b200_bases_t h, int group, const uint64_t* scalars, size_t n, uint64_t* out) {
  Bases* b = find_bases(h, group);
  if (!b) return fail(B200_EINVAL, "msm: bad handle");
  if ((!scalars && n) || !out) return fail(B200_EINVAL, "msm: null pointer");
  if (n) CU(cudaMemcpyAsync(b->scalars.p, scalars, n * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  int rc = msm_enqueue<F>(b, b->scalars.as<Fr>(), n, 0, b->result.as<XYZZ<F>>(), g_d_err, g_ctx[0].main);
  if (rc) return rc;
  k_finalize<F><<<1, 32, 0, g_ctx[0].main>>>(b->result.as<XYZZ<F>>(), b->out_std.as<F>());
  CU(cudaMemcpyAsync(out, b->out_std.p, 3 * sizeof(F), cudaMemcpyDeviceToHost, g_ctx[0].main));
  rc = check_err_flag("msm", g_d_err);  // synchronises the stream
  return rc;
}

template <class F>
int sum_partials(const void* d_xyzz, size_t count, uint64_t* out, cudaStream_t st) {
  if (!d_xyzz || !out || count == 0 || count > (1u << 20)) return fail(B200_EINVAL, "sum_partials: bad arguments");
  DevBuf res, std_out;
  CU(res.alloc(sizeof(XYZZ<F>)));
  CU(std_out.alloc(3 * sizeof(F)));
  k_sum_points<F><<<1, 256, 0, st>>>(reinterpret_cast<const XYZZ<F>*>(d_xyzz), (uint32_t)count, (uint32_t)count, res.as<XYZZ<F>>());
  k_finalize<F><<<1, 32, 0, st>>>(res.as<XYZZ<F>>(), std_out.as<F>());
  CU(cudaMemcpyAsync(out, std_out.p, 3 * sizeof(F), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return B200_OK;
}

template <class F>
int mul_batch(const uint64_t* pts, int bcast, const uint64_t* scalars, size_t n, uint64_t* out) {
  if (!pts || !scalars || !out) return fail(B200_EINVAL, "mul_batch: null pointer");
  if (n == 0) return B200_OK;
  DevBuf dp, ds, dout;
  size_t np = bcast ? 1 : n;
  CU(dp.alloc(np * 3 * sizeof(F)));
  CU(ds.alloc(n * sizeof(Fr)));
  CU(dout.alloc(n * 3 * sizeof(F)));
  CU(cudaMemcpyAsync(dp.p, pts, np * 3 * sizeof(F), cudaMemcpyHostToDevice, g_ctx[0].main));
  CU(cudaMemcpyAsync(ds.p, scalars, n * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  k_mul_batch_ref<F><<<nblk(n, 128), 128, 0, g_ctx[0].main>>>(dp.as<F>(), bcast, ds.as<Fr>(), n, dout.as<F>(), g_d_err);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, dout.p, n * 3 * sizeof(F), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("mul_batch", g_d_err);
}

int poly_mul_host(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out) {
  if (!a || !b || !out || na == 0 || nb == 0) return fail(B200_EINVAL, "poly_mul: bad arguments");
  if (na + nb - 1 > ((size_t)1 << 27)) return fail(B200_EINVAL, "poly_mul: product too long");
  DevBuf da, db, dout;
  CU(da.alloc(na * sizeof(Fr)));
  CU(db.alloc(nb * sizeof(Fr)));
  CU(dout.alloc((na + nb - 1) * sizeof(Fr)));
  CU(cudaMemcpyAsync(da.p, a, na * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  CU(cudaMemcpyAsync(db.p, b, nb * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  if (int rc = scratch_acquire(g_ctx[0], g_ctx[0].main)) return rc;
  CU(poly_mul_device(*g_ctx[0].poly, da.as<Fr>(), na, 0, db.as<Fr>(), nb, 0, dout.as<Fr>(), g_d_err, g_ctx[0].main));
  if (int rc = scratch_release(g_ctx[0], g_ctx[0].main)) return rc;
  CU(cudaMemcpyAsync(out, dout.p, (na + nb - 1) * sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("poly_mul", g_d_err);
}

// The divisor b (nb standard-form coefficients) from device memory (d_b) or, with d_b null, from the host (b).
int divisor_init(Divisor& dv, const uint64_t* b, size_t nb, const Fr* d_b = nullptr) {
  DevBuf tmp;
  if (!d_b) {
    CU(tmp.alloc(nb * sizeof(Fr)));
    CU(cudaMemcpyAsync(tmp.p, b, nb * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
    d_b = tmp.as<Fr>();
  }
  CU(dv.b_mont.alloc(nb * sizeof(Fr)));
  k_poly_load<<<nblk(nb, 256), 256, 0, g_ctx[0].main>>>(d_b, (uint32_t)nb, (uint32_t)nb, 0, 0, dv.b_mont.as<Fr>(),
                                                    (uint32_t)nb, g_d_err);
  CU(cudaStreamSynchronize(g_ctx[0].main));
  dv.nb = nb;
  return B200_OK;
}

int poly_div_host(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* q, uint64_t* rem) {
  if (!a || !b || na == 0 || nb == 0) return fail(B200_EINVAL, "poly_div: bad arguments");
  if (na < nb) {  // reference: empty quotient, rem = a (r1csqap.go:70-84 loop never runs)
    if (rem) memcpy(rem, a, na * sizeof(Fr));
    return B200_OK;
  }
  if (!q) return fail(B200_EINVAL, "poly_div: null quotient buffer");
  Divisor dv;
  int rc = divisor_init(dv, b, nb);
  if (rc) return rc;
  size_t nq = na - nb + 1;
  DevBuf da, dq, dr;
  CU(da.alloc(na * sizeof(Fr)));
  CU(dq.alloc(nq * sizeof(Fr)));
  if (rem && nb > 1) CU(dr.alloc((nb - 1) * sizeof(Fr)));
  CU(cudaMemcpyAsync(da.p, a, na * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  if ((rc = scratch_acquire(g_ctx[0], g_ctx[0].main))) return rc;
  CU(poly_div_device(*g_ctx[0].poly, dv, da.as<Fr>(), na, 0, dq.as<Fr>(), dr.as<Fr>(), g_d_err, g_ctx[0].main));
  if ((rc = scratch_release(g_ctx[0], g_ctx[0].main))) return rc;
  CU(cudaMemcpyAsync(q, dq.p, nq * sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  if (rem && nb > 1) CU(cudaMemcpyAsync(rem, dr.p, (nb - 1) * sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("poly_div", g_d_err);
}

#include "prove_host.cuh"

#include "qap_sparse_host.cuh"

// groth16.GenerateProofs fed from the DEVICE-resident witness d_w (m standard-form scalars): px = CombinePolynomials(w,
// R1CSToQAP(a, b, c)) — or the quotient h directly — is computed on the device from the resident sparse R1CS (never
// leaving HBM) and handed to the prove pipeline, all on `st` and the key's side streams with the key's R1CS workspace,
// so proofs on keys of the two prove contexts may be in flight together.  No host synchronisation after the first call
// on an (R1CS, context) pair.  A sharded rank that holds no PowersTauDelta index needs no quotient and runs no QAP kernel.
int groth16_witness_enqueue(ProvingKey* pk, R1cs* r1, const Fr* d_w, const uint64_t* r, const uint64_t* s, Fq* d_out,
                            cudaStream_t st, int* err) {
  if (fr_load_std(r).geq_modulus() || fr_load_std(s).geq_modulus())
    return fail(B200_ERANGE, "groth16_prove_witness: r or s >= field order");
  const size_t npx = 2 * r1->n - 1;
  if (!pk_needs_px(pk)) return groth16_enqueue(pk, d_w, pk->m, nullptr, npx, r, s, d_out, st, err);
  // the quotient is only consumed on side stream 3 (groth16_enqueue): compute it THERE, so the QAP front end (NTT passes,
  // HBM-bound) overlaps the A / B1 / B2 bucket phases (multiply-bound) on the other streams
  cudaStream_t sq = g_serial ? st : pk->pctx().side[2];
  if (sq != st) {
    CU(cudaEventRecord(pk->ev[0], st));
    CU(cudaStreamWaitEvent(sq, pk->ev[0], 0));
  }
  const Fr *h, *px;   // h itself, or px for groth16_enqueue's division; that releases the scratch behind its last read
  int rc = scratch_acquire(pk->pctx(), sq);
  if (rc) return rc;
  rc = qap_quotient_enqueue(r1, pk->Z.nb, pk->ctx, *pk->pctx().poly, d_w, err, sq, &h, &px);
  if (rc) return rc;
  return groth16_enqueue(pk, d_w, pk->m, px, npx, r, s, d_out, st, err, /*px_mont=*/1, h);
}

int groth16_prove_witness(b200_pk_t h, b200_r1cs_t hr, const uint64_t* w, size_t nw, const uint64_t* r, const uint64_t* s,
                          uint64_t* pi_a, uint64_t* pi_b, uint64_t* pi_c, std::unique_lock<std::mutex>* lk) {
  ProvingKey* pk = find_pk(h, 1);
  R1cs* r1 = find_r1cs(hr);
  if (!pk || !r1) return fail(B200_EINVAL, "groth16_prove_witness: bad handle");
  if (!w || !r || !s || !pi_a || !pi_b || !pi_c) return fail(B200_EINVAL, "groth16_prove_witness: null pointer");
  if (nw != pk->m || nw != r1->m) return fail(B200_EINVAL, "groth16_prove_witness: witness length %zu, NVars %zu, R1CS columns %zu", nw, pk->m, r1->m);
  int rc = check_sharded_host_call(pk, "groth16_prove_witness", "b200_groth16_prove_witness_device");
  if (rc) return rc;
  cudaStream_t st = pk->pctx().main;
  // the QAP front end reads the whole witness; a rank that runs none reads only its own index ranges
  if ((rc = stage_witness(pk, w, pk_needs_px(pk), st))) return rc;
  Fq* o = pk->out_std.as<Fq>();
  if ((rc = groth16_witness_enqueue(pk, r1, pk->w_stage.as<Fr>(), r, s, o, st, pk->d_err_sync.as<int>()))) return rc;
  return finish_host_proof(pk, pk->h_out, o, 1, "groth16_prove_witness", st, lk, {{pi_a, 12}, {pi_c, 12}, {pi_b, 24}});
}

// ---- batches: k witness-fed proofs under one key (b200_groth16_prove_witness_batch) ---------------------------------
// Proof p is the proof of groth16_witness_enqueue for (w_p, r_p, s_p).  The four MSMs run as batched MSMs over k scalar
// vectors (W_p = w_p ++ [1, r_p, s_p] for A, B1, B2 with one shared sort; C||PTD_p), the quotients as one batched front
// end (qap_quotient_batch_enqueue; len(Z) = n + 1 or n), the blinding products with one warp per proof: the launches of
// one proof, whatever k.
// On a key shard every vector is the rank's part of it (G16Slices), and the batch ends in k partial records.

// Everything that is refused before anything is allocated or enqueued.  On a key shard every refusal is decided on
// values every rank of the shard shares (the arguments, the R1CS, every rank's cut), so all ranks return the same code
// and none is left waiting in the all-gather of its peers.
int groth16_batch_check(const ProvingKey* pk, const R1cs* r1, size_t nw, size_t k, const uint64_t* r, const uint64_t* s,
                        const char* what) {
  if (k == 0) return fail(B200_EINVAL, "%s: k = 0", what);
  if (nw != pk->m || nw != r1->m) return fail(B200_EINVAL, "%s: witness length %zu, NVars %zu, R1CS columns %zu", what, nw, pk->m, r1->m);
  const size_t npx = 2 * r1->n - 1;
  if (npx < pk->Z.nb) return fail(B200_EINVAL, "%s: len(px) < len(Z)", what);
  if (npx - pk->Z.nb + 1 > pk->n_h_bases)
    return fail(B200_EINVAL, "%s: len(hx)=%zu exceeds len(PowersTauDelta)=%zu", what, npx - pk->Z.nb + 1, pk->n_h_bases);
  const size_t terms[4] = {pk->m + 3, pk->m + 3, pk->m + 3, pk->n_c_full + pk->n_h_bases + 1};
  uint32_t nwin;
  if (pk->world == 1) {
    for (int j = 0; j < 4; j++)
      if (!pk_batch_fits(pk, j, k, terms[j], &nwin))
        return fail(B200_EINVAL, "%s: k * nwin * terms = %zu * %u * %zu sort entries (or the buckets) of set %d exceed 2^31", what, k,
                    nwin, terms[j], j);
  } else {   // the largest part any rank holds: the shape each rank's set was built with, from its cut
    for (int g = 0; g < pk->world; g++) {
      const G16Slices sl = g16_slices(pk, g);
      for (int j = 0; j < 4; j++)
        if (sl.terms[j] && !pk_batch_fits(pk, j, k, sl.terms[j], &nwin))
          return fail(B200_EINVAL, "%s: k * nwin * terms = %zu * %u * %zu sort entries (or the buckets) of set %d on rank %d/%d exceed 2^31",
                      what, k, nwin, sl.terms[j], j, g, pk->world);
    }
  }
  int rc = qap_batch_check(r1, k, what);
  if (rc) return rc;
  // the scalar vectors are laid out by 2-D copies whose row pitch (one vector, one witness) the device bounds; the
  // unsharded widths bound every rank's
  int max_pitch = 0;
  CU(cudaDeviceGetAttribute(&max_pitch, cudaDevAttrMaxPitch, g_device));
  const uint64_t widest = std::max(terms[0], terms[3]) * sizeof(Fr);
  if (widest > (uint64_t)max_pitch)
    return fail(B200_EINVAL, "%s: a scalar vector of %llu bytes exceeds the device's copy pitch of %d bytes", what,
                (unsigned long long)widest, max_pitch);
  for (size_t p = 0; p < k; p++)
    if (fr_load_std(r + 4 * p).geq_modulus() || fr_load_std(s + 4 * p).geq_modulus())
      return fail(B200_ERANGE, "%s: r or s of proof %zu >= field order", what, p);
  return B200_OK;
}

// A sharded key whose batches end in the all-gather: a communicator of the key's world (its rank checked by the caller).
bool groth16_gathers(const ProvingKey* pk) { return pk->world > 1 && comm_active() && g_comm.world == pk->world; }

// The entries that return proofs: a sharded key needs its communicator (checked before anything is enqueued).
int groth16_batch_comm_check(const ProvingKey* pk, const char* what) {
  if (pk->world == 1) return B200_OK;
  if (!groth16_gathers(pk))
    return fail(B200_EINVAL, "%s: sharded key (rank %d/%d) without a matching communicator: call b200_comm_init, or use "
                             "b200_groth16_prove_witness_batch_partial_device + b200_groth16_finalize_batch_device around "
                             "your own all-gather", what, pk->rank, pk->world);
  if (g_comm.rank != pk->rank) return fail(B200_EINVAL, "%s: key shard %d on communicator rank %d", what, pk->rank, g_comm.rank);
  return B200_OK;
}

// d_w: k witnesses (device, standard form, witness p at d_w + p*m); r, s: host, k x 4 limbs.  d_recs null (one GPU only):
// k proofs at d_proofs + 48p (u64, PiA | PiC | PiB).  Else k partial records of this rank at d_recs + 1 KB * p.  After
// groth16_batch_check.  No host synchronisation unless a scratch grows (or the first batch on this R1CS and context
// builds its domains).  Records no `done` event (groth16_batch_enqueue does, behind what reads the records).
int groth16_batch_parts(ProvingKey* pk, R1cs* r1, const Fr* d_w, size_t k, const uint64_t* r, const uint64_t* s,
                        Fq* d_proofs, uint8_t* d_recs, cudaStream_t st, int* err, R1csBatch** fb_used) {
  const size_t m = pk->m, l1 = pk->npublic + 1;
  const G16Slices sl = g16_slices(pk, pk->rank);
  size_t woff[3];
  g16_w_layout(pk, sl, woff);
  const size_t nch = sl.terms[3], n_c = sl.n_c, n_p = sl.n_p;
  const bool quotient = pk->g[3] && pk_needs_px(pk);   // only a rank that holds PowersTauDelta indices runs the front end
  // host: {1, r_p, s_p, -r_p s_p} and the GLV splits of (s_p, r_p)
  std::vector<Fr> small(4 * k);
  std::vector<GlvScalars> glv(k);
  Fr one = Fr::zero();
  one.l[0] = 1;
  for (size_t p = 0; p < k; p++) {
    Fr fr_r = fr_load_std(r + 4 * p), fr_s = fr_load_std(s + 4 * p);
    small[4 * p] = one;
    small[4 * p + 1] = fr_r;
    small[4 * p + 2] = fr_s;
    small[4 * p + 3] = (fr_r.to_mont() * fr_s.to_mont()).neg().from_mont();
    if (glv_decompose(fr_s, glv[p].k[0], glv[p].neg[0]) || glv_decompose(fr_r, glv[p].k[1], glv[p].neg[1]))
      return fail(B200_EINVAL, "groth16_prove_witness_batch: GLV decomposition out of range");
  }
  // every scratch first: growing one waits for the batch that used it last, so nothing of this batch is enqueued yet
  R1csWork* ws = nullptr;
  R1csBatch* fb = nullptr;
  int rc;
  if (quotient && (rc = qap_quotient_batch_prepare(r1, pk->Z.nb, pk->ctx, k, &ws, &fb))) return rc;
  *fb_used = fb;
  if ((rc = groth16_batch_scratch(pk, k, false))) return rc;
  for (int j = 0; j < 3; j++) {
    if (!pk->g[j]) continue;
    const bool own = pk->sort_src[j] == j;
    const uint32_t n = (uint32_t)sl.terms[j];
    CU(j == 2 ? batch_scratch<Fq2>(pk->g[j].get(), (uint32_t)k, n, own) : batch_scratch<Fq>(pk->g[j].get(), (uint32_t)k, n, own));
  }
  if (pk->g[3]) CU(batch_scratch<Fq>(pk->g[3].get(), (uint32_t)k, (uint32_t)nch));
  for (int j = 0; j < 3; j++)
    if (pk->g[j] && !batch_shares_sort(pk->g[j].get(), pk->g[pk->sort_src[j]].get()))
      return fail(B200_EINVAL, "groth16_prove_witness_batch: batch scratch of set %d does not match the sort of set %d", j, pk->sort_src[j]);
  ProveBatch& b = *pk->batch;
  cudaStream_t s1 = pk->pctx().side[0], s2 = pk->pctx().side[1], s3 = pk->pctx().side[2];
  if (g_serial) s1 = s2 = s3 = st;   // measurement mode (b200_profile bit 1)
  cudaEvent_t e_in = b.ev[0], e_sorted[3] = {b.ev[1], b.ev[2], b.ev[3]}, e_a = b.ev[4], e_b1 = b.ev[5], e_b2 = b.ev[6],
              e_ch = b.ev[7], e_prod = b.ev[8];
  Fr* W = b.W.as<Fr>();
  Fr* CH = b.CH.as<Fr>();
  Fr* rs = b.rs.as<Fr>();
  XYZZ<Fq>* rA = b.rec.as<XYZZ<Fq>>();
  XYZZ<Fq>* rB1 = rA + k;
  XYZZ<Fq>* rCH = rB1 + k;
  XYZZ<Fq>* prod = rCH + k;
  XYZZ<Fq2>* rB2 = reinterpret_cast<XYZZ<Fq2>*>(prod + 2 * k);
  const size_t F = sizeof(Fr);
  CU(cudaMemcpyAsync(rs, small.data(), 4 * k * F, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(b.glv.p, glv.data(), k * sizeof(GlvScalars), cudaMemcpyHostToDevice, st));
  // a shard's sets it does not hold, and its products when it holds no part of A or B1, stay at infinity
  if (pk->world > 1) CU(cudaMemsetAsync(b.rec.p, 0, b.rec.bytes, st));
  for (int j = 0; j < 3; j++) {    // W_p = w_p[lo_j, hi_j) ++ [1, r_p, s_p] (the latter with set j's tail)
    if (!pk->g[j] || pk->sort_src[j] != j) continue;
    const size_t nt = sl.terms[j], cnt = sl.hi[j] - sl.lo[j];
    Fr* Wj = W + k * woff[j];
    if (cnt) CU(cudaMemcpy2DAsync(Wj, nt * F, d_w + sl.lo[j], m * F, cnt * F, k, cudaMemcpyDeviceToDevice, st));
    if (sl.tail[j]) CU(cudaMemcpy2DAsync(Wj + cnt, nt * F, rs, 4 * F, 3 * F, k, cudaMemcpyDeviceToDevice, st));
  }
  if (pk->g[3] && n_c) CU(cudaMemcpy2DAsync(CH, nch * F, d_w + l1 + sl.c_lo, m * F, n_c * F, k, cudaMemcpyDeviceToDevice, st));
  EV_REC(e_in, st);
  // --- side stream 3: the quotients into the C||PTD vectors (h_p[p_lo, p_lo + n_p), zeros beyond len(h), -r_p s_p with
  // the tail), then the C||PTD MSMs
  EV_WAIT(s3, e_in);
  if (quotient) {
    if ((rc = scratch_acquire(pk->pctx(), s3))) return rc;
    if ((rc = qap_quotient_batch_enqueue(r1, ws, fb, *pk->pctx().poly, pk->Z, pk->h_full.as<Fr>(), d_w, k, CH + n_c, nch, n_p,
                                         sl.p_lo, sl.tail[3] ? rs + 3 : nullptr, s3, err)))
      return rc;
    if ((rc = scratch_release(pk->pctx(), s3))) return rc;
  }
  MsmShape sh;
  if (Bases* gch = pk->g[3].get()) {
    sh = gch->sh;
    sh.vecs = (uint32_t)k;
    sh.vec_stride = (uint32_t)nch;
    if ((rc = msm_sort(gch->batch->sort, sh, CH, nch, 0, err, s3, gch->batch->scan_totals.as<unsigned long long>()))) return rc;
    if ((rc = bucket_phase<Fq>(gch, gch->batch->sort, gch->batch->bk, (uint32_t)k, nch, rCH, s3))) return rc;
  }
  EV_REC(e_ch, s3);
  // --- A, B1, B2: one batched sort per distinct slice on the main stream, the bucket phases on st / s1 / s2 (B2 first:
  // the longest)
  for (int j = 0; j < 3; j++) {
    if (!pk->g[j] || pk->sort_src[j] != j) continue;
    Bases* g = pk->g[j].get();
    sh = g->sh;
    sh.vecs = (uint32_t)k;
    sh.vec_stride = (uint32_t)sl.terms[j];
    if ((rc = msm_sort(g->batch->sort, sh, W + k * woff[j], sl.terms[j], 0, err, st, g->batch->scan_totals.as<unsigned long long>()))) return rc;
    EV_REC(e_sorted[j], st);
  }
  cudaStream_t sk[3] = {st, s1, s2};
  for (int j = 2; j >= 0; j--) {
    if (!pk->g[j]) continue;
    const int src = pk->sort_src[j];
    const SortScratch& ss = pk->g[src]->batch->sort;
    Bases* g = pk->g[j].get();
    if (sk[j] != st) EV_WAIT(sk[j], e_sorted[src]);
    if (j == 2) rc = bucket_phase<Fq2>(g, ss, g->batch->bk, (uint32_t)k, sl.terms[j], rB2, sk[2]);
    else rc = bucket_phase<Fq>(g, ss, g->batch->bk, (uint32_t)k, sl.terms[j], j ? rB1 : rA, sk[j]);
    if (rc) return rc;
  }
  EV_REC(e_a, st);
  EV_REC(e_b1, s1);
  EV_REC(e_b2, s2);
  // s_p * A_p and r_p * B1_p on side stream 1, one warp per proof, while B2 / C||PTD still run; a shard that holds no
  // part of A or B1 skips them (its products are infinity, as in groth16_enqueue)
  EV_WAIT(s1, e_a);
  if (pk->g[0] || pk->g[1]) {
    k_groth16_products_batch<<<(unsigned)k, 32, 0, s1>>>(rA, rB1, b.glv.as<GlvScalars>(), prod);
    g_launches += 1;
  }
  EV_REC(e_prod, s1);
  EV_WAIT(st, e_prod);
  EV_WAIT(st, e_b2);
  EV_WAIT(st, e_ch);
  if (!d_recs) {
    k_groth16_combine_batch<<<nblk(3 * k, 96), 96, 0, st>>>(rA, rB2, rCH, prod, (uint32_t)k, d_proofs);
  } else {   // fold the products into each proof's C part: k partial records
    CU(cudaMemsetAsync(d_recs, 0, k * kPartialBytes, st));
    k_groth16_fold_products_batch<<<nblk(k, 64), 64, 0, st>>>(rA, rB1, rB2, rCH, prod, (uint32_t)k, d_recs);
  }
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}

// Behind everything of a batch on `st`: what the next regrowth of any of its scratches waits for (the key's, every set's
// and the quotient front end's, fb, when the batch used it).
int batch_done_record(ProvingKey* pk, R1csBatch* fb, cudaStream_t st) {
  EV_REC(pk->batch->done, st);
  for (const auto& g : pk->g)
    if (g && g->batch) EV_REC(g->batch->done, st);
  if (fb) EV_REC(fb->done, st);
  return B200_OK;
}

// The k proofs of a batch at d_out + 48p (u64), or with `records` this rank's k partial records at d_out + 1 KB * p.  A
// sharded key without `records` computes its records, all-gathers them (k records per rank, on the key's prove-context
// communicator, on `st`) and finalises: every rank receives the k proofs.  After groth16_batch_check and, without
// `records`, groth16_batch_comm_check.  Once the records' scratch exists the all-gather runs whatever else fails, so no
// peer is left waiting; the error is then returned and nothing is finalised.
int groth16_batch_enqueue(ProvingKey* pk, R1cs* r1, const Fr* d_w, size_t k, const uint64_t* r, const uint64_t* s, Fq* d_out,
                          bool records, cudaStream_t st, int* err) {
  int rc;
  R1csBatch* fb = nullptr;   // the front end's scratch, if the batch used it
  if (pk->world == 1 || records) {
    rc = groth16_batch_parts(pk, r1, d_w, k, r, s, d_out, records ? reinterpret_cast<uint8_t*>(d_out) : nullptr, st, err, &fb);
  } else {
    if ((rc = groth16_batch_scratch(pk, k, false))) return rc;
    CU(pk->gather.ensure(kPartialBytes * k * (size_t)pk->world));
    ProveBatch& b = *pk->batch;
    rc = groth16_batch_parts(pk, r1, d_w, k, r, s, nullptr, b.parts.as<uint8_t>(), st, err, &fb);
    ncclResult_t nrc = g_comm.api.AllGather(b.parts.p, pk->gather.p, kPartialBytes * k, ncclUint8, pk->pctx().comm, st);
    if (rc) return rc;
    if (nrc != ncclSuccess) return fail(B200_ECOMM, "ncclAllGather: %s", g_comm.api.GetErrorString(nrc));
    k_groth16_finalize_batch<<<groth16_finalize_blocks((uint32_t)k), kG16FinalizeBlock, 0, st>>>(pk->gather.as<uint8_t>(), pk->world,
                                                                                                   (uint32_t)k, d_out);
    g_launches += 1;
    CU(cudaGetLastError());
  }
  if (rc) return rc;
  return batch_done_record(pk, fb, st);
}

int groth16_prove_witness_batch(b200_pk_t h, b200_r1cs_t hr, const uint64_t* w, size_t nw, size_t k, const uint64_t* r,
                                const uint64_t* s, uint64_t* pi_a, uint64_t* pi_b, uint64_t* pi_c, std::unique_lock<std::mutex>* lk) {
  const char* what = "groth16_prove_witness_batch";
  ProvingKey* pk = find_pk(h, 1);
  R1cs* r1 = find_r1cs(hr);
  if (!pk || !r1) return fail(B200_EINVAL, "%s: bad handle", what);
  if (!w || !r || !s || !pi_a || !pi_b || !pi_c) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = groth16_batch_check(pk, r1, nw, k, r, s, what);
  if (rc) return rc;
  if ((rc = groth16_batch_comm_check(pk, what))) return rc;
  if ((rc = groth16_batch_scratch(pk, k, true))) return rc;
  ProveBatch& b = *pk->batch;
  cudaStream_t st = pk->pctx().main;
  // a shard that runs no QAP front end reads only its witness ranges
  if (pk->world == 1) CU(cudaMemcpyAsync(b.w_stage.p, w, k * nw * sizeof(Fr), cudaMemcpyHostToDevice, st));
  else if ((rc = stage_witness(pk, w, pk_needs_px(pk), st, b.w_stage.as<Fr>(), k))) return rc;
  Fq* o = b.out.as<Fq>();
  if ((rc = groth16_batch_enqueue(pk, r1, b.w_stage.as<Fr>(), k, r, s, o, false, st, pk->d_err_sync.as<int>()))) return rc;
  return finish_host_proof(pk, b.h_out, o, k, what, st, lk, {{pi_a, 12}, {pi_c, 12}, {pi_b, 24}});
}

// ---- witness-fed Pinocchio proving (b200_pinocchio_prove_witness and its _device / _batch twins) ---------------------------
// snark.GenerateProofs fed from the DEVICE-resident witness d_w, as groth16_witness_enqueue: the quotient comes from the
// resident sparse R1CS on the key's side stream 3, where the G1T MSM consumes it, so the QAP front end overlaps the seven
// witness MSMs.  On a sharded key only the rank that holds G1T runs it; every other rank launches no QAP kernel.  d_out
// and `record` as in pinocchio_enqueue.  No host synchronisation after the first call on an (R1CS, context) pair.
int pinocchio_witness_enqueue(ProvingKey* pk, R1cs* r1, const Fr* d_w, Fq* d_out, bool record, cudaStream_t st, int* err) {
  const size_t npx = 2 * r1->n - 1;
  if (!pk->g[7]) return pinocchio_enqueue(pk, d_w, nullptr, npx, 0, nullptr, d_out, record, st, err);
  cudaStream_t sq = g_serial ? st : pk->pctx().side[2];   // measurement mode: the front end on the caller's stream
  if (sq != st) {
    CU(cudaEventRecord(pk->ev[0], st));
    CU(cudaStreamWaitEvent(sq, pk->ev[0], 0));
  }
  const Fr *h, *px;   // h itself, or px for pinocchio_enqueue's division; that releases the scratch behind its last read
  int rc = scratch_acquire(pk->pctx(), sq);
  if (rc) return rc;
  rc = qap_quotient_enqueue(r1, pk->Z.nb, pk->ctx, *pk->pctx().poly, d_w, err, sq, &h, &px);
  if (rc) return rc;
  return pinocchio_enqueue(pk, d_w, px, npx, /*px_mont=*/1, h, d_out, record, st, err);
}

// What every witness-fed Pinocchio entry refuses before anything is allocated or enqueued.
int pinocchio_witness_check(const ProvingKey* pk, const R1cs* r1, size_t nw, const char* what) {
  if (nw != pk->m || nw != r1->m) return fail(B200_EINVAL, "%s: witness length %zu, NVars %zu, R1CS columns %zu", what, nw, pk->m, r1->m);
  return pinocchio_check_px(pk, 2 * r1->n - 1, what);
}

int pinocchio_prove_witness(b200_pk_t h, b200_r1cs_t hr, const uint64_t* w, size_t nw, uint64_t* out_g1, uint64_t* pi_b,
                            std::unique_lock<std::mutex>* lk) {
  const char* what = "pinocchio_prove_witness";
  ProvingKey* pk = find_pk(h, 2);
  R1cs* r1 = find_r1cs(hr);
  if (!pk || !r1) return fail(B200_EINVAL, "%s: bad handle", what);
  if (!w || !out_g1 || !pi_b) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = pinocchio_witness_check(pk, r1, nw, what);
  if (rc) return rc;
  if (pk->world > 1 && !pinocchio_gathers(pk))
    return fail(B200_EINVAL, "%s: sharded key (rank %d/%d) without a matching communicator: call b200_comm_init, or use "
                             "b200_pinocchio_prove_witness_device + b200_pinocchio_finalize_records around your own all-gather",
                what, pk->rank, pk->world);
  cudaStream_t st = pk->pctx().main;
  Fr* dw = pk->s1.as<Fr>();
  CU(cudaMemcpyAsync(dw, w, nw * sizeof(Fr), cudaMemcpyHostToDevice, st));
  Fq* o = pk->out_std.as<Fq>();
  if ((rc = pinocchio_witness_enqueue(pk, r1, dw, o, false, st, pk->d_err_sync.as<int>()))) return rc;
  return finish_host_proof(pk, pk->h_out, o, 1, what, st, lk, {{out_g1, 84}, {pi_b, 24}});
}

// ---- batches: k witness-fed Pinocchio proofs under one key (b200_pinocchio_prove_witness_batch) -------------------------
// Proof p is the proof of pinocchio_witness_enqueue for w_p.  Pinocchio has no blinding, so the scalar vectors of the seven
// witness MSMs are the caller's witnesses where they lie (stride m): one batched sort of d_w serves B, Bp, C, Cp, Kp, one
// of d_w + l1 serves A, Ap, and one of the k quotient vectors serves G1T; eight batched bucket phases and one
// finalisation kernel follow: the launches of one proof, whatever k.

// Sets whose batches share one digit sort (the set's own index: it sorts), as the groups of pinocchio_enqueue.
constexpr int kPinSortSrc[8] = {0, 0, 2, 2, 2, 2, 2, 7};

// Everything refused before anything is allocated or enqueued.  On a key shard the sets' sizes are the same on every rank
// (whole MSMs are dealt) and every set is checked with the shape its owner built it with, so every rank of the shard
// returns the same code.
int pinocchio_batch_check(const ProvingKey* pk, const R1cs* r1, size_t nw, size_t k, const char* what) {
  if (k == 0) return fail(B200_EINVAL, "%s: k = 0", what);
  int rc = pinocchio_witness_check(pk, r1, nw, what);
  if (rc) return rc;
  const size_t ma = pk->m - pk->npublic - 1;
  const size_t terms[8] = {ma, ma, pk->m, pk->m, pk->m, pk->m, pk->m, pk->n_h_bases};
  uint32_t nwin;
  for (int j = 0; j < 8; j++)
    if ((pk->world == 1 ? pk->g[j] != nullptr : terms[j] != 0) && !pk_batch_fits(pk, j, k, terms[j], &nwin))
      return fail(B200_EINVAL, "%s: k * nwin * terms = %zu * %u * %zu sort entries (or the buckets) of set %d exceed 2^31", what, k,
                  nwin, terms[j], j);
  return qap_batch_check(r1, k, what);
}

// The entries that return proofs: a sharded key needs its communicator (checked before anything is enqueued).
int pinocchio_batch_comm_check(const ProvingKey* pk, const char* what) {
  if (pk->world == 1 || pinocchio_gathers(pk)) return B200_OK;
  return fail(B200_EINVAL, "%s: sharded key (rank %d/%d) without a matching communicator: call b200_comm_init, or use "
                           "b200_pinocchio_prove_witness_batch_record_device + b200_pinocchio_finalize_records_batch_device "
                           "around your own all-gather", what, pk->rank, pk->world);
}

// d_w: k witnesses (device, standard form, witness p at d_w + p*m).  d_recs null (one GPU only): k proofs at d_out + 108p
// (u64: the seven G1 points, then PiB).  Else this rank's k records at d_recs + 2 KB * p, the slots of sets it does not
// own at infinity.  A key shard runs only the sets it owns (pinocchio_owners): a sort group whose sorting set lives on
// another rank is sorted by its first owned member, and only the G1T owner runs the QAP front end.  After
// pinocchio_batch_check.  No host synchronisation unless a scratch grows (or the first batch on this R1CS and context
// builds its domains).  Records no `done` event (pinocchio_batch_enqueue does, behind what reads the records).
int pinocchio_batch_parts(ProvingKey* pk, R1cs* r1, const Fr* d_w, size_t k, Fq* d_out, uint8_t* d_recs, cudaStream_t st,
                          int* err, R1csBatch** fb_used) {
  const size_t m = pk->m, l1 = pk->npublic + 1, ng = pk->n_h_bases;
  const size_t terms[8] = {m - l1, m - l1, m, m, m, m, m, ng};
  // the set that sorts for set j: the first set of j's group (kPinSortSrc) this key holds
  int src[8];
  for (int j = 0; j < 8; j++) {
    src[j] = -1;
    for (int q = 0; q < 8 && src[j] < 0; q++)
      if (kPinSortSrc[q] == kPinSortSrc[j] && pk->g[q]) src[j] = q;
  }
  // every scratch first: growing one waits for the batch that used it last, so nothing of this batch is enqueued yet
  R1csWork* ws = nullptr;
  R1csBatch* fb = nullptr;
  int rc;
  if (pk->g[7] && (rc = qap_quotient_batch_prepare(r1, pk->Z.nb, pk->ctx, k, &ws, &fb))) return rc;
  *fb_used = fb;
  if ((rc = pinocchio_batch_scratch(pk, k, false))) return rc;
  for (int j = 0; j < 8; j++) {
    if (!pk->g[j]) continue;   // a set another rank owns, or A, Ap of a circuit whose signals are all public
    const bool own = src[j] == j;
    CU(j == 2 ? batch_scratch<Fq2>(pk->g[j].get(), (uint32_t)k, (uint32_t)terms[j], own)
              : batch_scratch<Fq>(pk->g[j].get(), (uint32_t)k, (uint32_t)terms[j], own));
  }
  for (int j = 0; j < 8; j++)
    if (pk->g[j] && !batch_shares_sort(pk->g[j].get(), pk->g[src[j]].get()))
      return fail(B200_EINVAL, "pinocchio_prove_witness_batch: batch scratch of set %d does not match the sort of set %d", j, src[j]);
  ProveBatch& b = *pk->batch;
  cudaStream_t side[3] = {pk->pctx().side[0], pk->pctx().side[1], pk->pctx().side[2]};
  if (g_serial) side[0] = side[1] = side[2] = st;   // measurement mode (b200_profile bit 1)
  cudaEvent_t e_in = b.ev[0], e_sorted[2] = {b.ev[1], b.ev[2]}, e_done[3] = {b.ev[3], b.ev[4], b.ev[5]};
  XYZZ<Fq>* rec1 = b.rec.as<XYZZ<Fq>>();                         // slot s of proof p at rec1[s*k + p]
  XYZZ<Fq2>* rec2 = reinterpret_cast<XYZZ<Fq2>*>(rec1 + 7 * k);
  auto sort_of = [&](int j, const Fr* sc, size_t stride, cudaStream_t s) {
    Bases* g = pk->g[j].get();
    MsmShape sh = g->sh;
    sh.vecs = (uint32_t)k;
    sh.vec_stride = (uint32_t)stride;
    return msm_sort(g->batch->sort, sh, sc, terms[j], 0, err, s, g->batch->scan_totals.as<unsigned long long>());
  };
  auto buckets_of = [&](int j, cudaStream_t s) {
    Bases* g = pk->g[j].get();
    const SortScratch& ss = pk->g[src[j]]->batch->sort;
    if (j == 2) return bucket_phase<Fq2>(g, ss, g->batch->bk, (uint32_t)k, terms[j], rec2, s);
    return bucket_phase<Fq>(g, ss, g->batch->bk, (uint32_t)k, terms[j], rec1 + kPinSlot[j] * k, s);
  };
  // sets the key does not hold (another rank's; A, Ap when every signal is public) leave their records at infinity, as in
  // pinocchio_enqueue
  CU(cudaMemsetAsync(b.rec.p, 0, k * (7 * sizeof(XYZZ<Fq>) + sizeof(XYZZ<Fq2>)), st));
  EV_REC(e_in, st);
  // --- side stream 3 (the G1T owner): the k quotients into the G1T scalar vectors (zero-filled to len(G1T)), then the
  // G1T MSMs
  cudaStream_t s3 = side[2];
  if (pk->g[7]) {
    if (s3 != st) EV_WAIT(s3, e_in);
    Fr* H = b.CH.as<Fr>();   // len(h) <= len(G1T) (pinocchio_check_px): every quotient is divided straight into its vector
    if ((rc = scratch_acquire(pk->pctx(), s3))) return rc;
    if ((rc = qap_quotient_batch_enqueue(r1, ws, fb, *pk->pctx().poly, pk->Z, nullptr, d_w, k, H, ng, ng, 0, nullptr, s3, err)))
      return rc;
    if ((rc = scratch_release(pk->pctx(), s3))) return rc;
    if ((rc = sort_of(7, H, ng, s3))) return rc;
    if ((rc = buckets_of(7, s3))) return rc;
  }
  // --- the witness MSMs: the sorts on the main stream, then the bucket phases fan out as in pinocchio_enqueue (G2 first);
  // the first set issued stays on the main stream
  const int group_src[2] = {src[0] >= 0 ? src[0] : src[1], src[2]};   // w[l1..) for A, Ap; w for B .. Kp
  if (group_src[1] >= 0) {
    if ((rc = sort_of(group_src[1], d_w, m, st))) return rc;
    EV_REC(e_sorted[1], st);
  }
  if (group_src[0] >= 0) {
    if ((rc = sort_of(group_src[0], d_w + l1, m, st))) return rc;
    EV_REC(e_sorted[0], st);
  }
  int next_side = 0;
  bool first = true;
  bool used[3] = {false, false, pk->g[7] != nullptr};   // G1T runs on side stream 3
  for (int j : {2, 3, 4, 5, 6, 0, 1}) {
    if (!pk->g[j]) continue;
    cudaStream_t sk = st;
    if (!first) {
      const int si = next_side++ % 3;
      sk = side[si];
      used[si] = true;
    }
    first = false;
    if (sk != st) EV_WAIT(sk, e_sorted[kPinSortSrc[j] == 2 ? 1 : 0]);
    if ((rc = buckets_of(j, sk))) return rc;
  }
  for (int si = 0; si < 3; si++)
    if (side[si] != st && (used[si] || pk->world == 1)) {
      EV_REC(e_done[si], side[si]);
      EV_WAIT(st, e_done[si]);
    }
  if (!d_recs) {
    k_pinocchio_finalize_batch<<<nblk(7 * k, kPinFinalizeBlock) + nblk(k, kPinFinalizeBlock), kPinFinalizeBlock, 0, st>>>(
        rec1, rec2, (uint32_t)k, d_out);
  } else {
    CU(cudaMemsetAsync(d_recs, 0, k * kPinRecordBytes, st));
    k_pinocchio_records_batch<<<nblk(8 * k, 256), 256, 0, st>>>(rec1, rec2, (uint32_t)k, d_recs);
  }
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}

// The k proofs of a batch at d_out + 108p (u64), or with `records` this rank's k records at d_out + 2 KB * p.  A sharded
// key without `records` computes its records, all-gathers them (k records per rank, on the key's prove-context
// communicator, on `st`) and finalises: every rank receives the k proofs.  After pinocchio_batch_check and, without
// `records`, pinocchio_batch_comm_check.  Once the records' scratch exists the all-gather runs whatever else fails, so no
// peer is left waiting; the error is then returned and nothing is finalised.
int pinocchio_batch_enqueue(ProvingKey* pk, R1cs* r1, const Fr* d_w, size_t k, Fq* d_out, bool records, cudaStream_t st,
                            int* err) {
  int rc;
  R1csBatch* fb = nullptr;
  if (pk->world == 1 || records) {
    rc = pinocchio_batch_parts(pk, r1, d_w, k, d_out, records ? reinterpret_cast<uint8_t*>(d_out) : nullptr, st, err, &fb);
  } else {
    if ((rc = pinocchio_batch_scratch(pk, k, false))) return rc;
    CU(pk->gather.ensure(kPinRecordBytes * k * (size_t)pk->world));
    ProveBatch& b = *pk->batch;
    rc = pinocchio_batch_parts(pk, r1, d_w, k, nullptr, b.parts.as<uint8_t>(), st, err, &fb);
    ncclResult_t nrc = g_comm.api.AllGather(b.parts.p, pk->gather.p, kPinRecordBytes * k, ncclUint8, pk->pctx().comm, st);
    if (rc) return rc;
    if (nrc != ncclSuccess) return fail(B200_ECOMM, "ncclAllGather: %s", g_comm.api.GetErrorString(nrc));
    k_pinocchio_gather_finalize_batch<<<pinocchio_finalize_blocks((uint32_t)k), kPinFinalizeBlock, 0, st>>>(
        pk->gather.as<uint8_t>(), pk->world, (uint32_t)k, d_out);
    g_launches += 1;
    CU(cudaGetLastError());
  }
  if (rc) return rc;
  return batch_done_record(pk, fb, st);
}

int pinocchio_prove_witness_batch(b200_pk_t h, b200_r1cs_t hr, const uint64_t* w, size_t nw, size_t k, uint64_t* out_g1,
                                  uint64_t* pi_b, std::unique_lock<std::mutex>* lk) {
  const char* what = "pinocchio_prove_witness_batch";
  ProvingKey* pk = find_pk(h, 2);
  R1cs* r1 = find_r1cs(hr);
  if (!pk || !r1) return fail(B200_EINVAL, "%s: bad handle", what);
  if (!w || !out_g1 || !pi_b) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = pinocchio_batch_check(pk, r1, nw, k, what);
  if (rc) return rc;
  if ((rc = pinocchio_batch_comm_check(pk, what))) return rc;
  if ((rc = pinocchio_batch_scratch(pk, k, true))) return rc;
  ProveBatch& b = *pk->batch;
  cudaStream_t st = pk->pctx().main;
  CU(cudaMemcpyAsync(b.w_stage.p, w, k * nw * sizeof(Fr), cudaMemcpyHostToDevice, st));
  Fq* o = b.out.as<Fq>();
  if ((rc = pinocchio_batch_enqueue(pk, r1, b.w_stage.as<Fr>(), k, o, false, st, pk->d_err_sync.as<int>()))) return rc;
  return finish_host_proof(pk, b.h_out, o, k, what, st, lk, {{out_g1, 84}, {pi_b, 24}});
}

// ---- dense QAP API (small n) -------------------------------------------------
int r1cs_to_qap_host(const uint64_t* a, const uint64_t* b, const uint64_t* c, size_t n, size_t m, uint64_t* alphas,
                     uint64_t* betas, uint64_t* gammas, uint64_t* z) {
  if (!a || !b || !c || !alphas || !betas || !gammas || !z) return fail(B200_EINVAL, "r1cs_to_qap: null pointer");
  if (n == 0 || m < 2 || n > 8191 || m > 8193) return fail(B200_EINVAL, "r1cs_to_qap: dense API supports 1 <= n <= 8191");
  cudaStream_t st = g_ctx[0].main;
  DevBuf zn, L, M, out, zz;
  size_t nz = m - 2;  // Z = prod_{i=1}^{m-2} (x - i)   (r1csqap.go:177-186)
  size_t zmax = (n > nz ? n : nz) + 1;
  CU(zn.alloc(zmax * sizeof(Fr)));
  CU(L.alloc(n * n * sizeof(Fr)));
  CU(M.alloc(n * m * sizeof(Fr)));
  CU(out.alloc(m * n * sizeof(Fr)));
  CU(zz.alloc((nz + 1) * sizeof(Fr)));
  k_zero_poly<<<1, 1024, 0, st>>>(zn.as<Fr>(), (uint32_t)n);
  k_lagrange_basis<<<nblk(n, 128), 128, 0, st>>>(zn.as<Fr>(), (uint32_t)n, L.as<Fr>());
  const uint64_t* in[3] = {a, b, c};
  uint64_t* outs[3] = {alphas, betas, gammas};
  for (int k = 0; k < 3; k++) {
    CU(cudaMemcpyAsync(M.p, in[k], n * m * sizeof(Fr), cudaMemcpyHostToDevice, st));
    dim3 grid(nblk(n, 128), (unsigned)m);
    k_qap_interpolate<<<grid, 128, 0, st>>>(M.as<Fr>(), (uint32_t)n, (uint32_t)m, L.as<Fr>(), out.as<Fr>(), g_d_err);
    CU(cudaMemcpyAsync(outs[k], out.p, m * n * sizeof(Fr), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  k_zero_poly<<<1, 1024, 0, st>>>(zn.as<Fr>(), (uint32_t)nz);
  k_poly_store<<<nblk(nz + 1, 256), 256, 0, st>>>(zn.as<Fr>(), (uint32_t)(nz + 1), 0, 1, zz.as<Fr>());
  CU(cudaMemcpyAsync(z, zz.p, (nz + 1) * sizeof(Fr), cudaMemcpyDeviceToHost, st));
  CU(cudaGetLastError());
  return check_err_flag("r1cs_to_qap", g_d_err);
}

int combine_polynomials_host(const uint64_t* r, size_t m, const uint64_t* ap, const uint64_t* bp, const uint64_t* cp,
                             size_t n, uint64_t* ax, uint64_t* bx, uint64_t* cx, uint64_t* px) {
  if (!r || !ap || !bp || !cp || !ax || !bx || !cx || !px || m == 0 || n == 0)
    return fail(B200_EINVAL, "combine_polynomials: bad arguments");
  cudaStream_t st = g_ctx[0].main;
  DevBuf dr, dP, mont[3], stdv[3], prod;
  CU(dr.alloc(m * sizeof(Fr)));
  CU(dP.alloc(m * n * sizeof(Fr)));
  CU(prod.alloc((2 * n - 1) * sizeof(Fr)));
  CU(cudaMemcpyAsync(dr.p, r, m * sizeof(Fr), cudaMemcpyHostToDevice, st));
  const uint64_t* in[3] = {ap, bp, cp};
  uint64_t* outs[3] = {ax, bx, cx};
  for (int k = 0; k < 3; k++) {
    CU(mont[k].alloc(n * sizeof(Fr)));
    CU(stdv[k].alloc(n * sizeof(Fr)));
    CU(cudaMemcpyAsync(dP.p, in[k], m * n * sizeof(Fr), cudaMemcpyHostToDevice, st));
    k_combine<<<nblk(n, 128), 128, 0, st>>>(dr.as<Fr>(), (uint32_t)m, dP.as<Fr>(), (uint32_t)n, mont[k].as<Fr>(),
                                            stdv[k].as<Fr>(), g_d_err);
    CU(cudaMemcpyAsync(outs[k], stdv[k].p, n * sizeof(Fr), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  // px = ax*bx - cx   (r1csqap.go:208)
  if (int rc = scratch_acquire(g_ctx[0], st)) return rc;
  CU(poly_mul_device(*g_ctx[0].poly, mont[0].as<Fr>(), n, 1, mont[1].as<Fr>(), n, 1, prod.as<Fr>(), g_d_err, st));
  if (int rc = scratch_release(g_ctx[0], st)) return rc;
  k_poly_addsub<<<nblk(2 * n - 1, 256), 256, 0, st>>>(prod.as<Fr>(), (uint32_t)(2 * n - 1), stdv[2].as<Fr>(), (uint32_t)n, 1,
                                                      prod.as<Fr>(), g_d_err);
  CU(cudaMemcpyAsync(px, prod.p, (2 * n - 1) * sizeof(Fr), cudaMemcpyDeviceToHost, st));
  CU(cudaGetLastError());
  return check_err_flag("combine_polynomials", g_d_err);
}

int poly_addsub_host(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, int sub, uint64_t* out) {
  size_t n = na > nb ? na : nb;
  if (n == 0) return B200_OK;
  if ((na && !a) || (nb && !b) || !out) return fail(B200_EINVAL, "poly_add/sub: null pointer");
  DevBuf da, db, dout;
  CU(da.alloc((na ? na : 1) * sizeof(Fr)));
  CU(db.alloc((nb ? nb : 1) * sizeof(Fr)));
  CU(dout.alloc(n * sizeof(Fr)));
  if (na) CU(cudaMemcpyAsync(da.p, a, na * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  if (nb) CU(cudaMemcpyAsync(db.p, b, nb * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  k_poly_addsub<<<nblk(n, 256), 256, 0, g_ctx[0].main>>>(da.as<Fr>(), (uint32_t)na, db.as<Fr>(), (uint32_t)nb, sub, dout.as<Fr>(), g_d_err);
  CU(cudaMemcpyAsync(out, dout.p, n * sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("poly_add/sub", g_d_err);
}

int poly_eval_host(const uint64_t* v, size_t n, const uint64_t* x, uint64_t* out) {
  if (!x || !out || (n && !v)) return fail(B200_EINVAL, "poly_eval: null pointer");
  DevBuf dv, dout;
  CU(dv.alloc((n ? n : 1) * sizeof(Fr)));
  CU(dout.alloc(sizeof(Fr)));
  if (n) CU(cudaMemcpyAsync(dv.p, v, n * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  Fr xs = fr_load_std(x);
  if (xs.geq_modulus()) return fail(B200_ERANGE, "poly_eval: x >= r");
  k_poly_eval<<<1, 256, 0, g_ctx[0].main>>>(dv.as<Fr>(), (uint32_t)n, xs, dout.as<Fr>(), g_d_err);
  CU(cudaMemcpyAsync(out, dout.p, sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("poly_eval", g_d_err);
}

int poly_eval_batch_host(const uint64_t* polys, size_t m, size_t n, const uint64_t* x, uint64_t* out) {
  if (!polys || !x || !out || m == 0 || n == 0) return fail(B200_EINVAL, "poly_eval_batch: bad arguments");
  Fr xs = fr_load_std(x);
  if (xs.geq_modulus()) return fail(B200_ERANGE, "poly_eval_batch: x >= r");
  DevBuf dp, dout;
  CU(dp.alloc(m * n * sizeof(Fr)));
  CU(dout.alloc(m * sizeof(Fr)));
  CU(cudaMemcpyAsync(dp.p, polys, m * n * sizeof(Fr), cudaMemcpyHostToDevice, g_ctx[0].main));
  k_poly_eval_batch<<<(unsigned)m, 64, 0, g_ctx[0].main>>>(dp.as<Fr>(), (uint32_t)n, xs, dout.as<Fr>(), g_d_err);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, dout.p, m * sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("poly_eval_batch", g_d_err);
}

// zz = the n + 1 standard-form coefficients of prod_{i=1..n} (x - i), on the device, enqueued on context 0's main stream
int zero_poly_enqueue(size_t n, DevBuf& zz) {
  if (n > ((size_t)1 << 26)) return fail(B200_EINVAL, "zero_poly: bad arguments (n <= 2^26)");
  DevBuf zn;
  CU(zz.alloc((n + 1) * sizeof(Fr)));
  if (n <= 2048) {   // one-block schoolbook; above: Newton basis element n through the subproduct tree (qap_sparse.cuh)
    CU(zn.alloc((n + 1) * sizeof(Fr)));
    k_zero_poly<<<1, 1024, 0, g_ctx[0].main>>>(zn.as<Fr>(), (uint32_t)n);
  } else {
    int rc = zero_poly_device(n, zn, g_ctx[0].main);
    if (rc) return rc;
  }
  k_poly_store<<<nblk(n + 1, 256), 256, 0, g_ctx[0].main>>>(zn.as<Fr>(), (uint32_t)(n + 1), 0, 1, zz.as<Fr>());
  CU(cudaGetLastError());
  return B200_OK;
}

int zero_poly_host(size_t n, uint64_t* out) {   // coefficients of prod_{i=1..n} (x - i), n + 1 of them
  if (!out) return fail(B200_EINVAL, "zero_poly: bad arguments (n <= 2^26)");
  DevBuf zz;
  int rc = zero_poly_enqueue(n, zz);
  if (rc) return rc;
  CU(cudaMemcpyAsync(out, zz.p, (n + 1) * sizeof(Fr), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("zero_poly", g_d_err);
}

#ifndef B200_NO_PAIRING
// ---- pairing / verification (SURVEY §8f row 2) -------------------------------------------------------
template <bool FAST_FE>
__device__ void pairing_from_jacobian(const Fq* g1, const Fq2* g2, F12& out, int* err) {
  bool bad = false;
  for (int k = 0; k < 3; k++) bad = bad || g1[k].geq_modulus() || g2[k].c0.geq_modulus() || g2[k].c1.geq_modulus();
  Jacobian<Fq> p{g1[0].to_mont(), g1[1].to_mont(), g1[2].to_mont()};
  Jacobian<Fq2> q{g2[0].to_mont(), g2[1].to_mont(), g2[2].to_mont()};
  if (bad || q.is_inf()) {  // G2 infinity: preComputeG2 panics "q1[2] != Fq2.One()" (bn128.go:238-241)
    atomicOr(err, bad ? 1 : 8);
    out = F12::one();
    return;
  }
  Affine<Fq> pa = jac_to_affine(p);                      // preComputeG1: G1.Affine, infinity -> (0, 0)
  Affine<Fq2> qa = jac_to_affine(q);
  F2::B px, py;
#pragma unroll
  for (int i = 0; i < 8; i++) { px.l[i] = pa.x.l[i]; py.l[i] = pa.y.l[i]; }
  out = pairing_affine_t<FAST_FE>(px, py, qa.x, qa.y);
}
__device__ void store_f12_std(const F12& f, Fq2* out) {
  out[0] = f.a.a.from_mont(); out[1] = f.a.b.from_mont(); out[2] = f.a.c.from_mont();
  out[3] = f.b.a.from_mont(); out[4] = f.b.b.from_mont(); out[5] = f.b.c.from_mont();
}
// out[i] = a[i] * b[i] in F_q^12 (fields/fq12.go:72-84), standard form in/out, [2][3][2] order
__global__ void __launch_bounds__(32) k_fq12_mul_batch(const Fq2* a, const Fq2* b, size_t n, Fq2* out, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F12 x, y;
  Fq2* xs = &x.a.a;
  Fq2* ys = &y.a.a;
  bool bad = false;
  for (int k = 0; k < 6; k++) {
    Fq2 u = a[6 * i + k], v = b[6 * i + k];
    bad = bad || u.geq_modulus() || v.geq_modulus();
    xs[k] = u.to_mont();
    ys[k] = v.to_mont();
  }
  if (bad) atomicOr(err, 1);
  store_f12_std(f12_mul(x, y), out + 6 * i);
}
template <bool FAST_FE>
__global__ void __launch_bounds__(32) k_pairing_batch(const Fq* g1, const Fq2* g2, size_t n, Fq2* out, int* err) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F12 f;
  pairing_from_jacobian<FAST_FE>(g1 + 3 * i, g2 + 3 * i, f, err);
  store_f12_std(f, out + 6 * i);
}
// ---- one warp per pairing (pairing_warp.cuh) ----------------------------------------------------------------------
constexpr int kPairWarps = 4;   // warps (pairings) per CTA: 4 x 9.5 KB of shared memory
// lane 0 validates and normalises the Jacobian inputs (preComputeG1 / G2.Affine); returns warp-uniformly whether a pairing
// is to be computed (false: out-of-range coordinate or G2 infinity — the reference panics, bn128.go:238-241 — result = one)
__device__ bool warp_pairing_inputs(wp::Ws& ws, const Fq* g1, const Fq2* g2, F2::B& px, F2::B& py, F2& qx, F2& qy, int* err) {
  int go = 1;
  if ((threadIdx.x & 31u) == 0) {
    bool bad = false;
    for (int k = 0; k < 3; k++) bad = bad || g1[k].geq_modulus() || g2[k].c0.geq_modulus() || g2[k].c1.geq_modulus();
    Jacobian<Fq> p{g1[0].to_mont(), g1[1].to_mont(), g1[2].to_mont()};
    Jacobian<Fq2> q{g2[0].to_mont(), g2[1].to_mont(), g2[2].to_mont()};
    if (bad || q.is_inf()) {
      atomicOr(err, bad ? 1 : 8);
      go = 0;
    } else {
      Affine<Fq> pa = jac_to_affine(p);
      Affine<Fq2> qa = jac_to_affine(q);
#pragma unroll
      for (int i = 0; i < 8; i++) { px.l[i] = pa.x.l[i]; py.l[i] = pa.y.l[i]; }
      qx = qa.x;
      qy = qa.y;
    }
  }
  (void)ws;
  return __shfl_sync(0xffffffffu, go, 0) != 0;
}
__global__ void __launch_bounds__(32 * kPairWarps) k_pairing_batch_warp(const Fq* g1, const Fq2* g2, size_t n, Fq2* out, int* err) {
  __shared__ wp::Ws wss[kPairWarps];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const size_t i = (size_t)blockIdx.x * kPairWarps + warp;
  if (i >= n) return;
  wp::Ws& ws = wss[warp];
  F2::B px, py;
  F2 qx, qy;
  if (warp_pairing_inputs(ws, g1 + 3 * i, g2 + 3 * i, px, py, qx, qy, err)) wp::pairing(ws, px, py, qx, qy);
  else wp::f12_set_one(ws, wp::RF);
  if (lane < 12) {  // standard form out, [2][3][2] order: one F_q component per lane
    const F2& c = ws.r[wp::RF][lane >> 1];
    F2::B v = ((lane & 1) ? c.c1 : c.c0).from_mont();
    Fq2* o = out + 6 * i + (lane >> 1);
    if (lane & 1) o->c1 = v;
    else o->c0 = v;
  }
}
// groth16.VerifyProof (groth16/groth16.go:281-305): e(A,B) == e(alpha,beta) * (e(icPubl,gamma) * e(C,delta)).
// Warp w of a 128-thread CTA pairs g1 with g2, the w-th of (A, alpha1, icPubl, C) and (B, beta2, gamma2, delta2) (Jacobian
// standard form); warp 0 then forms the right-hand side with two warp-wide F_q^12 products and compares.
__device__ void groth16_verify_cta(wp::Ws* wss, const Fq* g1, const Fq2* g2, int* ok, int* err) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  wp::Ws& ws = wss[warp];
  F2::B px, py;
  F2 qx, qy;
  if (warp_pairing_inputs(ws, g1, g2, px, py, qx, qy, err)) wp::pairing(ws, px, py, qx, qy);
  else wp::f12_set_one(ws, wp::RF);
  __syncthreads();
  if (warp == 0) {
    if (lane < 6) {
      ws.r[2][lane] = wss[1].r[wp::RF][lane];
      ws.r[3][lane] = wss[2].r[wp::RF][lane];
      ws.r[4][lane] = wss[3].r[wp::RF][lane];
    }
    wp::wsync();
    wp::f12_mul(ws, 3, 3, 4);
    wp::f12_mul(ws, 2, 2, 3);
    const int same = lane < 6 ? (ws.r[0][lane] == ws.r[2][lane] ? 1 : 0) : 1;
    const unsigned all = __ballot_sync(0xffffffffu, same);
    if (lane == 0) *ok = all == 0xffffffffu ? 1 : 0;
  }
}
// pts1: A, alpha1, icPubl, C ; pts2: B, beta2, gamma2, delta2
__global__ void __launch_bounds__(128) k_groth16_verify(const Fq* pts1, const Fq2* pts2, int* ok, int* err) {
  __shared__ wp::Ws wss[4];
  const uint32_t warp = threadIdx.x >> 5;
  groth16_verify_cta(wss, pts1 + 3 * warp, pts2 + 3 * warp, ok, err);
}
// k_groth16_verify over a batch, one CTA per proof (verify_batch.cuh): a regular proof under a passed aggregate is accepted
// at once, a bad one (coordinate >= q, signal >= r, PiB at infinity) gets 0, every other proof the single call's verdict.
__global__ void __launch_bounds__(128) k_vb_verify_each(const uint64_t* proofs, const vb::Vk* vk, const Fq* icp,
                                                        const uint32_t* flags, const uint32_t* agg, size_t k, int* ok,
                                                        uint32_t* status, int* err) {
  __shared__ wp::Ws wss[4];
  const size_t p = blockIdx.x;
  const uint32_t f = flags[p] | flags[k];
  if ((f & vb::kBad) || (!f && *agg)) {
    if (threadIdx.x == 0) ok[p] = (f & vb::kBad) ? 0 : 1;
    return;
  }
  if (threadIdx.x == 0) atomicOr(status, vb::kStPerProof);
  const uint32_t warp = threadIdx.x >> 5;
  const vb::ProofView v = vb::proof_at(proofs, p);
  const Fq* g1 = warp == 0 ? v.a : (warp == 1 ? vk->alpha : (warp == 2 ? icp + 3 * p : v.c));
  const Fq2* g2 = warp == 0 ? v.b : (warp == 1 ? vk->beta : (warp == 2 ? vk->gamma : vk->delta));
  groth16_verify_cta(wss, g1, g2, ok + p, err);
}
// snark.VerifyProof over a batch, one CTA per proof (verify_batch_pinocchio.cuh): a regular proof under a passed aggregate
// is accepted at once, a bad one (coordinate >= q, signal >= r, PiB at infinity) gets 0, every other proof the reference's
// verdict: its twelve pairings (warp w runs pairings 3w .. 3w + 2 with warp_pairing_inputs' semantics), the two F_q^12
// products e7 e8 and e9 e10, and the five comparisons of snark.go:292-372.
__global__ void __launch_bounds__(128) k_pvb_verify_each(const uint64_t* proofs, const vb::PVk* vk, const Fq* st,
                                                         const uint32_t* flags, const uint32_t* agg, size_t k, int* ok,
                                                         uint32_t* status, int* err) {
  __shared__ wp::Ws wss[4];
  __shared__ F2 e[vb::kPvbPairings][6];
  const size_t p = blockIdx.x;
  const uint32_t f = flags[p] | flags[k];
  if ((f & vb::kBad) || (!f && *agg)) {
    if (threadIdx.x == 0) ok[p] = (f & vb::kBad) ? 0 : 1;
    return;
  }
  if (threadIdx.x == 0) atomicOr(status, vb::kStPerProof);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  wp::Ws& ws = wss[warp];
  for (int j = 3 * (int)warp; j < 3 * (int)warp + 3; j++) {
    F2::B px, py;
    F2 qx, qy;
    if (warp_pairing_inputs(ws, vb::pvb_pairing_g1(proofs, vk, st, p, j), vb::pvb_pairing_g2(proofs, vk, p, j), px, py, qx, qy, err))
      wp::pairing(ws, px, py, qx, qy);
    else
      wp::f12_set_one(ws, wp::RF);
    if (lane < 6) e[j][lane] = ws.r[wp::RF][lane];
    wp::wsync();
  }
  __syncthreads();
  if (warp != 0) return;
  if (lane < 6) {
    ws.r[2][lane] = e[7][lane];
    ws.r[3][lane] = e[8][lane];
    ws.r[4][lane] = e[9][lane];
    ws.r[5][lane] = e[10][lane];
  }
  wp::wsync();
  wp::f12_mul(ws, 2, 2, 3);   // e(PiH, Vkz) e(PiC, g2)
  wp::f12_mul(ws, 4, 4, 5);   // e(T, G2Kbg) e(G1Kbg, PiB)
  int same = 1;
  if (lane < 6)
    same = e[0][lane] == e[1][lane] && e[2][lane] == e[3][lane] && e[4][lane] == e[5][lane] && e[6][lane] == ws.r[2][lane] &&
           ws.r[4][lane] == e[11][lane];
  const unsigned all = __ballot_sync(0xffffffffu, same);
  if (lane == 0) ok[p] = all == 0xffffffffu ? 1 : 0;
}
// icPubl = IC[0] + sum publicSignals[i] * IC[i+1] (groth16.go:283-286).  The products are independent: one half-warp each,
// with the GLV split of prove_host.cuh (128 doublings + ~12 additions deep instead of the 254 + ~127 of MulScalar's
// double-and-add; the same group element, which is all the pairing — it normalises its inputs — can see); the sum then runs
// in the reference's order with the reference's Add, so its degenerate cases (equal operands give Z = 0) are the reference's.
struct GlvScalar {
  uint64_t k[4];
  uint32_t neg[2];
};
__global__ void __launch_bounds__(32) k_ic_terms(const Fq* ic, const GlvScalar* gs, size_t npub, Jacobian<Fq>* terms, int* err) {
  const uint32_t t = threadIdx.x & 31u;
  const size_t i = (size_t)blockIdx.x * 2 + (t >> 4);
  const size_t ii = i < npub ? i : npub - 1;   // an odd count leaves the last half-warp a duplicate: every lane joins the shuffles
  const Fq* src = ic + 3 * (ii + 1);
  if (src[0].geq_modulus() || src[1].geq_modulus() || src[2].geq_modulus()) atomicOr(err, 1);
  Jacobian<Fq> p{src[0].to_mont(), src[1].to_mont(), src[2].to_mont()};
  GlvScalar g = gs[ii];
  Jacobian<Fq> r = glv_mul_halfwarp(p, g.k, g.neg, t);
  if (i < npub && (t & 15u) == 0) terms[i] = r;
}
__global__ void k_ic_sum(const Fq* ic, const Jacobian<Fq>* terms, size_t npub, Fq* out, int* err) {
  if (threadIdx.x | blockIdx.x) return;
  if (ic[0].geq_modulus() || ic[1].geq_modulus() || ic[2].geq_modulus()) atomicOr(err, 1);
  Jacobian<Fq> acc{ic[0].to_mont(), ic[1].to_mont(), ic[2].to_mont()};
  for (size_t i = 0; i < npub; i++) acc = jac_add_ref(acc, terms[i]);
  out[0] = acc.X.from_mont();
  out[1] = acc.Y.from_mont();
  out[2] = acc.Z.from_mont();
}

// Final exponentiation: Devegili-Scott-Dahab (easy part + hard part by the BN parameter), the SAME F_q^12 value as the
// reference's plain f^((q^12-1)/r) square-and-multiply (bn128.go:400-421) with ~13x fewer operations: validated on the
// GPU against the snarkjs golden vk_alfabeta_12 (K8), the bn128_test.go literal and the oracle (tests/test_gpu_verify.py,
// tests/test_host_pairing.py).  The plain routine stays in pairing.cuh as the step-by-step restatement used by the host tests.
constexpr bool kFastFinalExp = true;
int pairing_batch_host(const uint64_t* g1, const uint64_t* g2, size_t n, uint64_t* out) {
  if (!g1 || !g2 || !out) return fail(B200_EINVAL, "pairing_batch: null pointer");
  if (n == 0) return B200_OK;
  DevBuf d1, d2, dout;
  CU(d1.alloc(n * 3 * sizeof(Fq)));
  CU(d2.alloc(n * 3 * sizeof(Fq2)));
  CU(dout.alloc(n * 6 * sizeof(Fq2)));
  CU(cudaMemcpyAsync(d1.p, g1, n * 3 * sizeof(Fq), cudaMemcpyHostToDevice, g_ctx[0].main));
  CU(cudaMemcpyAsync(d2.p, g2, n * 3 * sizeof(Fq2), cudaMemcpyHostToDevice, g_ctx[0].main));
  // auto: a warp per pairing has the much shorter latency and wins for small calls; above that the thread-per-pairing
  // kernel keeps more pairings resident and has the higher throughput
  const bool thread_kernel = g_pairing_kernel == 1 || (g_pairing_kernel == 0 && n > 2048);
  if (thread_kernel) k_pairing_batch<kFastFinalExp><<<nblk(n, 32), 32, 0, g_ctx[0].main>>>(d1.as<Fq>(), d2.as<Fq2>(), n, dout.as<Fq2>(), g_d_err);
  else k_pairing_batch_warp<<<nblk(n, kPairWarps), 32 * kPairWarps, 0, g_ctx[0].main>>>(d1.as<Fq>(), d2.as<Fq2>(), n, dout.as<Fq2>(), g_d_err);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, dout.p, n * 6 * sizeof(Fq2), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("pairing_batch", g_d_err);
}

int fq12_mul_batch_host(const uint64_t* a, const uint64_t* b, size_t n, uint64_t* out) {
  if (!a || !b || !out) return fail(B200_EINVAL, "fq12_mul_batch: null pointer");
  if (n == 0) return B200_OK;
  DevBuf da, db, dout;
  size_t bytes = n * 6 * sizeof(Fq2);
  CU(da.alloc(bytes));
  CU(db.alloc(bytes));
  CU(dout.alloc(bytes));
  CU(cudaMemcpyAsync(da.p, a, bytes, cudaMemcpyHostToDevice, g_ctx[0].main));
  CU(cudaMemcpyAsync(db.p, b, bytes, cudaMemcpyHostToDevice, g_ctx[0].main));
  k_fq12_mul_batch<<<nblk(n, 32), 32, 0, g_ctx[0].main>>>(da.as<Fq2>(), db.as<Fq2>(), n, dout.as<Fq2>(), g_d_err);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, dout.p, bytes, cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("fq12_mul_batch", g_d_err);
}

int groth16_verify_host(const uint64_t* ic, size_t n_ic, const uint64_t* alpha1, const uint64_t* beta2,
                        const uint64_t* gamma2, const uint64_t* delta2, const uint64_t* pi_a, const uint64_t* pi_b,
                        const uint64_t* pi_c, const uint64_t* pub, size_t npub, int* ok) {
  if (!ic || !alpha1 || !beta2 || !gamma2 || !delta2 || !pi_a || !pi_b || !pi_c || !ok || (npub && !pub))
    return fail(B200_EINVAL, "groth16_verify: null pointer");
  if (n_ic < npub + 1) return fail(B200_EINVAL, "groth16_verify: len(IC) < len(publicSignals) + 1");
  // GLV split of every public signal on the host (they are the caller's host scalars anyway)
  std::vector<GlvScalar> gs(npub ? npub : 1);
  for (size_t i = 0; i < npub; i++) {
    Fr v = fr_load_std(pub + 4 * i);
    if (v.geq_modulus()) return fail(B200_ERANGE, "groth16_verify: scalar / coefficient >= r");
    if (glv_decompose(v, gs[i].k, gs[i].neg)) return fail(B200_EINVAL, "groth16_verify: GLV decomposition out of range");
  }
  DevBuf dic, dsig, dterms, d1, d2, dok;
  CU(dic.alloc(n_ic * 3 * sizeof(Fq)));
  CU(dsig.alloc(gs.size() * sizeof(GlvScalar)));
  CU(dterms.alloc(gs.size() * sizeof(Jacobian<Fq>)));
  CU(d1.alloc(4 * 3 * sizeof(Fq)));
  CU(d2.alloc(4 * 3 * sizeof(Fq2)));
  CU(dok.alloc(sizeof(int)));
  cudaStream_t st = g_ctx[0].main;
  CU(cudaMemcpyAsync(dic.p, ic, n_ic * 3 * sizeof(Fq), cudaMemcpyHostToDevice, st));
  if (npub) CU(cudaMemcpyAsync(dsig.p, gs.data(), npub * sizeof(GlvScalar), cudaMemcpyHostToDevice, st));
  Fq* p1 = d1.as<Fq>();
  Fq2* p2 = d2.as<Fq2>();
  CU(cudaMemcpyAsync(p1, pi_a, 3 * sizeof(Fq), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(p1 + 3, alpha1, 3 * sizeof(Fq), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(p1 + 9, pi_c, 3 * sizeof(Fq), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(p2, pi_b, 3 * sizeof(Fq2), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(p2 + 3, beta2, 3 * sizeof(Fq2), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(p2 + 6, gamma2, 3 * sizeof(Fq2), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(p2 + 9, delta2, 3 * sizeof(Fq2), cudaMemcpyHostToDevice, st));
  if (npub) k_ic_terms<<<(unsigned)((npub + 1) / 2), 32, 0, st>>>(dic.as<Fq>(), dsig.as<GlvScalar>(), npub, dterms.as<Jacobian<Fq>>(), g_d_err);
  k_ic_sum<<<1, 32, 0, st>>>(dic.as<Fq>(), dterms.as<Jacobian<Fq>>(), npub, p1 + 6, g_d_err);
  k_groth16_verify<<<1, 128, 0, st>>>(p1, p2, dok.as<int>(), g_d_err);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(ok, dok.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  return check_err_flag("groth16_verify", g_d_err);
}

// ---- batched verification (verify_batch.cuh) ----------------------------------------------------------------------------
// Stream-ordered device memory: freed behind the work queued on its stream, so a _device call returns without waiting.
struct StreamBuf {
  void* p = nullptr;
  cudaStream_t st = nullptr;
  StreamBuf() = default;
  StreamBuf(const StreamBuf&) = delete;
  StreamBuf& operator=(const StreamBuf&) = delete;
  ~StreamBuf() { if (p) cudaFreeAsync(p, st); }
  cudaError_t alloc(size_t b, cudaStream_t s) {
    st = s;
    return cudaMallocAsync(&p, b, s);
  }
};
// per-call scratch of verify_batch_enqueue, carved from one allocation
struct VbScratch {
  size_t off[10];
  size_t bytes;
  VbScratch(size_t k, size_t npub) {
    const size_t n = k + 3, nparts = (n + vb::kProdPerCta - 1) / vb::kProdPerCta;
    const size_t sz[10] = {(k + 1) * 4, 4, 4, 4, 3 * k * sizeof(Fq), (npub ? npub * k : 1) * sizeof(Jacobian<Fq>),
                           3 * k * sizeof(Jacobian<Fq>), 3 * sizeof(Jacobian<Fq>), 6 * n * sizeof(F2), 6 * nparts * sizeof(F2)};
    bytes = 0;
    for (int i = 0; i < 10; i++) {
      off[i] = bytes;
      bytes += (sz[i] + 255) & ~(size_t)255;
    }
  }
};
// Every launch of a batch verification, on `st`: d_ok[0..k) verdicts, *d_status the status bits (zeroed here first).
// A fixed launch sequence: no step waits for the host, whatever k and whatever the outcome.
int verify_batch_enqueue(const Fq* d_ic, const vb::Vk* d_vk, const uint64_t* d_proofs, const uint64_t* d_pub, size_t npub,
                         size_t k, const uint64_t* d_rho, int* d_ok, uint32_t* d_status, uint8_t* scratch, cudaStream_t st) {
  const VbScratch L(k, npub);
  uint32_t* flags = (uint32_t*)(scratch + L.off[0]);
  uint32_t* k_reg = (uint32_t*)(scratch + L.off[1]);
  uint32_t* agg = (uint32_t*)(scratch + L.off[2]);
  int* err = (int*)(scratch + L.off[3]);
  Fq* icp = (Fq*)(scratch + L.off[4]);
  Jacobian<Fq>* terms = (Jacobian<Fq>*)(scratch + L.off[5]);
  Jacobian<Fq>* rterms = (Jacobian<Fq>*)(scratch + L.off[6]);
  Jacobian<Fq>* sums = (Jacobian<Fq>*)(scratch + L.off[7]);
  F2* mvals = (F2*)(scratch + L.off[8]);
  F2* parts = (F2*)(scratch + L.off[9]);
  const size_t n = k + 3, nparts = (n + vb::kProdPerCta - 1) / vb::kProdPerCta;
  CU(cudaMemsetAsync(scratch, 0, L.off[4], st));
  CU(cudaMemsetAsync(d_status, 0, sizeof(uint32_t), st));
  vb::k_vb_classify<<<nblk(k + 1, 64), 64, 0, st>>>(d_proofs, d_vk, k, flags, d_status);
  if (npub) vb::k_vb_ic_terms<<<nblk(npub * k, 2), 32, 0, st>>>(d_ic, d_pub, npub, k, terms, flags, d_status);
  vb::k_vb_ic_sum<<<nblk(k, 64), 64, 0, st>>>(d_ic, terms, npub, k, icp, flags, d_status);
  vb::k_vb_rho_terms<<<nblk(3 * k, 2), 32, 0, st>>>(d_proofs, icp, d_rho, k, rterms);
  vb::k_vb_sums<<<1, vb::kSumThreads, 0, st>>>(d_vk, rterms, d_rho, flags, k, sums, k_reg);
  const vb::MlArgs ma{d_proofs, d_vk, rterms, sums, flags, k_reg, k};
  // the kernel rule of b200_pairing_batch (B200_CFG_PAIRING_KERNEL; auto: a warp per pair up to 2048 pairs)
  const bool thread_kernel = g_pairing_kernel == 1 || (g_pairing_kernel == 0 && n > 2048);
  if (thread_kernel) vb::k_vb_miller_thread<<<nblk(n, 32), 32, 0, st>>>(ma, n, mvals);
  else vb::k_vb_miller_warp<<<nblk(n, vb::kMlWarps), 32 * vb::kMlWarps, 0, st>>>(ma, n, mvals);
  vb::k_vb_product<<<(unsigned)nparts, 32 * vb::kProdWarps, 0, st>>>(mvals, n, parts);
  vb::k_vb_final<<<1, 32 * vb::kProdWarps, 0, st>>>(parts, nparts, k_reg, agg, d_status);
  k_vb_verify_each<<<(unsigned)k, 128, 0, st>>>(d_proofs, d_vk, icp, flags, agg, k, d_ok, d_status, err);
  g_launches += npub ? 9 : 8;
  CU(cudaGetLastError());
  return B200_OK;
}
Fq fq_load_std(const uint64_t* v) {
  Fq r;
  memcpy(&r, v, sizeof(Fq));
  return r;
}
// The checks both entries make on the host arguments of the Vk: b200_groth16_verify's, applied to the whole call.
int verify_batch_check_vk(const char* what, const uint64_t* ic, size_t n_ic, const uint64_t* alpha1, const uint64_t* beta2,
                          const uint64_t* gamma2, const uint64_t* delta2, size_t npub, size_t k, const uint64_t* rho) {
  if (!ic || !alpha1 || !beta2 || !gamma2 || !delta2 || !rho) return fail(B200_EINVAL, "%s: null pointer", what);
  if (n_ic < npub + 1) return fail(B200_EINVAL, "%s: len(IC) < len(publicSignals) + 1", what);
  if (k == 0 || k > vb::kMaxBatch) return fail(B200_EINVAL, "%s: k = %zu outside 1..%zu", what, k, vb::kMaxBatch);
  for (size_t i = 0; i < k; i++)
    if (!(rho[2 * i] | rho[2 * i + 1])) return fail(B200_EINVAL, "%s: rho[%zu] = 0", what, i);
  for (size_t i = 0; i < 3 * n_ic; i++)
    if (fq_load_std(ic + 4 * i).geq_modulus()) return fail(B200_ERANGE, "%s: IC coordinate >= q", what);
  const uint64_t* g2s[3] = {beta2, gamma2, delta2};
  for (int c = 0; c < 3; c++) {
    if (fq_load_std(alpha1 + 4 * c).geq_modulus()) return fail(B200_ERANGE, "%s: alpha1 coordinate >= q", what);
    for (int j = 0; j < 6; j++)
      if (fq_load_std(g2s[c] + 4 * j).geq_modulus()) return fail(B200_ERANGE, "%s: Vk G2 coordinate >= q", what);
  }
  for (int c = 0; c < 3; c++)
    if (!(g2s[c][16] | g2s[c][17] | g2s[c][18] | g2s[c][19] | g2s[c][20] | g2s[c][21] | g2s[c][22] | g2s[c][23]))
      return fail(B200_EINVAL, "%s: q1[2] != Fq2.One() (Vk G2 point at infinity; the reference panics, bn128.go:238-241)", what);
  return B200_OK;
}
// device image of the Vk, IC and rho: vb::Vk | IC | rho
size_t vb_vk_bytes(size_t n_ic, size_t k) { return sizeof(vb::Vk) + n_ic * 3 * sizeof(Fq) + 2 * k * sizeof(uint64_t); }
int vb_upload_vk(uint8_t* d, const uint64_t* ic, size_t n_ic, const uint64_t* alpha1, const uint64_t* beta2, const uint64_t* gamma2,
                 const uint64_t* delta2, size_t k, const uint64_t* rho, cudaStream_t st) {
  std::vector<uint8_t> h(vb_vk_bytes(n_ic, k));
  vb::Vk* v = (vb::Vk*)h.data();
  std::memcpy(v->alpha, alpha1, sizeof v->alpha);
  std::memcpy(v->beta, beta2, sizeof v->beta);
  std::memcpy(v->gamma, gamma2, sizeof v->gamma);
  std::memcpy(v->delta, delta2, sizeof v->delta);
  std::memcpy(h.data() + sizeof(vb::Vk), ic, n_ic * 3 * sizeof(Fq));
  std::memcpy(h.data() + sizeof(vb::Vk) + n_ic * 3 * sizeof(Fq), rho, 2 * k * sizeof(uint64_t));
  CU(cudaMemcpyAsync(d, h.data(), h.size(), cudaMemcpyHostToDevice, st));
  return B200_OK;
}
int groth16_verify_batch_host(const uint64_t* ic, size_t n_ic, const uint64_t* alpha1, const uint64_t* beta2, const uint64_t* gamma2,
                              const uint64_t* delta2, const uint64_t* pi_a, const uint64_t* pi_b, const uint64_t* pi_c,
                              const uint64_t* pub, size_t npub, size_t k, const uint64_t* rho, int* ok, uint32_t* status) {
  const char* what = "groth16_verify_batch";
  if (!pi_a || !pi_b || !pi_c || !ok || (npub && !pub)) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = verify_batch_check_vk(what, ic, n_ic, alpha1, beta2, gamma2, delta2, npub, k, rho);
  if (rc) return rc;
  for (size_t i = 0; i < k * npub; i++)
    if (fr_load_std(pub + 4 * i).geq_modulus()) return fail(B200_ERANGE, "%s: scalar / coefficient >= r", what);
  // the batch prover's layout, PiA | PiC | PiB per proof
  std::vector<uint64_t> proofs(48 * k);
  for (size_t p = 0; p < k; p++) {
    std::memcpy(&proofs[48 * p], pi_a + 12 * p, 12 * sizeof(uint64_t));
    std::memcpy(&proofs[48 * p + 12], pi_c + 12 * p, 12 * sizeof(uint64_t));
    std::memcpy(&proofs[48 * p + 24], pi_b + 24 * p, 24 * sizeof(uint64_t));
  }
  for (size_t i = 0; i < 12 * k; i++)
    if (fq_load_std(&proofs[4 * i]).geq_modulus()) return fail(B200_ERANGE, "%s: point coordinate >= q", what);
  for (size_t p = 0; p < k; p++) {
    const uint64_t* z = &proofs[48 * p + 40];
    if (!(z[0] | z[1] | z[2] | z[3] | z[4] | z[5] | z[6] | z[7]))
      return fail(B200_EINVAL, "%s: q1[2] != Fq2.One() (PiB of proof %zu at infinity; the reference panics, bn128.go:238-241)", what, p);
  }
  cudaStream_t st = g_ctx[0].main;
  const size_t vkb = vb_vk_bytes(n_ic, k), pb = proofs.size() * sizeof(uint64_t), ub = (npub ? npub : 1) * k * 32,
               okb = (k + 1) * sizeof(int);
  const VbScratch L(k, npub);
  StreamBuf buf;
  CU(buf.alloc(vkb + pb + ub + okb + L.bytes + 1024, st));
  uint8_t* d = (uint8_t*)buf.p;
  auto carve = [&](size_t b) { uint8_t* r = d; d += (b + 255) & ~(size_t)255; return r; };
  uint8_t* d_vk = carve(vkb);
  uint64_t* d_proofs = (uint64_t*)carve(pb);
  uint64_t* d_pub = (uint64_t*)carve(ub);
  int* d_ok = (int*)carve(okb);
  uint8_t* d_scratch = carve(L.bytes);
  if ((rc = vb_upload_vk(d_vk, ic, n_ic, alpha1, beta2, gamma2, delta2, k, rho, st))) return rc;
  CU(cudaMemcpyAsync(d_proofs, proofs.data(), pb, cudaMemcpyHostToDevice, st));
  if (npub) CU(cudaMemcpyAsync(d_pub, pub, npub * k * 32, cudaMemcpyHostToDevice, st));
  const Fq* d_ic = (const Fq*)(d_vk + sizeof(vb::Vk));
  const uint64_t* d_rho = (const uint64_t*)(d_vk + sizeof(vb::Vk) + n_ic * 3 * sizeof(Fq));
  if ((rc = verify_batch_enqueue(d_ic, (const vb::Vk*)d_vk, d_proofs, d_pub, npub, k, d_rho, d_ok, (uint32_t*)(d_ok + k),
                                 d_scratch, st)))
    return rc;
  std::vector<int> h_ok(k + 1);
  CU(cudaMemcpyAsync(h_ok.data(), d_ok, okb, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  std::memcpy(ok, h_ok.data(), k * sizeof(int));
  if (status) *status = (uint32_t)h_ok[k];
  return B200_OK;
}
int groth16_verify_batch_device(const uint64_t* ic, size_t n_ic, const uint64_t* alpha1, const uint64_t* beta2,
                                const uint64_t* gamma2, const uint64_t* delta2, const void* d_proofs, const void* d_public,
                                size_t npub, size_t k, const uint64_t* rho, void* d_ok, cudaStream_t st) {
  const char* what = "groth16_verify_batch_device";
  if (!d_proofs || !d_ok || (npub && !d_public)) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = verify_batch_check_vk(what, ic, n_ic, alpha1, beta2, gamma2, delta2, npub, k, rho);
  if (rc) return rc;
  const size_t vkb = (vb_vk_bytes(n_ic, k) + 255) & ~(size_t)255;
  const VbScratch L(k, npub);
  StreamBuf buf;
  CU(buf.alloc(vkb + L.bytes, st));
  uint8_t* d = (uint8_t*)buf.p;
  if ((rc = vb_upload_vk(d, ic, n_ic, alpha1, beta2, gamma2, delta2, k, rho, st))) return rc;
  return verify_batch_enqueue((const Fq*)(d + sizeof(vb::Vk)), (const vb::Vk*)d, (const uint64_t*)d_proofs,
                              (const uint64_t*)d_public, npub, k, (const uint64_t*)(d + sizeof(vb::Vk) + n_ic * 3 * sizeof(Fq)),
                              (int*)d_ok, (uint32_t*)((int*)d_ok + k), d + vkb, st);
}

// ---- batched Pinocchio verification (verify_batch_pinocchio.cuh) ------------------------------------------------------
// per-call scratch of pvb_enqueue, carved from one allocation
struct PvbScratch {
  size_t off[10];
  size_t bytes;
  PvbScratch(size_t k, size_t npub) {
    const size_t n = k + vb::kPvbSums, nparts = (n + vb::kProdPerCta - 1) / vb::kProdPerCta;
    const size_t sz[10] = {(k + 1) * 4, 4, 4, 4, 6 * k * sizeof(Fq), (npub ? npub * k : 1) * sizeof(Jacobian<Fq>),
                           vb::kPvbRhoTerms * k * sizeof(Jacobian<Fq>), vb::kPvbSums * sizeof(Jacobian<Fq>),
                           6 * n * sizeof(F2), 6 * nparts * sizeof(F2)};
    bytes = 0;
    for (int i = 0; i < 10; i++) {
      off[i] = bytes;
      bytes += (sz[i] + 255) & ~(size_t)255;
    }
  }
};
// Every launch of a batched Pinocchio verification, on `st`: d_ok[0..k) verdicts, *d_status the status bits (zeroed here
// first).  A fixed launch sequence: no step waits for the host, whatever k and whatever the outcome.
int pvb_enqueue(const Fq* d_ic, const vb::PVk* d_vk, const uint64_t* d_proofs, const uint64_t* d_pub, size_t npub, size_t k,
                const uint64_t* d_rho, int* d_ok, uint32_t* d_status, uint8_t* scratch, cudaStream_t st) {
  const PvbScratch L(k, npub);
  uint32_t* flags = (uint32_t*)(scratch + L.off[0]);
  uint32_t* k_reg = (uint32_t*)(scratch + L.off[1]);
  uint32_t* agg = (uint32_t*)(scratch + L.off[2]);
  int* err = (int*)(scratch + L.off[3]);
  Fq* sts = (Fq*)(scratch + L.off[4]);
  Jacobian<Fq>* terms = (Jacobian<Fq>*)(scratch + L.off[5]);
  Jacobian<Fq>* rterms = (Jacobian<Fq>*)(scratch + L.off[6]);
  Jacobian<Fq>* sums = (Jacobian<Fq>*)(scratch + L.off[7]);
  F2* mvals = (F2*)(scratch + L.off[8]);
  F2* parts = (F2*)(scratch + L.off[9]);
  const size_t n = k + vb::kPvbSums, nparts = (n + vb::kProdPerCta - 1) / vb::kProdPerCta;
  CU(cudaMemsetAsync(scratch, 0, L.off[4], st));
  CU(cudaMemsetAsync(d_status, 0, sizeof(uint32_t), st));
  vb::k_pvb_classify<<<nblk(k + 7, 64), 64, 0, st>>>(d_proofs, d_vk, k, flags, d_status);
  if (npub) vb::k_vb_ic_terms<<<nblk(npub * k, 2), 32, 0, st>>>(d_ic, d_pub, npub, k, terms, flags, d_status);
  vb::k_pvb_st<<<nblk(k, 64), 64, 0, st>>>(d_ic, terms, d_proofs, npub, k, sts, flags, d_status);
  vb::k_pvb_rho_terms<<<nblk(vb::kPvbRhoTerms * k, 2), 32, 0, st>>>(d_proofs, d_vk, sts, d_rho, k, rterms);
  vb::k_pvb_sums<<<vb::kPvbSums, vb::kSumThreads, 0, st>>>(rterms, flags, k, sums, k_reg);
  const vb::PvbMlArgs ma{d_proofs, d_vk, rterms, sums, flags, k_reg, k};
  // the kernel rule of b200_pairing_batch (B200_CFG_PAIRING_KERNEL; auto: a warp per pair up to 2048 pairs)
  const bool thread_kernel = g_pairing_kernel == 1 || (g_pairing_kernel == 0 && n > 2048);
  if (thread_kernel) vb::k_vb_miller_thread<<<nblk(n, 32), 32, 0, st>>>(ma, n, mvals);
  else vb::k_vb_miller_warp<<<nblk(n, vb::kMlWarps), 32 * vb::kMlWarps, 0, st>>>(ma, n, mvals);
  vb::k_vb_product<<<(unsigned)nparts, 32 * vb::kProdWarps, 0, st>>>(mvals, n, parts);
  vb::k_vb_final<<<1, 32 * vb::kProdWarps, 0, st>>>(parts, nparts, k_reg, agg, d_status);
  k_pvb_verify_each<<<(unsigned)k, 128, 0, st>>>(d_proofs, d_vk, sts, flags, agg, k, d_ok, d_status, err);
  g_launches += npub ? 9 : 8;
  CU(cudaGetLastError());
  return B200_OK;
}
// The checks both entries make on the host arguments of the Vk, IC and rho.
int pvb_check_vk(const char* what, const uint64_t* ic, size_t n_ic, const uint64_t* vk_g1, const uint64_t* vk_g2, size_t npub,
                 size_t k, const uint64_t* rho) {
  if (!ic || !vk_g1 || !vk_g2 || !rho) return fail(B200_EINVAL, "%s: null pointer", what);
  if (n_ic < npub + 1) return fail(B200_EINVAL, "%s: len(IC) < len(publicSignals) + 1", what);
  if (k == 0 || k > vb::kMaxBatch) return fail(B200_EINVAL, "%s: k = %zu outside 1..%zu", what, k, vb::kMaxBatch);
  for (size_t i = 0; i < 5 * k; i++)
    if (!(rho[2 * i] | rho[2 * i + 1])) return fail(B200_EINVAL, "%s: rho[%zu][%zu] = 0", what, i / 5, i % 5 + 1);
  for (size_t i = 0; i < 3 * n_ic; i++)
    if (fq_load_std(ic + 4 * i).geq_modulus()) return fail(B200_ERANGE, "%s: IC coordinate >= q", what);
  for (int i = 0; i < 6; i++)
    if (fq_load_std(vk_g1 + 4 * i).geq_modulus()) return fail(B200_ERANGE, "%s: Vk G1 coordinate >= q", what);
  for (int i = 0; i < 30; i++)
    if (fq_load_std(vk_g2 + 4 * i).geq_modulus()) return fail(B200_ERANGE, "%s: Vk G2 coordinate >= q", what);
  for (int c = 0; c < 5; c++) {
    const uint64_t* z = vk_g2 + 24 * c + 16;
    if (!(z[0] | z[1] | z[2] | z[3] | z[4] | z[5] | z[6] | z[7]))
      return fail(B200_EINVAL, "%s: q1[2] != Fq2.One() (Vk G2 point at infinity; the reference panics, bn128.go:238-241)", what);
  }
  return B200_OK;
}
// device image of the Vk, IC and rho: vb::PVk | IC | rho
size_t pvb_vk_bytes(size_t n_ic, size_t k) { return sizeof(vb::PVk) + n_ic * 3 * sizeof(Fq) + 10 * k * sizeof(uint64_t); }
int pvb_upload_vk(uint8_t* d, const uint64_t* ic, size_t n_ic, const uint64_t* vk_g1, const uint64_t* vk_g2, size_t k,
                  const uint64_t* rho, cudaStream_t st) {
  static_assert(sizeof(vb::PVk) == (24 + 120 + 24) * sizeof(uint64_t), "PVk is vk_g1 | vk_g2 | g2");
  std::vector<uint8_t> h(pvb_vk_bytes(n_ic, k));
  std::memcpy(h.data(), vk_g1, 24 * sizeof(uint64_t));
  std::memcpy(h.data() + 24 * sizeof(uint64_t), vk_g2, 120 * sizeof(uint64_t));
  std::memcpy(h.data() + 144 * sizeof(uint64_t), kG2GenJacStd, 24 * sizeof(uint64_t));
  std::memcpy(h.data() + sizeof(vb::PVk), ic, n_ic * 3 * sizeof(Fq));
  std::memcpy(h.data() + sizeof(vb::PVk) + n_ic * 3 * sizeof(Fq), rho, 10 * k * sizeof(uint64_t));
  CU(cudaMemcpyAsync(d, h.data(), h.size(), cudaMemcpyHostToDevice, st));
  return B200_OK;
}
int pinocchio_verify_batch_host(const uint64_t* ic, size_t n_ic, const uint64_t* vk_g1, const uint64_t* vk_g2,
                                const uint64_t* out_g1, const uint64_t* pi_b, const uint64_t* pub, size_t npub, size_t k,
                                const uint64_t* rho, int* ok, uint32_t* status) {
  const char* what = "pinocchio_verify_batch";
  if (!out_g1 || !pi_b || !ok || (npub && !pub)) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = pvb_check_vk(what, ic, n_ic, vk_g1, vk_g2, npub, k, rho);
  if (rc) return rc;
  for (size_t i = 0; i < k * npub; i++)
    if (fr_load_std(pub + 4 * i).geq_modulus()) return fail(B200_ERANGE, "%s: scalar / coefficient >= r", what);
  // the batch prover's device layout: the seven G1 points, then PiB, per proof
  std::vector<uint64_t> proofs(vb::kPvbProofWords * k);
  for (size_t p = 0; p < k; p++) {
    std::memcpy(&proofs[vb::kPvbProofWords * p], out_g1 + 84 * p, 84 * sizeof(uint64_t));
    std::memcpy(&proofs[vb::kPvbProofWords * p + 84], pi_b + 24 * p, 24 * sizeof(uint64_t));
  }
  for (size_t i = 0; i < 27 * k; i++)
    if (fq_load_std(&proofs[4 * i]).geq_modulus()) return fail(B200_ERANGE, "%s: point coordinate >= q", what);
  for (size_t p = 0; p < k; p++) {
    const uint64_t* z = &proofs[vb::kPvbProofWords * p + 100];
    if (!(z[0] | z[1] | z[2] | z[3] | z[4] | z[5] | z[6] | z[7]))
      return fail(B200_EINVAL, "%s: q1[2] != Fq2.One() (PiB of proof %zu at infinity; the reference panics, bn128.go:238-241)", what, p);
  }
  cudaStream_t st = g_ctx[0].main;
  const size_t vkb = pvb_vk_bytes(n_ic, k), pb = proofs.size() * sizeof(uint64_t), ub = (npub ? npub : 1) * k * 32,
               okb = (k + 1) * sizeof(int);
  const PvbScratch L(k, npub);
  StreamBuf buf;
  CU(buf.alloc(vkb + pb + ub + okb + L.bytes + 1024, st));
  uint8_t* d = (uint8_t*)buf.p;
  auto carve = [&](size_t b) { uint8_t* r = d; d += (b + 255) & ~(size_t)255; return r; };
  uint8_t* d_vk = carve(vkb);
  uint64_t* d_proofs = (uint64_t*)carve(pb);
  uint64_t* d_pub = (uint64_t*)carve(ub);
  int* d_ok = (int*)carve(okb);
  uint8_t* d_scratch = carve(L.bytes);
  if ((rc = pvb_upload_vk(d_vk, ic, n_ic, vk_g1, vk_g2, k, rho, st))) return rc;
  CU(cudaMemcpyAsync(d_proofs, proofs.data(), pb, cudaMemcpyHostToDevice, st));
  if (npub) CU(cudaMemcpyAsync(d_pub, pub, npub * k * 32, cudaMemcpyHostToDevice, st));
  const Fq* d_ic = (const Fq*)(d_vk + sizeof(vb::PVk));
  const uint64_t* d_rho = (const uint64_t*)(d_vk + sizeof(vb::PVk) + n_ic * 3 * sizeof(Fq));
  if ((rc = pvb_enqueue(d_ic, (const vb::PVk*)d_vk, d_proofs, d_pub, npub, k, d_rho, d_ok, (uint32_t*)(d_ok + k), d_scratch, st)))
    return rc;
  std::vector<int> h_ok(k + 1);
  CU(cudaMemcpyAsync(h_ok.data(), d_ok, okb, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  std::memcpy(ok, h_ok.data(), k * sizeof(int));
  if (status) *status = (uint32_t)h_ok[k];
  return B200_OK;
}
int pinocchio_verify_batch_device(const uint64_t* ic, size_t n_ic, const uint64_t* vk_g1, const uint64_t* vk_g2,
                                  const void* d_proofs, const void* d_public, size_t npub, size_t k, const uint64_t* rho,
                                  void* d_ok, cudaStream_t st) {
  const char* what = "pinocchio_verify_batch_device";
  if (!d_proofs || !d_ok || (npub && !d_public)) return fail(B200_EINVAL, "%s: null pointer", what);
  int rc = pvb_check_vk(what, ic, n_ic, vk_g1, vk_g2, npub, k, rho);
  if (rc) return rc;
  const size_t vkb = (pvb_vk_bytes(n_ic, k) + 255) & ~(size_t)255;
  const PvbScratch L(k, npub);
  StreamBuf buf;
  CU(buf.alloc(vkb + L.bytes, st));
  uint8_t* d = (uint8_t*)buf.p;
  if ((rc = pvb_upload_vk(d, ic, n_ic, vk_g1, vk_g2, k, rho, st))) return rc;
  return pvb_enqueue((const Fq*)(d + sizeof(vb::PVk)), (const vb::PVk*)d, (const uint64_t*)d_proofs, (const uint64_t*)d_public,
                     npub, k, (const uint64_t*)(d + sizeof(vb::PVk) + n_ic * 3 * sizeof(Fq)), (int*)d_ok,
                     (uint32_t*)((int*)d_ok + k), d + vkb, st);
}

#else  // experiment builds without the verifier side (ptxas 12.9 crashes on the pairing kernels under -DB200_KARATSUBA)
int pairing_batch_host(const uint64_t*, const uint64_t*, size_t, uint64_t*) { return fail(B200_EINVAL, "pairing: not in this build variant"); }
int groth16_verify_batch_host(const uint64_t*, size_t, const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*,
                              const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*, size_t, size_t, const uint64_t*,
                              int*, uint32_t*) {
  return fail(B200_EINVAL, "groth16_verify_batch: not in this build variant");
}
int groth16_verify_batch_device(const uint64_t*, size_t, const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*,
                                const void*, const void*, size_t, size_t, const uint64_t*, void*, cudaStream_t) {
  return fail(B200_EINVAL, "groth16_verify_batch_device: not in this build variant");
}
int pinocchio_verify_batch_host(const uint64_t*, size_t, const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*,
                                const uint64_t*, size_t, size_t, const uint64_t*, int*, uint32_t*) {
  return fail(B200_EINVAL, "pinocchio_verify_batch: not in this build variant");
}
int pinocchio_verify_batch_device(const uint64_t*, size_t, const uint64_t*, const uint64_t*, const void*, const void*, size_t,
                                  size_t, const uint64_t*, void*, cudaStream_t) {
  return fail(B200_EINVAL, "pinocchio_verify_batch_device: not in this build variant");
}
int fq12_mul_batch_host(const uint64_t*, const uint64_t*, size_t, uint64_t*) { return fail(B200_EINVAL, "fq12_mul: not in this build variant"); }
int groth16_verify_host(const uint64_t*, size_t, const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*, const uint64_t*,
                        const uint64_t*, const uint64_t*, const uint64_t*, size_t, int*) {
  return fail(B200_EINVAL, "groth16_verify: not in this build variant");
}
#endif

template <class F>
int group_op_host(int op, const uint64_t* p, const uint64_t* q, size_t n, uint64_t* out) {
  if (!p || !out || (op == 0 && !q)) return fail(B200_EINVAL, "group op: null pointer");
  if (n == 0) return B200_OK;
  DevBuf dp, dq, dout;
  size_t out_fe = op == 3 ? 2 : 3;
  CU(dp.alloc(n * 3 * sizeof(F)));
  CU(dout.alloc(n * out_fe * sizeof(F)));
  CU(cudaMemcpyAsync(dp.p, p, n * 3 * sizeof(F), cudaMemcpyHostToDevice, g_ctx[0].main));
  if (op == 0) {
    CU(dq.alloc(n * 3 * sizeof(F)));
    CU(cudaMemcpyAsync(dq.p, q, n * 3 * sizeof(F), cudaMemcpyHostToDevice, g_ctx[0].main));
  }
  if (op == 3)
    k_group_affine<F><<<nblk(n, 128), 128, 0, g_ctx[0].main>>>(dp.as<F>(), n, dout.as<F>(), g_d_err);
  else
    k_group_op<F><<<nblk(n, 128), 128, 0, g_ctx[0].main>>>(op, dp.as<F>(), dq.as<F>(), n, dout.as<F>(), g_d_err);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, dout.p, n * out_fe * sizeof(F), cudaMemcpyDeviceToHost, g_ctx[0].main));
  return check_err_flag("group op", g_d_err);
}

#include "setup_host.cuh"

}  // namespace

// On an error return, work already queued on the library's streams is drained first: no entry point leaves kernels in
// flight that still read the caller's (or the library's soon-to-be-reused) buffers.
inline int drain_on_error(int rc) {
  if (rc != B200_OK && g_init) cudaDeviceSynchronize();
  return rc;
}
extern "C" {

int b200_groth16_pk_load(const uint64_t* at, const uint64_t* b1, const uint64_t* b2, const uint64_t* bacdelta,
                         size_t m, const uint64_t* ptd, size_t n_ptd, const uint64_t* z, size_t nz,
                         const uint64_t alpha1[12], const uint64_t beta1[12], const uint64_t delta1[12],
                         const uint64_t beta2[24], const uint64_t delta2[24], size_t npublic, int window_bits,
                         b200_pk_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return groth16_pk_load(at, b1, b2, bacdelta, m, ptd, n_ptd, z, nz, alpha1, beta1, delta1, beta2, delta2, npublic,
                         window_bits, 0, 1, out);
}
int b200_groth16_pk_load_shard(const uint64_t* at, const uint64_t* b1, const uint64_t* b2, const uint64_t* bacdelta,
                               size_t m, const uint64_t* ptd, size_t n_ptd, const uint64_t* z, size_t nz,
                               const uint64_t alpha1[12], const uint64_t beta1[12], const uint64_t delta1[12],
                               const uint64_t beta2[24], const uint64_t delta2[24], size_t npublic, int window_bits,
                               int rank, int world, b200_pk_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return groth16_pk_load(at, b1, b2, bacdelta, m, ptd, n_ptd, z, nz, alpha1, beta1, delta1, beta2, delta2, npublic,
                         window_bits, rank, world, out);
}
int b200_groth16_finalize_device(b200_pk_t pk, const void* d_parts, int nparts, const uint64_t r[4],
                                 const uint64_t s[4], void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  ProvingKey* p = find_pk(pk, 1);
  if (!p || !d_parts || nparts < 1 || !r || !s || !d_out) return fail(B200_EINVAL, "groth16_finalize_device: bad arguments");
  return drain_on_error(groth16_finalize_enqueue(p, (const uint8_t*)d_parts, nparts, r, s, (Fq*)d_out,
                                  stream ? (cudaStream_t)stream : g_ctx[0].main));
}
int b200_groth16_prove(b200_pk_t pk, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx,
                       const uint64_t r[4], const uint64_t s[4], uint64_t pi_a[12], uint64_t pi_b[24],
                       uint64_t pi_c[12]) {
  std::unique_lock<std::mutex> lk(g_mu);
  NEED_INIT();
  return drain_on_error(groth16_prove(pk, w, nw, px, npx, r, s, pi_a, pi_b, pi_c, &lk));
}
int b200_pinocchio_pk_load(const uint64_t* a, const uint64_t* ap, const uint64_t* b2, const uint64_t* bp,
                           const uint64_t* c, const uint64_t* cp, const uint64_t* kp, size_t m,
                           const uint64_t* g1t, size_t n_g1t, const uint64_t* z, size_t nz, size_t npublic,
                           int window_bits, b200_pk_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return pinocchio_pk_load(a, ap, b2, bp, c, cp, kp, m, g1t, n_g1t, z, nz, npublic, window_bits, 0, 1, out);
}
int b200_pinocchio_pk_load_shard(const uint64_t* a, const uint64_t* ap, const uint64_t* b2, const uint64_t* bp,
                                 const uint64_t* c, const uint64_t* cp, const uint64_t* kp, size_t m,
                                 const uint64_t* g1t, size_t n_g1t, const uint64_t* z, size_t nz, size_t npublic,
                                 int window_bits, int rank, int world, b200_pk_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return pinocchio_pk_load(a, ap, b2, bp, c, cp, kp, m, g1t, n_g1t, z, nz, npublic, window_bits, rank, world, out);
}
int b200_pinocchio_prove_record_device(b200_pk_t pk, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx, void* d_record) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  if (!d_record) return fail(B200_EINVAL, "pinocchio_prove_record_device: null record pointer");
  return pinocchio_prove(pk, w, nw, px, npx, nullptr, nullptr, (uint8_t*)d_record);
}
int b200_pinocchio_finalize_records(const void* d_records, int world, uint64_t* out_g1, uint64_t pi_b[24]) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return pinocchio_finalize_records((const uint8_t*)d_records, world, out_g1, pi_b);
}
int b200_pinocchio_prove(b200_pk_t pk, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx,
                         uint64_t* out_g1 /* 7 x 12: PiA PiAp PiBp PiC PiCp PiH PiKp */, uint64_t pi_b[24]) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return drain_on_error(pinocchio_prove(pk, w, nw, px, npx, out_g1, pi_b));
}
int b200_groth16_prove_device(b200_pk_t pk, const void* d_w, size_t nw, const void* d_px, size_t npx,
                              const uint64_t r[4], const uint64_t s[4], void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  ProvingKey* p = find_pk(pk, 1);
  if (!p || !d_w || !d_px || !r || !s || !d_out) return fail(B200_EINVAL, "groth16_prove_device: bad arguments");
  return drain_on_error(groth16_enqueue(p, (const Fr*)d_w, nw, (const Fr*)d_px, npx, r, s, (Fq*)d_out,
                         stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_comm_unique_id(uint8_t out[128]) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!out) return fail(B200_EINVAL, "comm_unique_id: null pointer");
  if (const char* e = g_comm.api.load()) return fail(B200_ECOMM, "comm_unique_id: %s", e);
  ncclUniqueId id;
  ncclResult_t rc = g_comm.api.GetUniqueId(&id);
  if (rc != ncclSuccess) return fail(B200_ECOMM, "ncclGetUniqueId: %s", g_comm.api.GetErrorString(rc));
  memcpy(out, &id, 128);
  return B200_OK;
}
int b200_comm_init(const uint8_t id[128], int rank, int world) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  if (!id || world < 1 || rank < 0 || rank >= world) return fail(B200_EINVAL, "comm_init: bad arguments");
  if (comm_active()) return fail(B200_EINVAL, "comm_init: communicator already initialised (rank %d/%d)", g_comm.rank, g_comm.world);
  if (const char* e = g_comm.api.load()) return fail(B200_ECOMM, "comm_init: %s", e);
  ncclUniqueId uid;
  memcpy(&uid, id, 128);
  ncclComm_t comm = nullptr;
  ncclResult_t rc = g_comm.api.CommInitRank(&comm, world, uid, rank);
  if (rc != ncclSuccess) return fail(B200_ECOMM, "ncclCommInitRank: %s", g_comm.api.GetErrorString(rc));
  g_comm.rank = rank;
  g_comm.world = world;
  // context 1's communicator (collective: every rank is inside b200_comm_init); older NCCL without ncclCommSplit: both
  // contexts share context 0's and only ONE host thread may prove on sharded keys
  g_ctx[0].comm = g_ctx[1].comm = comm;
  ncclComm_t split = nullptr;
  if (g_comm.api.CommSplit && world > 1 && g_comm.api.CommSplit(comm, 0, rank, &split, nullptr) == ncclSuccess)
    g_ctx[1].comm = split;
  return B200_OK;
}
int b200_comm_destroy(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  comm_destroy_locked();
  return B200_OK;
}
int b200_groth16_shard_info(b200_pk_t pk, uint64_t out[12]) {
  std::lock_guard<std::mutex> lk(g_mu);
  ProvingKey* p = find_pk(pk, 1);
  if (!p || !out) return fail(B200_EINVAL, "groth16_shard_info: bad arguments");
  const size_t l1 = p->npublic + 1, ncf = p->n_c_full;
  for (int k = 0; k < 3; k++) { out[2 * k] = p->lo[k]; out[2 * k + 1] = p->hi[k]; }
  size_t lo3 = p->lo[3], hi3 = p->hi[3];
  size_t c_lo = lo3 < ncf ? lo3 : ncf, c_hi = hi3 < ncf ? hi3 : ncf;
  out[6] = l1 + c_lo;                       // witness range feeding this rank's C part
  out[7] = l1 + c_hi;
  out[8] = hi3 > ncf ? 1 : 0;               // holds PowersTauDelta indices => needs px
  out[9] = (uint64_t)p->rank;
  out[10] = (uint64_t)p->world;
  out[11] = p->m;
  return B200_OK;
}
int b200_profile(int enable) {
  std::lock_guard<std::mutex> lk(g_mu);
  g_prof = (enable & 1) != 0;
  g_serial = (enable & 2) != 0;
  return B200_OK;
}
int b200_profile_read(double out[8]) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  if (!out) return fail(B200_EINVAL, "profile_read: null pointer");
  for (int i = 0; i < 8; i++) out[i] = 0;
  CU(cudaDeviceSynchronize());
  for (auto& r : g_prof_recs) {
    float ms = 0;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    int o = r.group == 1 ? 0 : 3;
    out[o] += ms;
    out[o + 1] += 1;
    out[o + 2] += (double)r.terms;
    g_event_pool.push_back(r.e0);
    g_event_pool.push_back(r.e1);
  }
  g_prof_recs.clear();
  out[6] = (double)g_launches;
  g_launches = 0;
  return B200_OK;
}
int b200_pk_free(b200_pk_t pk) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_init) return fail(B200_EINVAL, "not initialised");
  cudaSetDevice(g_device);
  cudaStreamSynchronize(g_ctx[0].main);
  return g_pks.erase(pk) ? B200_OK : fail(B200_EINVAL, "pk_free: bad handle");
}
int b200_pk_device_bytes(b200_pk_t h, size_t* bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_pks.find(h);
  if (it == g_pks.end() || !bytes) return fail(B200_EINVAL, "pk_device_bytes: bad handle");
  *bytes = pk_device_bytes(*it->second);
  return B200_OK;
}

#define B200_API_BODY(expr)              \
  std::lock_guard<std::mutex> lk(g_mu);  \
  NEED_INIT();                           \
  return drain_on_error(expr);
int b200_r1cs_to_qap(const uint64_t* a, const uint64_t* b, const uint64_t* c, size_t n, size_t m, uint64_t* alphas,
                     uint64_t* betas, uint64_t* gammas, uint64_t* z) {
  B200_API_BODY(r1cs_to_qap_host(a, b, c, n, m, alphas, betas, gammas, z))
}
int b200_combine_polynomials(const uint64_t* r, size_t m, const uint64_t* ap, const uint64_t* bp, const uint64_t* cp,
                             size_t n, uint64_t* ax, uint64_t* bx, uint64_t* cx, uint64_t* px) {
  B200_API_BODY(combine_polynomials_host(r, m, ap, bp, cp, n, ax, bx, cx, px))
}
int b200_poly_add(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out) { B200_API_BODY(poly_addsub_host(a, na, b, nb, 0, out)) }
int b200_poly_sub(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out) { B200_API_BODY(poly_addsub_host(a, na, b, nb, 1, out)) }
int b200_poly_eval(const uint64_t* v, size_t n, const uint64_t x[4], uint64_t out[4]) { B200_API_BODY(poly_eval_host(v, n, x, out)) }
int b200_poly_eval_batch(const uint64_t* polys, size_t m, size_t n, const uint64_t x[4], uint64_t* out) { B200_API_BODY(poly_eval_batch_host(polys, m, n, x, out)) }
int b200_zero_poly(size_t n, uint64_t* out) { B200_API_BODY(zero_poly_host(n, out)) }
int b200_r1cs_load(size_t n, size_t m, const uint32_t* a_rowptr, const uint32_t* a_col, const uint64_t* a_val,
                   const uint32_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val, const uint32_t* c_rowptr,
                   const uint32_t* c_col, const uint64_t* c_val, b200_r1cs_t* out) {
  const uint32_t* const rp[3] = {a_rowptr, b_rowptr, c_rowptr};
  const uint32_t* const cl[3] = {a_col, b_col, c_col};
  const uint64_t* const vl[3] = {a_val, b_val, c_val};
  B200_API_BODY(r1cs_load(n, m, rp, cl, vl, out))
}
int b200_r1cs_free(b200_r1cs_t h) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_r1cs.erase(h)) return fail(B200_EINVAL, "r1cs_free: bad handle");
  return B200_OK;
}
int b200_qap_px(b200_r1cs_t h, const uint64_t* w, size_t nw, uint64_t* ax, uint64_t* bx, uint64_t* cx, uint64_t* px) {
  B200_API_BODY(qap_px_host(h, w, nw, ax, bx, cx, px))
}
int b200_qap_eval_at(b200_r1cs_t h, const uint64_t tau[4], size_t nz, uint64_t* at, uint64_t* bt, uint64_t* ct, uint64_t zt[4]) {
  B200_API_BODY(qap_eval_at_host(h, tau, nz, at, bt, ct, zt))
}
int b200_interpolate(const uint64_t* values, size_t n, uint64_t* coeffs) { B200_API_BODY(interpolate_host(values, n, coeffs)) }
int b200_groth16_setup(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[20], uint64_t* at, uint64_t* b1, uint64_t* b2,
                       uint64_t* bacdelta, uint64_t* ptd, uint64_t* z, uint64_t alpha1[12], uint64_t beta1[12],
                       uint64_t delta1[12], uint64_t beta2[24], uint64_t gamma2[24], uint64_t delta2[24], uint64_t* ic) {
  B200_API_BODY(groth16_setup_host(r1cs, npublic, toxic, at, b1, b2, bacdelta, ptd, z, alpha1, beta1, delta1, beta2, gamma2,
                                   delta2, ic))
}
int b200_pinocchio_setup(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[32], uint64_t* a, uint64_t* ap, uint64_t* b2,
                         uint64_t* bp, uint64_t* c, uint64_t* cp, uint64_t* kp, uint64_t* g1t, uint64_t* z, uint64_t vk_g1[24],
                         uint64_t vk_g2[120]) {
  B200_API_BODY(pinocchio_setup_host(r1cs, npublic, toxic, a, ap, b2, bp, c, cp, kp, g1t, z, vk_g1, vk_g2))
}
int b200_groth16_setup_pk(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[20], int window_bits, int rank, int world,
                          b200_pk_t* out, uint64_t alpha1[12], uint64_t beta2[24], uint64_t gamma2[24], uint64_t delta2[24],
                          uint64_t* ic) {
  B200_API_BODY(groth16_setup_pk(r1cs, npublic, toxic, window_bits, rank, world, out, alpha1, beta2, gamma2, delta2, ic))
}
int b200_pinocchio_setup_pk(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[32], int window_bits, int rank, int world,
                            b200_pk_t* out, uint64_t vk_g1[24], uint64_t vk_g2[120], uint64_t* ic) {
  B200_API_BODY(pinocchio_setup_pk(r1cs, npublic, toxic, window_bits, rank, world, out, vk_g1, vk_g2, ic))
}
int b200_groth16_prove_witness(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, const uint64_t r[4],
                               const uint64_t s[4], uint64_t pi_a[12], uint64_t pi_b[24], uint64_t pi_c[12]) {
  std::unique_lock<std::mutex> lk(g_mu);
  NEED_INIT();
  return drain_on_error(groth16_prove_witness(pk, r1cs, w, nw, r, s, pi_a, pi_b, pi_c, &lk));
}
int b200_groth16_prove_witness_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, const uint64_t r[4],
                                      const uint64_t s[4], void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  ProvingKey* p = find_pk(pk, 1);
  R1cs* r1 = find_r1cs(r1cs);
  if (!p || !r1 || !d_w || !r || !s || !d_out) return fail(B200_EINVAL, "groth16_prove_witness_device: bad arguments");
  if (nw != p->m || nw != r1->m)
    return fail(B200_EINVAL, "groth16_prove_witness_device: witness length %zu, NVars %zu, R1CS columns %zu", nw, p->m, r1->m);
  return drain_on_error(groth16_witness_enqueue(p, r1, (const Fr*)d_w, r, s, (Fq*)d_out,
                                                stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_groth16_prove_witness_batch(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, size_t k, const uint64_t* r,
                                     const uint64_t* s, uint64_t* pi_a, uint64_t* pi_b, uint64_t* pi_c) {
  std::unique_lock<std::mutex> lk(g_mu);
  NEED_INIT();
  return drain_on_error(groth16_prove_witness_batch(pk, r1cs, w, nw, k, r, s, pi_a, pi_b, pi_c, &lk));
}
int b200_groth16_prove_witness_batch_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                            const uint64_t* r, const uint64_t* s, void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  const char* what = "groth16_prove_witness_batch_device";
  ProvingKey* p = find_pk(pk, 1);
  R1cs* r1 = find_r1cs(r1cs);
  if (!p || !r1 || !d_w || !r || !s || !d_out) return fail(B200_EINVAL, "%s: bad arguments", what);
  int rc = groth16_batch_check(p, r1, nw, k, r, s, what);
  if (rc) return rc;
  if ((rc = groth16_batch_comm_check(p, what))) return rc;
  return drain_on_error(groth16_batch_enqueue(p, r1, (const Fr*)d_w, k, r, s, (Fq*)d_out, false,
                                              stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_groth16_prove_witness_batch_partial_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                                    const uint64_t* r, const uint64_t* s, void* d_parts, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  const char* what = "groth16_prove_witness_batch_partial_device";
  ProvingKey* p = find_pk(pk, 1);
  R1cs* r1 = find_r1cs(r1cs);
  if (!p || !r1 || !d_w || !r || !s || !d_parts) return fail(B200_EINVAL, "%s: bad arguments", what);
  int rc = groth16_batch_check(p, r1, nw, k, r, s, what);
  if (rc) return rc;
  return drain_on_error(groth16_batch_enqueue(p, r1, (const Fr*)d_w, k, r, s, (Fq*)d_parts, true,
                                              stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_groth16_finalize_batch_device(b200_pk_t pk, const void* d_parts, int world, size_t k, void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  if (!find_pk(pk, 1) || !d_parts || !d_out || world < 1 || k == 0 || k > 0xffffffffull)
    return fail(B200_EINVAL, "groth16_finalize_batch_device: bad arguments");
  cudaStream_t st = stream ? (cudaStream_t)stream : g_ctx[0].main;
  k_groth16_finalize_batch<<<groth16_finalize_blocks((uint32_t)k), kG16FinalizeBlock, 0, st>>>((const uint8_t*)d_parts, world,
                                                                                                 (uint32_t)k, (Fq*)d_out);
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}
int b200_pinocchio_prove_device(b200_pk_t pk, const void* d_w, size_t nw, const void* d_px, size_t npx, void* d_out,
                                void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  const char* what = "pinocchio_prove_device";
  ProvingKey* p = find_pk(pk, 2);
  if (!p || !d_w || !d_px || !d_out) return fail(B200_EINVAL, "%s: bad arguments", what);
  if (nw != p->m) return fail(B200_EINVAL, "%s: witness length %zu != NVars %zu", what, nw, p->m);
  int rc = pinocchio_check_px(p, npx, what);
  if (rc) return rc;
  return drain_on_error(pinocchio_enqueue(p, (const Fr*)d_w, (const Fr*)d_px, npx, 0, nullptr, (Fq*)d_out,
                                          p->world > 1 && !pinocchio_gathers(p),
                                          stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_pinocchio_prove_witness(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, uint64_t* out_g1,
                                 uint64_t pi_b[24]) {
  std::unique_lock<std::mutex> lk(g_mu);
  NEED_INIT();
  return drain_on_error(pinocchio_prove_witness(pk, r1cs, w, nw, out_g1, pi_b, &lk));
}
int b200_pinocchio_prove_witness_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  const char* what = "pinocchio_prove_witness_device";
  ProvingKey* p = find_pk(pk, 2);
  R1cs* r1 = find_r1cs(r1cs);
  if (!p || !r1 || !d_w || !d_out) return fail(B200_EINVAL, "%s: bad arguments", what);
  int rc = pinocchio_witness_check(p, r1, nw, what);
  if (rc) return rc;
  return drain_on_error(pinocchio_witness_enqueue(p, r1, (const Fr*)d_w, (Fq*)d_out, p->world > 1 && !pinocchio_gathers(p),
                                                  stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_pinocchio_prove_witness_batch(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, size_t k,
                                       uint64_t* out_g1, uint64_t* pi_b) {
  std::unique_lock<std::mutex> lk(g_mu);
  NEED_INIT();
  return drain_on_error(pinocchio_prove_witness_batch(pk, r1cs, w, nw, k, out_g1, pi_b, &lk));
}
int b200_pinocchio_prove_witness_batch_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                              void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  const char* what = "pinocchio_prove_witness_batch_device";
  ProvingKey* p = find_pk(pk, 2);
  R1cs* r1 = find_r1cs(r1cs);
  if (!p || !r1 || !d_w || !d_out) return fail(B200_EINVAL, "%s: bad arguments", what);
  int rc = pinocchio_batch_check(p, r1, nw, k, what);
  if (rc) return rc;
  if ((rc = pinocchio_batch_comm_check(p, what))) return rc;
  return drain_on_error(pinocchio_batch_enqueue(p, r1, (const Fr*)d_w, k, (Fq*)d_out, false,
                                                stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_pinocchio_prove_witness_batch_record_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                                     void* d_records, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  const char* what = "pinocchio_prove_witness_batch_record_device";
  ProvingKey* p = find_pk(pk, 2);
  R1cs* r1 = find_r1cs(r1cs);
  if (!p || !r1 || !d_w || !d_records) return fail(B200_EINVAL, "%s: bad arguments", what);
  int rc = pinocchio_batch_check(p, r1, nw, k, what);
  if (rc) return rc;
  return drain_on_error(pinocchio_batch_enqueue(p, r1, (const Fr*)d_w, k, (Fq*)d_records, true,
                                                stream ? (cudaStream_t)stream : g_ctx[0].main, p->d_err.as<int>()));
}
int b200_pinocchio_finalize_records_batch_device(const void* d_records, int world, size_t k, void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  if (!d_records || !d_out || world < 1 || k == 0 || k >= (1ull << 28))
    return fail(B200_EINVAL, "pinocchio_finalize_records_batch_device: bad arguments");
  cudaStream_t st = stream ? (cudaStream_t)stream : g_ctx[0].main;
  k_pinocchio_gather_finalize_batch<<<pinocchio_finalize_blocks((uint32_t)k), kPinFinalizeBlock, 0, st>>>(
      (const uint8_t*)d_records, world, (uint32_t)k, (Fq*)d_out);
  g_launches += 1;
  CU(cudaGetLastError());
  return B200_OK;
}
int b200_fq12_mul_batch(const uint64_t* a, const uint64_t* b, size_t n, uint64_t* out) { B200_API_BODY(fq12_mul_batch_host(a, b, n, out)) }
int b200_pairing_batch(const uint64_t* g1_jac, const uint64_t* g2_jac, size_t n, uint64_t* out) { B200_API_BODY(pairing_batch_host(g1_jac, g2_jac, n, out)) }
int b200_groth16_verify(const uint64_t* ic, size_t n_ic, const uint64_t alpha1[12], const uint64_t beta2[24],
                        const uint64_t gamma2[24], const uint64_t delta2[24], const uint64_t pi_a[12],
                        const uint64_t pi_b[24], const uint64_t pi_c[12], const uint64_t* public_signals, size_t n_public,
                        int* ok) {
  B200_API_BODY(groth16_verify_host(ic, n_ic, alpha1, beta2, gamma2, delta2, pi_a, pi_b, pi_c, public_signals, n_public, ok))
}
int b200_groth16_verify_batch(const uint64_t* ic, size_t n_ic, const uint64_t alpha1[12], const uint64_t beta2[24],
                              const uint64_t gamma2[24], const uint64_t delta2[24], const uint64_t* pi_a, const uint64_t* pi_b,
                              const uint64_t* pi_c, const uint64_t* public_signals, size_t n_public, size_t k, const uint64_t* rho,
                              int* ok, uint32_t* status) {
  B200_API_BODY(groth16_verify_batch_host(ic, n_ic, alpha1, beta2, gamma2, delta2, pi_a, pi_b, pi_c, public_signals, n_public, k,
                                          rho, ok, status))
}
int b200_groth16_verify_batch_device(const uint64_t* ic, size_t n_ic, const uint64_t alpha1[12], const uint64_t beta2[24],
                                     const uint64_t gamma2[24], const uint64_t delta2[24], const void* d_proofs,
                                     const void* d_public, size_t n_public, size_t k, const uint64_t* rho, void* d_ok,
                                     void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return groth16_verify_batch_device(ic, n_ic, alpha1, beta2, gamma2, delta2, d_proofs, d_public, n_public, k, rho, d_ok,
                                     stream ? (cudaStream_t)stream : g_ctx[0].main);
}
int b200_pinocchio_verify_batch(const uint64_t* ic, size_t n_ic, const uint64_t vk_g1[24], const uint64_t vk_g2[120],
                                const uint64_t* out_g1, const uint64_t* pi_b, const uint64_t* public_signals, size_t n_public,
                                size_t k, const uint64_t* rho, int* ok, uint32_t* status) {
  B200_API_BODY(pinocchio_verify_batch_host(ic, n_ic, vk_g1, vk_g2, out_g1, pi_b, public_signals, n_public, k, rho, ok, status))
}
int b200_pinocchio_verify_batch_device(const uint64_t* ic, size_t n_ic, const uint64_t vk_g1[24], const uint64_t vk_g2[120],
                                       const void* d_proofs, const void* d_public, size_t n_public, size_t k, const uint64_t* rho,
                                       void* d_ok, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return pinocchio_verify_batch_device(ic, n_ic, vk_g1, vk_g2, d_proofs, d_public, n_public, k, rho, d_ok,
                                       stream ? (cudaStream_t)stream : g_ctx[0].main);
}
int b200_g1_add_batch(const uint64_t* p, const uint64_t* q, size_t n, uint64_t* out) { B200_API_BODY(group_op_host<Fq>(0, p, q, n, out)) }
int b200_g1_double_batch(const uint64_t* p, size_t n, uint64_t* out) { B200_API_BODY(group_op_host<Fq>(1, p, nullptr, n, out)) }
int b200_g1_neg_batch(const uint64_t* p, size_t n, uint64_t* out) { B200_API_BODY(group_op_host<Fq>(2, p, nullptr, n, out)) }
int b200_g1_affine_batch(const uint64_t* p, size_t n, uint64_t* out_xy) { B200_API_BODY(group_op_host<Fq>(3, p, nullptr, n, out_xy)) }
int b200_g2_add_batch(const uint64_t* p, const uint64_t* q, size_t n, uint64_t* out) { B200_API_BODY(group_op_host<Fq2>(0, p, q, n, out)) }
int b200_g2_double_batch(const uint64_t* p, size_t n, uint64_t* out) { B200_API_BODY(group_op_host<Fq2>(1, p, nullptr, n, out)) }
int b200_g2_neg_batch(const uint64_t* p, size_t n, uint64_t* out) { B200_API_BODY(group_op_host<Fq2>(2, p, nullptr, n, out)) }
int b200_g2_affine_batch(const uint64_t* p, size_t n, uint64_t* out_xy) { B200_API_BODY(group_op_host<Fq2>(3, p, nullptr, n, out_xy)) }

int b200_poly_mul(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return poly_mul_host(a, na, b, nb, out);
}
int b200_poly_div(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* q, uint64_t* rem) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return poly_div_host(a, na, b, nb, q, rem);
}


int b200_version(void) { return 200; }
int b200_config(int key, int value) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (key == B200_CFG_ACC_MODE && value >= 0 && value <= 2) {
    g_acc_mode = value;
    return B200_OK;
  }
  if (key >= 10 && key <= 13 && value > 0) {   // shard-partition tuning (tools/shard_times.py sweeps them)
    (key == 10 ? g_w_ab : key == 11 ? g_w_g2 : key == 12 ? g_aff_min_g1 : g_aff_min_g2) = value;
    return B200_OK;
  }
  if (key == B200_CFG_PAIRING_KERNEL && value >= 0 && value <= 2) {
    g_pairing_kernel = value;
    return B200_OK;
  }
  if (key == B200_CFG_PK_CONTEXT && (value == 0 || value == 1)) {
    g_pk_ctx = value;
    return B200_OK;
  }
  if (key == B200_CFG_TMA_STAGING && value >= 0 && value <= 2) {
    g_tma_staging = value;
    return B200_OK;
  }
  if (key == B200_CFG_TABLE_WINDOWS && value >= 0) {
    g_table_windows = value;
    return B200_OK;
  }
  return fail(B200_EINVAL, "b200_config: unknown key %d or bad value %d", key, value);
}

const char* b200_last_error(void) { return g_err.c_str(); }

int b200_init(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  return init_locked(device);
}

int b200_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_init) return B200_OK;
  cudaSetDevice(g_device);
  comm_destroy_locked();
  g_bases.clear();
  g_pks.clear();
  g_r1cs.clear();
  g_domains.clear();
  if (g_d_err) cudaFree(g_d_err);
  g_d_err = nullptr;
  for (auto& c : g_ctx) {
    if (c.main) cudaStreamDestroy(c.main);
    for (auto sd : c.side) if (sd) cudaStreamDestroy(sd);
    c = ProveCtx{};   // also frees the polynomial workspace
  }
  g_init = false;
  return B200_OK;
}

int b200_g1_bases_load(const uint64_t* p, size_t n, int c, b200_bases_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return bases_load<Fq>(p, n, c, 1, out);
}
int b200_g2_bases_load(const uint64_t* p, size_t n, int c, b200_bases_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return bases_load<Fq2>(p, n, c, 2, out);
}
int b200_bases_free(b200_bases_t h) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_init) return fail(B200_EINVAL, "not initialised");
  cudaSetDevice(g_device);
  cudaStreamSynchronize(g_ctx[0].main);
  return g_bases.erase(h) ? B200_OK : fail(B200_EINVAL, "bases_free: bad handle");
}
int b200_bases_info(b200_bases_t h, size_t* n, int* group, int* window_bits, int* n_windows) {
  std::lock_guard<std::mutex> lk(g_mu);
  Bases* b = find_bases(h, 0);
  if (!b) return fail(B200_EINVAL, "bases_info: bad handle");
  if (n) *n = b->n;
  if (group) *group = b->group;
  if (window_bits) *window_bits = (int)b->sh.c;
  if (n_windows) *n_windows = (int)b->sh.nwin;
  return B200_OK;
}

int b200_bases_table_windows(b200_bases_t h, int* t) {
  std::lock_guard<std::mutex> lk(g_mu);
  Bases* b = find_bases(h, 0);
  if (!b || !t) return fail(B200_EINVAL, "bases_table_windows: bad handle");
  *t = (int)b->sh.rows;
  return B200_OK;
}
int b200_bases_device_bytes(b200_bases_t h, size_t* bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  Bases* b = find_bases(h, 0);
  if (!b || !bytes) return fail(B200_EINVAL, "bases_device_bytes: bad handle");
  *bytes = bases_device_bytes(*b);
  return B200_OK;
}

int b200_bases_acc_mode(b200_bases_t h, int* mode) {
  std::lock_guard<std::mutex> lk(g_mu);
  Bases* b = find_bases(h, 0);
  if (!b || !mode) return fail(B200_EINVAL, "bases_acc_mode: bad handle");
  *mode = b->affine_S ? 1 : 2;
  return B200_OK;
}
int b200_g1_msm(b200_bases_t h, const uint64_t* s, size_t n, uint64_t out[12]) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return msm_host<Fq>(h, 1, s, n, out);
}
int b200_g2_msm(b200_bases_t h, const uint64_t* s, size_t n, uint64_t out[24]) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return msm_host<Fq2>(h, 2, s, n, out);
}

int b200_msm_device(b200_bases_t h, const void* d_scalars, size_t n, int mont, void* d_out, void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  Bases* b = find_bases(h, 0);
  if (!b || !d_out || (!d_scalars && n)) return fail(B200_EINVAL, "msm_device: bad arguments");
  cudaStream_t st = stream ? (cudaStream_t)stream : g_ctx[0].main;
  int* err = b->d_err.as<int>();
  if (b->group == 1) return msm_enqueue<Fq>(b, (const Fr*)d_scalars, n, mont, (XYZZ<Fq>*)d_out, err, st);
  return msm_enqueue<Fq2>(b, (const Fr*)d_scalars, n, mont, (XYZZ<Fq2>*)d_out, err, st);
}
int b200_msm_device_batch(b200_bases_t h, const void* d_scalars, size_t n, size_t k, size_t stride, int mont, void* d_out,
                          void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  Bases* b = find_bases(h, 0);
  if (!b || !d_out || (!d_scalars && n)) return fail(B200_EINVAL, "msm_device_batch: bad arguments");
  cudaStream_t st = stream ? (cudaStream_t)stream : g_ctx[0].main;
  if (k == 0) return fail(B200_EINVAL, "msm_device_batch: k = 0");
  if (n > b->n) return fail(B200_EINVAL, "msm_device_batch: n=%zu exceeds base set size %zu", n, b->n);
  if (stride > 0xffffffffull) return fail(B200_EINVAL, "msm_device_batch: stride %zu exceeds 2^32 - 1", stride);
  if (!batch_fits(b, k, n ? n : 1))
    return fail(B200_EINVAL, "msm_device_batch: k * nwin * n = %zu * %u * %zu sort entries (or the buckets) exceed 2^31", k,
                b->sh.nwin, n);
  int* err = b->d_err.as<int>();
  if (b->group == 1) CU(msm_batch_enqueue<Fq>(msm_env(), b, (const Fr*)d_scalars, n, k, stride, mont, (XYZZ<Fq>*)d_out, err, st));
  else CU(msm_batch_enqueue<Fq2>(msm_env(), b, (const Fr*)d_scalars, n, k, stride, mont, (XYZZ<Fq2>*)d_out, err, st));
  return B200_OK;
}

int b200_g1_sum_partials(const void* d, size_t count, uint64_t out[12], void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return sum_partials<Fq>(d, count, out, stream ? (cudaStream_t)stream : g_ctx[0].main);
}
int b200_g2_sum_partials(const void* d, size_t count, uint64_t out[24], void* stream) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return sum_partials<Fq2>(d, count, out, stream ? (cudaStream_t)stream : g_ctx[0].main);
}

int b200_g1_mul_batch(const uint64_t* p, const uint64_t* s, size_t n, uint64_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return mul_batch<Fq>(p, 0, s, n, out);
}
int b200_g2_mul_batch(const uint64_t* p, const uint64_t* s, size_t n, uint64_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return mul_batch<Fq2>(p, 0, s, n, out);
}
int b200_g1_mul_batch_bcast(const uint64_t* p, const uint64_t* s, size_t n, uint64_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return mul_batch<Fq>(p, 1, s, n, out);
}
int b200_g2_mul_batch_bcast(const uint64_t* p, const uint64_t* s, size_t n, uint64_t* out) {
  std::lock_guard<std::mutex> lk(g_mu);
  NEED_INIT();
  return mul_batch<Fq2>(p, 1, s, n, out);
}

}  // extern "C"
