/* libb200snark — C ABI of the H100-native Groth16 / Pinocchio prove path.
 *
 * The reference (arnaucube/go-snark-study) has no FFI: its boundary is the
 * exported Go package API.  Each entry point below names the Go function(s)
 * whose body a cgo shim replaces (file:line in the upstream tree); the shim
 * itself is shown in INTEGRATION.md.  Conventions:
 *
 *   - field elements / scalars: 4 little-endian uint64 limbs, STANDARD form
 *     (not Montgomery), canonical (< modulus) — i.e. big.Int.Bits() on amd64,
 *     zero-padded.  Scalars must be reduced mod r (the shim sends |e| mod r:
 *     the reference's MulScalar consumes |e|, fields/fq.go:138-140, SURVEY H7).
 *   - G1 point  = [3]*big.Int  Jacobian (X, Y, Z)            -> 12 uint64
 *     G2 point  = [3][2]*big.Int Jacobian (X.c0, X.c1, Y.., Z..) -> 24 uint64
 *     Z == 0 (e.g. the (0,0,0) entries of Pk.BACDelta, groth16.go:177-180) is
 *     the point at infinity.  Outputs are normalised: (x, y, 1), infinity as
 *     all-zero — valid inputs to every reference function (SURVEY H1).
 *   - every function returns 0 (B200_OK) or a negative B200_E* code; no
 *     exceptions or panics cross the ABI; b200_last_error() gives the text.
 *   - all pointers are HOST pointers unless the name ends in _device.
 *   - thread-safety: calls are serialised per process by an internal mutex
 *     (cgo may migrate goroutines between OS threads).
 *   - there is NO CPU fallback: without a CUDA device every call fails with
 *     B200_ENODEVICE.
 */
#ifndef B200SNARK_H
#define B200SNARK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ENODEVICE (-1) /* no CUDA device / init failed                         */
#define B200_ECUDA (-2)     /* CUDA runtime error (see b200_last_error)              */
#define B200_EINVAL (-3)    /* bad argument (null pointer, size mismatch, handle)    */
#define B200_ERANGE (-4)    /* a field element >= modulus or a scalar >= r           */
#define B200_EDIVZERO (-5)  /* polynomial division by a zero leading coefficient     */
#define B200_ENOMEM (-6)
#define B200_ECOMM (-7)     /* NCCL: library not found, or a collective failed       */

typedef uint64_t b200_bases_t; /* device-resident, window-precomputed base-point set */
typedef uint64_t b200_pk_t;    /* device-resident proving key                        */
typedef uint64_t b200_r1cs_t;  /* device-resident sparse R1CS (CSR + CSC)            */

/* ---- context ------------------------------------------------------------ */
int b200_init(int device);        /* idempotent; selects the CUDA device of this process */
int b200_shutdown(void);
const char* b200_last_error(void);
int b200_version(void);
/* Process-wide options for objects created AFTERWARDS.  B200_CFG_ACC_MODE: bucket-accumulation kernel of base sets and
 * proving keys — 0 auto (batched affine where bucket population and shard size amortise its rounds, else XYZZ mixed
 * adds), 1 batched affine, 2 XYZZ.  Same results either way; the parity tests run every MSM size under both.          */
#define B200_CFG_ACC_MODE 1
/* B200_CFG_TMA_STAGING: the batched-affine backward pass with its operands staged into shared memory — TMA bulk
 * copies (cp.async.bulk + per-warp mbarrier) in the contiguous rounds, cp.async gathers in round 1.  0 (default) the
 * register-load kernel (the kernel is bound by the multiply pipe, not by the fetch); 1 staged in every round, 2 staged in rounds >= 2 only.  Same results.          */
#define B200_CFG_TMA_STAGING 2
/* B200_CFG_PK_CONTEXT: prove context (0 or 1) of proving keys loaded AFTERWARDS.  The two contexts own separate main and
 * side streams, polynomial workspaces and NCCL communicators, so a device-resident proof on a context-1 key
 * (b200_groth16_prove_device on the caller's second stream) may be in flight beside one on a context-0 key: a prover that
 * keeps two proofs in flight hides the latency-bound sort / bucket-tail / blinding-product chains of one behind the
 * accumulation of the other (bench.py `proofs_in_flight`; the keys are independent objects, each with its own tables,
 * scratch and error words).  Host-pointer proofs run on their key's context and report only their own input errors, also
 * when two host threads prove at once.  Other calls run on context 0 and share its scratch with its proofs: each use
 * of a context's scratch waits for the previous one on the device, in the order the calls were made, so a library call
 * made while a context-0 proof is in flight on another stream waits on the device for that proof's quotient.          */
#define B200_CFG_PK_CONTEXT 4
/* B200_CFG_PAIRING_KERNEL: b200_pairing_batch with one THREAD per pairing (1: the step-by-step restatement of
 * bn128.go:179-421, a long chain of dependent multiplications per pairing) or one WARP per pairing (2: F_q^12 in shared
 * memory, 27 F_q^2 products of a tower multiplication on 27 lanes; csrc/pairing_warp.cuh); 0 = auto: a warp per
 * pairing up to 2048 pairings per call (latency), a thread per pairing above (throughput).
 * Bit-identical F_q^12 values.  b200_groth16_verify always runs four warps.  The same rule picks the Miller-loop
 * kernel of b200_groth16_verify_batch(_device) over its k_reg + 3 pairs and of b200_pinocchio_verify_batch(_device)
 * over its k_reg + 6.                                                                                                  */
#define B200_CFG_PAIRING_KERNEL 5
/* Partition tuning of SHARDED proving keys loaded afterwards (defaults = the measured best for one proof at a time):
 * cost weight x100 of an A / B1 term (10) and of a G2 term (11) in C||PTD terms, and the
 * smallest per-rank set that still takes the batched-affine tree, in G1 (12) / G2 (13) terms — below it the set runs
 * the XYZZ kernel, whose single launch has the shorter latency chain.  With two proofs in flight (B200_CFG_PK_CONTEXT)
 * that latency is hidden and the affine tree's 6 multiplications per add win at every shard size: set 12 and 13 to 1. */
#define B200_CFG_SHARD_W_AB 10
#define B200_CFG_SHARD_W_G2 11
#define B200_CFG_SHARD_AFFINE_MIN_G1 12
#define B200_CFG_SHARD_AFFINE_MIN_G2 13
/* B200_CFG_TABLE_WINDOWS: t, the number of precomputed window rows 2^(c*j) * P (j < t) that base sets and proving keys
 * loaded AFTERWARDS store (b200_g1/g2_bases_load, b200_groth16_pk_load(_shard), b200_pinocchio_pk_load(_shard)).
 * 0 (default) or any t >= the set's nwin = ceil(255/c) keeps every window: one bucket set, no doublings.  With t < nwin
 * the table holds t*n points instead of nwin*n; the nwin windows fall into ceil(nwin/t) groups with their own buckets,
 * recombined by doublings in the bucket tail.  Same results, less memory, a slower MSM: the setting for circuits whose
 * keys do not fit on the GPU with full tables (INTEGRATION.md "Large circuits").  B200_CFG_ACC_MODE 0 (auto) gives a
 * set with t < nwin the XYZZ kernel, since the batched-affine scratch alone is about the size of a full table; mode 1
 * still forces batched affine (with its scratch) where the mean population of the G*2^(c-1) buckets allows it.
 * Negative: B200_EINVAL.  The trusted setup's own fixed-base table is not affected.                                  */
#define B200_CFG_TABLE_WINDOWS 14
int b200_config(int key, int value);

/* ---- base-point sets (the CRS arrays of groth16.Pk / snark.Pk) ---------- */
/* Upload n Jacobian points, normalise to affine Montgomery form on the device
 * and precompute 2^(c*w) * P for every window w (the CRS is static, so all
 * windows of one MSM share a single bucket set; see DESIGN.md §3).
 * window_bits = 0 picks c from n.  Replaces nothing in the reference (its Pk
 * is consumed directly); this is the "load proving key once" step of H9.     */
int b200_g1_bases_load(const uint64_t* points_jac, size_t n, int window_bits, b200_bases_t* out);
int b200_g2_bases_load(const uint64_t* points_jac, size_t n, int window_bits, b200_bases_t* out);
int b200_bases_free(b200_bases_t h);
int b200_bases_info(b200_bases_t h, size_t* n, int* group, int* window_bits, int* n_windows);
/* which bucket-accumulation kernel the set was built for: 1 batched affine, 2 XYZZ (see b200_config) */
int b200_bases_acc_mode(b200_bases_t h, int* mode);
/* t: the window rows the set's table stores (B200_CFG_TABLE_WINDOWS at load; nwin for full tables).  b200_bases_info's
 * n_windows stays ceil(255/c). */
int b200_bases_table_windows(b200_bases_t h, int* t);
/* device memory the set holds: window table, sort and bucket scratch, batched-affine scratch, result buffers */
int b200_bases_device_bytes(b200_bases_t h, size_t* bytes);

/* ---- multi-scalar multiplication ---------------------------------------- */
/* out = sum_i scalars[i] * P_i over the first n bases of the set.
 * Replaces the hot loops  acc = G1.Add(acc, G1.MulScalar(P_i, w_i))  of
 * groth16/groth16.go:243-250,269-271 and snark.go:265-286 (G1: bn128/g1.go:32-155;
 * G2: bn128/g2.go:32-181).                                                    */
int b200_g1_msm(b200_bases_t h, const uint64_t* scalars, size_t n, uint64_t out_jac[12]);
int b200_g2_msm(b200_bases_t h, const uint64_t* scalars, size_t n, uint64_t out_jac[24]);

/* Same, scalars already resident in device memory (n * 32 bytes, standard form,
 * or Montgomery form when scalars_mont != 0), result left on the device as an
 * XYZZ record (4 field elements, Montgomery form; 128 B for G1, 256 B for G2)
 * on `stream` (a cudaStream_t, may be NULL).  No host synchronisation.  Used by
 * the prove pipeline, by bench.py's device-resident timing and by the
 * multi-GPU path (each rank's partial record is what the NCCL gather moves).
 * Record layout: X | Y | ZZ | ZZZ, each F_q element 4 little-endian uint64 limbs
 * (F_q^2: c0 then c1), Montgomery form (value * 2^256 mod q); x = X/ZZ, y = Y/ZZZ,
 * ZZ^3 = ZZZ^2; ZZ = 0 is the point at infinity (n = 0 gives it).  n > the set's
 * size returns B200_EINVAL.
 * Scalars are not range-checked here: the call does not wait for the device,
 * so it cannot return B200_ERANGE.  With scalars_mont = 0 a scalar >= r is read
 * as 0, and neither this call nor any later one reports it.  With
 * scalars_mont != 0 any 256-bit value v is accepted and read as v * 2^-256 mod r. */
int b200_msm_device(b200_bases_t h, const void* d_scalars, size_t n, int scalars_mont,
                    void* d_out_xyzz, void* stream);
/* k MSMs over the same first n bases in one set of launches: record p (k XYZZ
 * records, 128 B / 256 B apart in d_out_xyzz) is sum_i d_scalars[p*stride + i] * P_i.
 * The contract is that of b200_msm_device (device memory, no host synchronisation,
 * scalars_mont, no range report); k = 1 gives b200_msm_device's record.  Any stride
 * (0 included) is accepted; the scalar buffer holds (k-1)*stride + n scalars.
 * One digit recode, counting sort, bucket accumulation and bucket tail serve all k
 * vectors, so a batch of small MSMs costs about one MSM of k*n terms.  The launches
 * are those of one MSM, plus one when k*G*2^(c-1) bucket counters exceed 64 Ki
 * (G = window groups: 1 for full tables; the counter scan then runs on several
 * blocks) and one or two per further 65535 (vector, group) rows of the tail.
 * Scratch: the first batch on a set allocates sort, bucket and (batched-affine
 * sets) node buffers for k vectors of n terms, about k times those of one n-term
 * MSM; a later batch with more vectors or terms grows them (the host first waits
 * for the set's previous batch) and they are never shrunk.
 * b200_bases_device_bytes / b200_pk_device_bytes count them.  Single MSMs keep
 * their own buffers.
 * Each base set has ONE scratch for its single MSMs (b200_msm_device,
 * b200_g*_msm) and one for its batches: calls on the same set must be ordered,
 * e.g. issued on one stream; sets are independent of each other.
 * B200_EINVAL: k = 0, n > the set's size, stride >= 2^32, or k*ceil(255/c)*n sort
 * entries (or k times the set's buckets) reaching 2^31; nothing is allocated then. */
int b200_msm_device_batch(b200_bases_t h, const void* d_scalars, size_t n, size_t k, size_t stride,
                          int scalars_mont, void* d_out_xyzz, void* stream);
/* Sum `count` XYZZ partial records (device memory, e.g. the gathered per-rank
 * partials) and normalise: out_jac = (x, y, 1) in standard form on the host,
 * infinity as all-zero.  1 <= count <= 2^20, else B200_EINVAL.  Synchronises `stream`. */
int b200_g1_sum_partials(const void* d_xyzz, size_t count, uint64_t out_jac[12], void* stream);
int b200_g2_sum_partials(const void* d_xyzz, size_t count, uint64_t out_jac[24], void* stream);

/* ---- batch scalar multiplication, reference operation order -------------- */
/* out[i] = MulScalar(points[i], scalars[i]) with the reference's MSB-first
 * double-and-add and its add-2007-bl / dbl-2009-l formulas, one thread per
 * term: X,Y,Z-exact drop-in for bn128.G1.MulScalar (bn128/g1.go:140-155) and
 * bn128.G2.MulScalar (bn128/g2.go:142-181).  Also mints CRSs on the GPU
 * (groth16/groth16.go:139-219: every Pk/Vk entry is G.MulScalar(g, k)).       */
int b200_g1_mul_batch(const uint64_t* points_jac, const uint64_t* scalars, size_t n, uint64_t* out_jac);
int b200_g2_mul_batch(const uint64_t* points_jac, const uint64_t* scalars, size_t n, uint64_t* out_jac);
/* points_jac may hold a single point broadcast to all scalars when n_points == 1 */
int b200_g1_mul_batch_bcast(const uint64_t* point_jac, const uint64_t* scalars, size_t n, uint64_t* out_jac);
int b200_g2_mul_batch_bcast(const uint64_t* point_jac, const uint64_t* scalars, size_t n, uint64_t* out_jac);

/* ---- proving keys and the prove path -------------------------------------- */
/* Upload a Groth16 proving key (groth16.Pk, groth16/groth16.go:15-32) once:
 *   at        = Pk.G1.At[0..m)            b1 = Pk.G1.BACGamma[0..m)   (G1, 12 u64 each)
 *   b2        = Pk.G2.BACGamma[0..m)      (G2, 24 u64 each)
 *   bacdelta  = Pk.BACDelta[0..m)         (entries 0..npublic are ignored, as in groth16.go:248)
 *   ptd       = Pk.PowersTauDelta[0..n_ptd)
 *   z         = Pk.Z[0..nz) coefficients  alpha1/beta1/delta1 = Pk.G1.{Alpha,Beta,Delta}
 *   beta2/delta2 = Pk.G2.{Beta,Delta}     npublic = circuit.NPublic, m = circuit.NVars
 * The blinding points are appended to the MSM base sets so that
 * A = sum w_i At_i + alpha + r*delta etc. are single MSMs (DESIGN.md §4).          */
int b200_groth16_pk_load(const uint64_t* at, const uint64_t* b1, const uint64_t* b2, const uint64_t* bacdelta,
                         size_t m, const uint64_t* ptd, size_t n_ptd, const uint64_t* z, size_t nz,
                         const uint64_t alpha1[12], const uint64_t beta1[12], const uint64_t delta1[12],
                         const uint64_t beta2[24], const uint64_t delta2[24], size_t npublic, int window_bits,
                         b200_pk_t* out);
/* groth16.GenerateProofs (groth16/groth16.go:225-278) with the randomness r, s
 * supplied by the caller (the Go shim draws them with Fq.Rand, fields/fq.go:116-132,
 * exactly as the reference does at groth16.go:231-238).  w: nw = NVars witness
 * scalars (|w_i| mod r); px: npx coefficients.  Outputs are Jacobian points (Z != 1
 * in general, like the reference's own), standard form.  Like DivisorPolynomial
 * (r1csqap.go:213-216: quotient kept, remainder dropped) the proof depends only on the
 * top npx - len(Z) + 1 coefficients of px; only those are read from the host buffer. */
int b200_groth16_prove(b200_pk_t pk, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx,
                       const uint64_t r[4], const uint64_t s[4], uint64_t pi_a[12], uint64_t pi_b[24],
                       uint64_t pi_c[12]);
/* Same with the witness and px already resident in DEVICE memory (standard form)
 * and the 48-u64 result (PiA | PiC | PiB) left in device memory on `stream`; no
 * host synchronisation.  This is the region bench.py times as `value`.
 * As in b200_msm_device, a witness entry or a px coefficient >= r is read as 0,
 * and neither this call nor any later one reports it (nor a proof on another
 * key).  r and s are host values and are checked (B200_ERANGE).                   */
int b200_groth16_prove_device(b200_pk_t pk, const void* d_w, size_t nw, const void* d_px, size_t npx,
                              const uint64_t r[4], const uint64_t s[4], void* d_out, void* stream);
/* Multi-GPU (one process per GPU): rank `rank` of `world` keeps the contiguous
 * index slice [m*rank/world, m*(rank+1)/world) of every CRS array (and the same
 * fraction of PowersTauDelta); the blinding points ride on rank 0.  With such a key
 * b200_groth16_prove_device leaves a 1024-byte PARTIAL record (XYZZ sums A | B1 |
 * B2 | CH) in d_out instead of a proof WHEN NO COMMUNICATOR IS ACTIVE (b200_comm_init):
 * the caller then all-gathers the records of all ranks itself and calls
 * b200_groth16_finalize_device, which adds them and applies groth16.go:272-275 (this is
 * how the one-GPU tests emulate N ranks).  With a communicator the gather + finalize run
 * inside the call and d_out receives the proof.  No EC-point reduction exists in NCCL,
 * hence gather-then-add (SURVEY §5).                                               */
int b200_groth16_pk_load_shard(const uint64_t* at, const uint64_t* b1, const uint64_t* b2, const uint64_t* bacdelta,
                               size_t m, const uint64_t* ptd, size_t n_ptd, const uint64_t* z, size_t nz,
                               const uint64_t alpha1[12], const uint64_t beta1[12], const uint64_t delta1[12],
                               const uint64_t beta2[24], const uint64_t delta2[24], size_t npublic, int window_bits,
                               int rank, int world, b200_pk_t* out);
/* ---- multi-GPU inside the library (one process per GPU) -------------------------------------------------
 * b200_comm_unique_id (on one rank) mints an NCCL id; the caller distributes the 128 bytes by whatever means it has
 * (a file, a socket, MPI, torch.distributed) and every rank calls b200_comm_init(id, rank, world) after b200_init.
 * With a communicator, b200_groth16_prove / b200_groth16_prove_device on a key loaded with
 * b200_groth16_pk_load_shard(.., rank, world) return the FINAL proof on every rank: each rank computes its partial
 * sums, the 1 KB records are all-gathered over NVLink (ncclAllGather on the library's stream) and added.  All ranks
 * must make the same call with the same witness, px, r and s (SPMD), as N copies of a Go process calling
 * groth16.GenerateProofs (groth16/groth16.go:225) would.  libnccl.so.2 is dlopen'ed; absent -> B200_ECOMM.           */
int b200_comm_unique_id(uint8_t out[128]);
int b200_comm_init(const uint8_t id[128], int rank, int world);
int b200_comm_destroy(void);
/* What a sharded key reads: out = { A lo, hi, B1 lo, hi, B2 lo, hi (witness index ranges), C-part witness
 * range lo, hi, needs_px (0/1), rank, world, NVars }.  A caller that stages inputs per proof only has to upload
 * those witness ranges, and px only when needs_px is set.                                                        */
int b200_groth16_shard_info(b200_pk_t pk, uint64_t out[12]);
int b200_groth16_finalize_device(b200_pk_t pk, const void* d_parts, int nparts, const uint64_t r[4],
                                 const uint64_t s[4], void* d_out, void* stream);
/* Pinocchio proving key (snark.Pk, snark.go:16-26): A, Ap, Bp, C, Cp, Kp in G1 and
 * B in G2, each m points; G1T n_g1t points; Z.                                     */
int b200_pinocchio_pk_load(const uint64_t* a, const uint64_t* ap, const uint64_t* b2, const uint64_t* bp,
                           const uint64_t* c, const uint64_t* cp, const uint64_t* kp, size_t m,
                           const uint64_t* g1t, size_t n_g1t, const uint64_t* z, size_t nz, size_t npublic,
                           int window_bits, b200_pk_t* out);
/* snark.GenerateProofs (snark.go:254-289).  out_g1 = 7 Jacobian G1 points in the
 * order PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp (84 u64); pi_b = PiB (G2).           */
int b200_pinocchio_prove(b200_pk_t pk, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx,
                         uint64_t* out_g1, uint64_t pi_b[24]);
/* Multi-GPU Pinocchio: the eight MSMs of snark.GenerateProofs are independent, so rank `rank` of `world` keeps WHOLE MSMs
 * (dealt greedily by cost, identically on every rank; no MSM is split).  With a communicator (b200_comm_init)
 * b200_pinocchio_prove on such a key computes the rank's MSMs, all-gathers the 2 KB result records and returns the whole
 * proof on every rank.  Without one, b200_pinocchio_prove_record_device leaves the rank's record (8 XYZZ slots, 256 B
 * each, device memory) to the caller and b200_pinocchio_finalize_records sums `world` gathered records — how the
 * one-GPU tests emulate N ranks.                                                                                      */
int b200_pinocchio_pk_load_shard(const uint64_t* a, const uint64_t* ap, const uint64_t* b2, const uint64_t* bp,
                                 const uint64_t* c, const uint64_t* cp, const uint64_t* kp, size_t m,
                                 const uint64_t* g1t, size_t n_g1t, const uint64_t* z, size_t nz, size_t npublic,
                                 int window_bits, int rank, int world, b200_pk_t* out);
int b200_pinocchio_prove_record_device(b200_pk_t pk, const uint64_t* w, size_t nw, const uint64_t* px, size_t npx,
                                       void* d_record);
int b200_pinocchio_finalize_records(const void* d_records, int world, uint64_t* out_g1, uint64_t pi_b[24]);
int b200_pk_free(b200_pk_t pk);
/* device memory the key holds: its base sets (b200_bases_device_bytes), the divisor Z and its inverse-series cache, the
 * scalar, quotient, staging and proof buffers (buffers sized on a key's first proof are counted once allocated) */
int b200_pk_device_bytes(b200_pk_t pk, size_t* bytes);

/* ---- instrumentation (bench.py) -------------------------------------------- */
/* b200_profile(flags): bit 0 brackets every bucket-accumulation phase (the dominant
 * kernels) with CUDA events on its stream; bit 1 additionally issues all MSMs of a
 * proof on the caller's stream instead of overlapping them on side streams, so that
 * those event times are exclusive (measurement mode, slower).  b200_profile_read synchronises and returns
 * out = { G1 ms total, G1 launches, G1 terms total, G2 ms total, G2 launches,
 *         G2 terms total, kernel launches since the last read, 0 } and resets.      */
int b200_profile(int enable);
int b200_profile_read(double out[8]);

/* ---- polynomials over F_r (coefficient arrays, index = power of x) -------- */
/* out[0..na+nb-1) = a * b.   Replaces PolynomialField.Mul (r1csqap/r1csqap.go:57-67). */
int b200_poly_mul(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out);
/* q[0..na-nb+1) = a div b, rem[0..nb-1) = a mod b (rem may be NULL).
 * Replaces PolynomialField.Div / DivisorPolynomial (r1csqap/r1csqap.go:70-84,213-216).
 * b[nb-1] must be non-zero (B200_EDIVZERO; the reference panics on ModInverse(0)).
 * na < nb: quotient is empty and rem = a (na coefficients), as in the reference. */
int b200_poly_div(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* q, uint64_t* rem);

int b200_poly_add(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out); /* r1csqap.go:94-103, max(na,nb) out */
int b200_poly_sub(const uint64_t* a, size_t na, const uint64_t* b, size_t nb, uint64_t* out); /* r1csqap.go:106-115 */
int b200_poly_eval(const uint64_t* v, size_t n, const uint64_t x[4], uint64_t out[4]);        /* r1csqap.go:118-126 */

/* out[i] = Eval(polys[i], x) for m polynomials of n coefficients each (row-major): the At/Bt/Ct loops of
 * GenerateTrustedSetup (groth16/groth16.go:164-205, snark.go:181-218).                                        */
int b200_poly_eval_batch(const uint64_t* polys, size_t m, size_t n, const uint64_t x[4], uint64_t* out);
/* out[0..n] = coefficients of prod_{i=1}^{n} (x - i): the "z pol" of groth16.go:122-132 / snark.go:221-232; n <= 2^26. */
int b200_zero_poly(size_t n, uint64_t* out);

/* ---- verifier side (SURVEY §8f row 2) ------------------------------------------------------------------ */
/* out[i] = Bn128.Pairing(g1[i], g2[i]) (bn128/bn128.go:179-186): optimal-ate Miller loop + a fast final
 * exponentiation (easy part, then the hard part by the BN parameter) that gives the same F_q^12 value as the
 * reference's plain f^((q^12-1)/r); 48 uint64 per result in the reference's [2][3][2]*big.Int order.  The kernel is
 * B200_CFG_PAIRING_KERNEL's: by default one warp per pairing up to 2048 pairings per call, one thread per pairing above.
 * Bit-identical to the reference (golden: externalVerif/circom-test/verification_key.json vk_alfabeta_12).
 * A G2 point at infinity returns B200_EINVAL where the reference panics "q1[2] != Fq2.One()" (bn128.go:238-241);
 * a G1 point at infinity is processed like the reference does (Affine -> (0,0)).                                    */
int b200_pairing_batch(const uint64_t* g1_jac, const uint64_t* g2_jac, size_t n, uint64_t* out);
/* out[i] = a[i] * b[i] in F_q^12 (fields/fq12.go:72-84; 48 uint64 per element, same order as b200_pairing_batch):
 * the product step of the verification equations (snark.go:338-341,357; groth16.go:297-301).                      */
int b200_fq12_mul_batch(const uint64_t* a, const uint64_t* b, size_t n, uint64_t* out);
/* groth16.VerifyProof (groth16/groth16.go:281-305): *ok = 1 iff e(A,B) == e(alpha,beta) * (e(icPubl,gamma) * e(C,delta)),
 * icPubl = IC[0] + sum publicSignals[i] * IC[i+1].  The four pairings run concurrently.                              */
int b200_groth16_verify(const uint64_t* ic, size_t n_ic, const uint64_t alpha1[12], const uint64_t beta2[24],
                        const uint64_t gamma2[24], const uint64_t delta2[24], const uint64_t pi_a[12],
                        const uint64_t pi_b[24], const uint64_t pi_c[12], const uint64_t* public_signals, size_t n_public,
                        int* ok);
/* ok[i] = groth16.VerifyProof(vk, proof_i, publicSignals_i) for k proofs under one Vk, by one random linear combination:
 *   prod_i e(rho_i A_i, B_i) * e(-(sum rho_i) alpha, beta) * e(-sum rho_i icPubl_i, gamma) * e(-sum rho_i C_i, delta) == 1
 * over the REGULAR proofs: k_reg + 3 Miller loops, one F_q^12 product and ONE final exponentiation for the batch.
 * A proof is regular when PiA and PiC are on y^2 = x^3 + 3 and not infinity, PiB is on the twist and in the order-r
 * subgroup, and its icPubl_i (computed as b200_groth16_verify does, in the reference's order with its Add) is not
 * infinity; under a Vk whose alpha1, beta2, gamma2, delta2 fail the same tests no proof is regular.  The contract:
 *   - every irregular proof gets exactly b200_groth16_verify's verdict (the reference pairs a G1 infinity as (0, 0),
 *     which is not bilinear, so such proofs never enter the aggregate);
 *   - when the aggregate fails, every proof gets exactly b200_groth16_verify's verdict (the per-proof check runs);
 *   - when it passes, every regular proof is accepted.  A batch holding an invalid regular proof passes with probability
 *     below 2^-127 over that proof's rho_i, PROVIDED the randomisers are unpredictable to whoever made the proofs: draw
 *     them from a cryptographic source per call.  The caller supplies them so that runs are reproducible.
 * rho: k x 2 limbs, each 1 <= rho_i < 2^128.  pi_a, pi_c: k x 12, pi_b: k x 24, public_signals: k x n_public x 4,
 * standard-form Jacobian / scalars as b200_groth16_verify takes them.  1 <= k <= 65536.
 * status (may be NULL): bit 0 the aggregate ran over at least one proof and passed; bit 1 the per-proof check ran for
 * some proof; bit 2 an irregular proof or Vk was routed around the aggregate.
 * Errors are b200_groth16_verify's applied to the whole call: B200_ERANGE for a coordinate >= q or a public signal >= r,
 * B200_EINVAL for a G2 input at infinity (the reference panics), a null pointer, n_ic < n_public + 1, k outside
 * 1..65536, or a rho_i of 0.  Runs on context 0's main stream; synchronous.
 * Launches: a fixed sequence of 9 kernels (8 when n_public = 0), whatever k and whatever the outcome.              */
int b200_groth16_verify_batch(const uint64_t* ic, size_t n_ic, const uint64_t alpha1[12], const uint64_t beta2[24],
                              const uint64_t gamma2[24], const uint64_t delta2[24], const uint64_t* pi_a, const uint64_t* pi_b,
                              const uint64_t* pi_c, const uint64_t* public_signals, size_t n_public, size_t k, const uint64_t* rho,
                              int* ok, uint32_t* status);
/* b200_groth16_verify_batch on proofs already in device memory, queued on `stream` (NULL: context 0's main stream)
 * without waiting: d_proofs is k x 48 uint64, PiA | PiC | PiB per proof — exactly b200_groth16_prove_witness_batch_device's
 * d_out, so a batch is verified where it lies; d_public is k x n_public x 4 (standard form); d_ok receives k int32
 * verdicts followed by one uint32 status word (bits 0..2 as above; bit 3: an out-of-range input was seen).
 * The Vk, IC and rho are host arguments and are checked as b200_groth16_verify_batch checks them (B200_ERANGE /
 * B200_EINVAL).  A proof coordinate >= q or a public signal >= r gives that proof verdict 0 and sets status bit 3; a PiB
 * at infinity gives verdict 0.  Neither returns an error code, and nothing of either reaches a later call.  Scratch is
 * stream-ordered device memory (cudaMallocAsync), freed behind the work.                                             */
int b200_groth16_verify_batch_device(const uint64_t* ic, size_t n_ic, const uint64_t alpha1[12], const uint64_t beta2[24],
                                     const uint64_t gamma2[24], const uint64_t delta2[24], const void* d_proofs,
                                     const void* d_public, size_t n_public, size_t k, const uint64_t* rho, void* d_ok,
                                     void* stream);
/* ok[i] = snark.VerifyProof(vk, proof_i, publicSignals_i) (snark.go:292-372) for k Pinocchio proofs under one Vk, by one
 * random linear combination of the five checks of every proof (check c of proof i raised to rho_ic):
 *   prod_i e(P_i, PiB_i) * e(sum rho_i1 PiA_i, Vka) * e(sum rho_i3 PiC_i, Vkc) * e(-sum rho_i4 PiH_i, Vkz)
 *     * e(sum rho_i5 T_i, G2Kbg) * e(-sum rho_i5 PiKp_i, G2Kg)
 *     * e(-sum (rho_i1 PiAp_i + rho_i2 PiBp_i + rho_i3 PiCp_i + rho_i4 PiC_i), g2) == 1,
 *   P_i = rho_i2 Vkb + rho_i4 S_i + rho_i5 G1Kbg,
 * over the REGULAR proofs: k_reg + 6 Miller loops, one F_q^12 product and ONE final exponentiation for the batch.
 * Vkx_i = IC[0] + sum_j pub_ij IC[j+1], S_i = Add(Vkx_i, PiA_i) and T_i = Add(S_i, PiC_i) are the reference's sums, in its
 * order and with its Add (no doubling branch: Vkx_i == PiA_i makes S_i infinity).
 * A proof is regular when every G1 point one of its checks pairs (PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp, S_i, T_i) is on
 * y^2 = x^3 + 3 and not infinity, and PiB is on the twist and in the order-r subgroup; under a Vk whose Vkb, G1Kbg (as G1
 * points) or Vka, Vkc, G2Kbg, G2Kg, Vkz (as G2 points) fail the same tests no proof is regular.  The contract:
 *   - every irregular proof gets exactly snark.VerifyProof's verdict (the reference pairs a G1 infinity as (0, 0), which
 *     is not bilinear, so such proofs never enter the aggregate);
 *   - when the aggregate fails, every proof gets exactly snark.VerifyProof's verdict (the per-proof check runs);
 *   - when it passes, every regular proof is accepted.  A batch holding an invalid regular proof passes with probability
 *     below 2^-127 over that proof's rho_ic, PROVIDED the randomisers are unpredictable to whoever made the proofs: draw
 *     them from a cryptographic source per call.  The caller supplies them so that runs are reproducible.
 * vk_g1 = Vkb | G1Kbg and vk_g2 = Vka | Vkc | G2Kbg | G2Kg | Vkz, as b200_pinocchio_setup / b200_pinocchio_setup_pk return
 * them; ic = A[0..n_ic).  out_g1: k x 84 (PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp) and pi_b: k x 24, exactly
 * b200_pinocchio_prove_witness_batch's outputs; public_signals: k x n_public x 4; standard-form Jacobian / scalars.
 * rho: k x 5 x 2 limbs, rho[10 i + 2 (c - 1)] the low word of rho_ic, each 1 <= rho_ic < 2^128.  1 <= k <= 65536.
 * status (may be NULL): bit 0 the aggregate ran over at least one proof and passed; bit 1 the per-proof check ran for
 * some proof; bit 2 an irregular proof or Vk was routed around the aggregate.
 * Errors: B200_ERANGE for a coordinate >= q (proofs, Vk, IC) or a public signal >= r; B200_EINVAL for PiB or a Vk G2 point
 * at infinity (the reference panics, bn128.go:238-241), a null pointer, n_ic < n_public + 1, k outside 1..65536, or a
 * rho_ic of 0.  Runs on context 0's main stream; synchronous.
 * Launches: a fixed sequence of 9 kernels (8 when n_public = 0), whatever k and whatever the outcome.              */
int b200_pinocchio_verify_batch(const uint64_t* ic, size_t n_ic, const uint64_t vk_g1[24], const uint64_t vk_g2[120],
                                const uint64_t* out_g1, const uint64_t* pi_b, const uint64_t* public_signals, size_t n_public,
                                size_t k, const uint64_t* rho, int* ok, uint32_t* status);
/* b200_pinocchio_verify_batch on proofs already in device memory, queued on `stream` (NULL: context 0's main stream)
 * without waiting: d_proofs is k x 108 uint64, the seven G1 points and then PiB per proof — exactly
 * b200_pinocchio_prove_witness_batch_device's d_out, so a batch is verified where it lies; d_public is k x n_public x 4
 * (standard form); d_ok receives k int32 verdicts followed by one uint32 status word (bits 0..2 as above; bit 3: an
 * out-of-range input was seen).  The Vk, IC and rho are host arguments and are checked as b200_pinocchio_verify_batch
 * checks them (B200_ERANGE / B200_EINVAL).  A proof coordinate >= q or a public signal >= r gives that proof verdict 0
 * and sets status bit 3; a PiB at infinity gives verdict 0.  Neither returns an error code, and nothing of either reaches
 * a later call.  Scratch is stream-ordered device memory (cudaMallocAsync), freed behind the work.  The same 9 (8)
 * launches.                                                                                                          */
int b200_pinocchio_verify_batch_device(const uint64_t* ic, size_t n_ic, const uint64_t vk_g1[24], const uint64_t vk_g2[120],
                                       const void* d_proofs, const void* d_public, size_t n_public, size_t k,
                                       const uint64_t* rho, void* d_ok, void* stream);

/* ---- dense QAP API upstream of GenerateProofs (small n; the prove path consumes px) ---- */
/* PolynomialField.R1CSToQAP (r1csqap/r1csqap.go:161-188).  a, b, c: n x m row-major R1CS matrices (coefficients
 * reduced mod r).  alphas/betas/gammas: m x n (row i = coefficients of signal i's polynomial over the domain {1..n});
 * z: m-1 coefficients of prod_{i=1}^{m-2}(x-i).  Exact big-integer Lagrange denominators: identical to the reference
 * for n <= 21, and the mathematically intended result where the reference's native-int factorial overflows
 * (r1csqap.go:130-136, SURVEY E3).  1 <= n <= 8191.                                                                   */
int b200_r1cs_to_qap(const uint64_t* a, const uint64_t* b, const uint64_t* c, size_t n, size_t m, uint64_t* alphas,
                     uint64_t* betas, uint64_t* gammas, uint64_t* z);
/* PolynomialField.CombinePolynomials (r1csqap/r1csqap.go:191-210): ax = sum r_i*ap[i] (likewise bx, cx; n coefficients
 * each, ap/bp/cp m x n row-major) and px = ax*bx - cx (2n-1 coefficients).                                            */
int b200_combine_polynomials(const uint64_t* r, size_t m, const uint64_t* ap, const uint64_t* bp, const uint64_t* cp,
                             size_t n, uint64_t* ax, uint64_t* bx, uint64_t* cx, uint64_t* px);

/* ---- sparse QAP front end (any n): the same mathematics without the dense m x n polynomial matrices -------- */
/* A sparse R1CS, n constraints x m signals, three CSR matrices (rowptr n+1 entries, col/val nnz entries; val = 4-limb
 * coefficients reduced mod r, negative coefficients of circuitcompiler (circuit.go:78) sent as r - |v|).  Stays on
 * the device; also stored transposed for the trusted setup.  Replaces the dense a, b, c [][]*big.Int arguments of
 * PolynomialField.R1CSToQAP (r1csqap/r1csqap.go:161) where m*n coefficients cannot exist (137 GB per matrix at
 * n = 2^16, SURVEY H4).                                                                                              */
int b200_r1cs_load(size_t n, size_t m, const uint32_t* a_rowptr, const uint32_t* a_col, const uint64_t* a_val,
                   const uint32_t* b_rowptr, const uint32_t* b_col, const uint64_t* b_val, const uint32_t* c_rowptr,
                   const uint32_t* c_col, const uint64_t* c_val, b200_r1cs_t* out);
int b200_r1cs_free(b200_r1cs_t h);
/* CombinePolynomials(w, R1CSToQAP(a, b, c)) (r1csqap/r1csqap.go:161-210) fused: ax, bx, cx (n coefficients each, any
 * may be NULL) and px = ax*bx - cx (2n-1 coefficients).  ax is the unique polynomial of degree < n with
 * ax(j+1) = (A w)_j: one sparse mat-vec and one O(n log^2 n) interpolation over {1..n} per matrix.  Field-exact, so
 * equal to the reference's coefficients wherever the reference can run (n <= 21, SURVEY E3).                          */
int b200_qap_px(b200_r1cs_t h, const uint64_t* w, size_t nw, uint64_t* ax, uint64_t* bx, uint64_t* cx, uint64_t* px);
/* at[i] = Eval(alphas[i], tau), bt[i], ct[i] for every signal i < m — the loops of GenerateTrustedSetup
 * (groth16/groth16.go:164-205, snark.go:171-189) — as A^T l(tau) with l the Lagrange basis of {1..n} at tau, and
 * zt = prod_{i=1..nz} (tau - i) (groth16.go:122-136 with nz = len(alphas) - 2).  tau must not be one of 1..n.          */
int b200_qap_eval_at(b200_r1cs_t h, const uint64_t tau[4], size_t nz, uint64_t* at, uint64_t* bt, uint64_t* ct,
                     uint64_t zt[4]);
/* ---- trusted setup for a sparse R1CS of any size ----
 * groth16.GenerateTrustedSetup (groth16/groth16.go:94-222) and snark.GenerateTrustedSetup (snark.go:98-251) from the
 * resident R1CS (m = its signals, n = its constraints): at / bt / ct = A^T l(T) etc. as in b200_qap_eval_at,
 * Z = prod_{i=1..m-2}(x - i) as in b200_zero_poly, every CRS scalar derived on the device, and every point minted by a
 * fixed-base windowed kernel.  The outputs have the shapes b200_groth16_pk_load(_shard) / b200_pinocchio_pk_load(_shard)
 * take.  All pointers are host pointers; the call is synchronous and runs on the library stream.
 *   - Points are affine (x, y, 1) in standard form, infinity all zero.  They are the same group elements as the
 *     reference's for the same toxic values, not its Jacobian representatives (use the dense setup through
 *     b200_g1/g2_mul_batch_bcast for X,Y,Z-exact points).
 *   - A bad handle, a null pointer, m < 3, or npublic >= m returns B200_EINVAL.
 *   - A toxic value >= r returns B200_ERANGE.
 *   - T in {1..n} returns B200_EINVAL (as b200_qap_eval_at).
 * The reference's k == a + b + c self-check (snark.go:194-199) holds by construction and is not repeated.            */
/* toxic = T, Kalpha, Kbeta, Kgamma, Kdelta (4 limbs each); Kgamma or Kdelta = 0 returns B200_EINVAL.
 * Outputs: at, b1, bacdelta: m G1 points (BACDelta[0..npublic] infinity); b2: m G2 points; ptd: m-1 G1 points;
 * z: m-1 coefficients; ic: npublic+1 G1 points.                                                                     */
int b200_groth16_setup(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[20], uint64_t* at, uint64_t* b1,
                       uint64_t* b2, uint64_t* bacdelta, uint64_t* ptd, uint64_t* z, uint64_t alpha1[12],
                       uint64_t beta1[12], uint64_t delta1[12], uint64_t beta2[24], uint64_t gamma2[24],
                       uint64_t delta2[24], uint64_t* ic);
/* toxic = T, Ka, Kb, Kc, Kbeta, Kgamma, RhoA, RhoB (RhoC = RhoA * RhoB).
 * Outputs: a, ap, bp, c, cp, kp: m G1 points; b2: m G2 points; g1t: m-1 G1 points (T^0 .. T^(m-2)); z: m-1
 * coefficients; vk_g1 = Vkb | G1Kbg; vk_g2 = Vka | Vkc | G2Kbg | G2Kg | Vkz.  The Vk's IC is a[0..npublic].           */
int b200_pinocchio_setup(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[32], uint64_t* a, uint64_t* ap,
                         uint64_t* b2, uint64_t* bp, uint64_t* c, uint64_t* cp, uint64_t* kp, uint64_t* g1t, uint64_t* z,
                         uint64_t vk_g1[24], uint64_t vk_g2[120]);
/* ---- trusted setup straight into a device-resident proving key ----
 * The key that b200_groth16_setup followed by b200_groth16_pk_load_shard(.., window_bits, rank, world) gives (Pinocchio:
 * b200_pinocchio_setup, then b200_pinocchio_pk_load_shard), for the same toxic values and the same b200_config state
 * (B200_CFG_ACC_MODE, B200_CFG_TABLE_WINDOWS, B200_CFG_PK_CONTEXT, B200_CFG_SHARD_*): the same window-table words, the
 * same b200_groth16_shard_info and b200_pk_device_bytes, and the same proofs (as group elements: a proof's Jacobian words
 * vary from run to run on any key, with the order of additions inside a bucket).  No CRS passes
 * through host memory: the scalars and Z stay on the device and every point of the key is minted straight into its
 * table.  A rank mints only what it holds (Groth16: its slices of A, B1, B2 and C||PTD and the blinding points of the
 * sets whose tails it holds; Pinocchio: the whole sets dealt to it); the R1CS evaluation and Z are computed whole on every
 * rank.  rank = 0, world = 1 gives the whole key.
 *   - Call every rank with the same R1CS, npublic and toxic values.  No collective runs and no communicator is read.
 *     Ranks given different toxic values hold parts of different keys: no call can detect it, and their proofs are wrong.
 *   - Outputs (host): the Vk points as b200_groth16_setup / b200_pinocchio_setup return them, and ic (npublic+1 G1
 *     points; Pinocchio: A[0..npublic]).  *out receives the key's handle (free with b200_pk_free).
 *   - Synchronous, on the library stream.
 *   - Errors: those of the setup (a bad handle, a null pointer, m < 3, npublic >= m, T in {1..n}, Kgamma or Kdelta = 0:
 *     B200_EINVAL; a toxic value >= r: B200_ERANGE) and of the load (a bad rank / world, window_bits outside [2, 24]
 *     and not 0, a set beyond 2^26 points or nwin * n >= 2^31: B200_EINVAL; B200_ENOMEM).  On any error no handle is
 *     created and everything allocated is freed.  The Vk outputs may have been written.                            */
int b200_groth16_setup_pk(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[20], int window_bits, int rank, int world,
                          b200_pk_t* out, uint64_t alpha1[12], uint64_t beta2[24], uint64_t gamma2[24], uint64_t delta2[24],
                          uint64_t* ic);
int b200_pinocchio_setup_pk(b200_r1cs_t r1cs, size_t npublic, const uint64_t toxic[32], int window_bits, int rank, int world,
                            b200_pk_t* out, uint64_t vk_g1[24], uint64_t vk_g2[120], uint64_t* ic);
/* PolynomialField.LagrangeInterpolation over x = 1..n (r1csqap/r1csqap.go:150-158) at any n <= 2^26: n values ->
 * n coefficients.                                                                                                    */
int b200_interpolate(const uint64_t* values, size_t n, uint64_t* coeffs);
/* groth16.GenerateProofs fed from the witness: px is computed on the device from the resident R1CS (b200_qap_px) and
 * never leaves HBM; otherwise identical to b200_groth16_prove (groth16/groth16.go:225-278 after the caller's
 * CombinePolynomials step, cli/main.go:339-349).  When len(Z) = n + 1 or len(Z) = n (n >= 2: m = n + 2 or n + 1 signals)
 * the quotient h = DivisorPolynomial(px, Z) is computed without forming px or C w (for len(Z) = n, h = (x - n) q + kappa
 * with one dot product of the witness against a per-R1CS vector); like the reference, it drops the remainder, so a
 * witness that does not satisfy the R1CS gets the same proof as from b200_groth16_prove with its px (which does not
 * verify).  nw must equal the key's m and the R1CS's m.  Like b200_groth16_prove
 * it runs on the key's prove context (B200_CFG_PK_CONTEXT) and waits with the library mutex released, so two host
 * threads proving on keys of contexts 0 and 1 overlap, also when both keys share one R1CS handle.  A sharded key needs
 * a matching communicator (b200_comm_init; SPMD, the proof is returned on every rank); without one the call returns
 * B200_EINVAL — use b200_groth16_prove_witness_device + b200_groth16_finalize_device instead.                         */
int b200_groth16_prove_witness(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, const uint64_t r[4],
                               const uint64_t s[4], uint64_t pi_a[12], uint64_t pi_b[24], uint64_t pi_c[12]);
/* groth16.GenerateProofs fed from a DEVICE-resident witness (m standard-form scalars): b200_groth16_prove_witness with
 * the result left in device memory on `stream`, as in b200_groth16_prove_device (48 u64 PiA | PiC | PiB; on a sharded
 * key without a communicator, the 1 KB partial record for b200_groth16_finalize_device).  Any witness is proved, as
 * by the reference: the quotient drops the remainder of px / Z, as b200_groth16_prove_device does with the same px.
 *   - No host synchronisation, except on the FIRST call for a given (R1CS, prove context) pair: that call builds the
 *     R1CS's interpolation domains (shared by both contexts) and the context's workspaces, and may synchronise.
 *   - Proofs on keys of the two prove contexts may be in flight together on two streams, also on one R1CS handle (each
 *     context has its own workspace on the R1CS).  Two proofs on the SAME context must be ordered by the caller.
 *   - A witness entry >= r is read as 0, and neither this call nor any later one reports it (nor a proof on another
 *     key), as in b200_groth16_prove_device.  r and s are host values and are checked (B200_ERANGE).
 *   - A bad handle, a null pointer, or nw different from the key's m or the R1CS's m returns B200_EINVAL.
 *   - On a sharded key only a rank that holds PowersTauDelta indices (b200_groth16_shard_info needs_px) runs the QAP
 *     front end, and reads the whole witness; every other rank reads only its witness ranges.                       */
int b200_groth16_prove_witness_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw,
                                      const uint64_t r[4], const uint64_t s[4], void* d_out, void* stream);
/* k witness-fed Groth16 proofs under one key in one set of launches.  Proof p is the group element triple that
 * b200_groth16_prove_witness(_device) returns for (w_p, r_p, s_p), satisfied witness or not (compare affine: the
 * Jacobian representatives may differ).  Witness p is at w + p*nw*4 words (k*nw standard-form scalars, row-major); r and
 * s are host arrays of k x 4 limbs (the host splits them for the blinding products).  Outputs: pi_a k x 12, pi_b k x 24,
 * pi_c k x 12 words.
 *   - One batched sort serves the A, B1 and B2 MSMs of all k proofs (scalar vectors w_p ++ [1, r_p, s_p]); C||PTD has
 *     its own.  Each set runs one batched bucket phase (b200_msm_device_batch), the blinding products take one warp per
 *     proof and one kernel combines the k proofs.
 *   - len(Z) = n + 1 or n, n >= 2 (the shapes whose proofs can verify: m = n + 2 or n + 1): the k quotients come from
 *     one batched front end (witness load, one sparse product of A and B over all k witnesses, Newton coefficients,
 *     shift products, interpolation; for len(Z) = n one more launch, the k dot products), so a batch issues the
 *     launches of a batch of one, plus the documented extras of b200_msm_device_batch (one more launch when
 *     k*G*2^(c-1) bucket counters of a set exceed 64 Ki, one or two per further 65535 tail rows).  Any other len(Z)
 *     (m > n + 2, or n = 1) takes px and the division like the single entry, once per witness: correct, but not
 *     batched.
 *   - Runs on the key's prove context; calls on keys of one context must be ordered.  Batches on keys of contexts 0 and
 *     1 may be in flight together, also on one R1CS handle.  Waits with the library mutex released.
 *   - Scratch: about k times one proof's sort, bucket and front-end scratch.  The key's (counted by
 *     b200_pk_device_bytes: scalar vectors, records, the sets' batch sorts and bucket phases) and the R1CS workspace's
 *     are allocated on the first batch and grown (never shrunk) by a larger one, which first waits for the previous
 *     batch; the pinned landing area of this entry holds k*48 + 1 words.
 *   - B200_EINVAL before anything is allocated or enqueued: k = 0, a bad handle or null pointer, nw different from the
 *     key's m or the R1CS's m, a sharded key without a matching communicator (use
 *     b200_groth16_prove_witness_batch_partial_device + b200_groth16_finalize_batch_device around your own all-gather),
 *     or a batch too large for 32-bit indexing: k*ceil(255/c)*(m+3) sort entries (or k times a set's buckets) reaching
 *     2^31, the same for the C||PTD set, or 3k*2N >= 2^32 transform elements (N = the power of two >= n).
 *   - B200_ERANGE: any r_p or s_p >= r (before anything is enqueued); a witness entry >= r in any witness (the outputs
 *     are left untouched, and the next call starts from a clear error word).
 *   - A sharded key (b200_groth16_pk_load_shard) with a matching communicator (b200_comm_init; SPMD, every rank calls
 *     with the same witnesses, r and s): each rank computes its part of the k proofs (the launches of its part of one
 *     proof, whatever k), one ncclAllGather of k 1 KB records per rank runs on the key's prove-context communicator
 *     on the key's main stream, and one launch finalises: every rank returns all k proofs.  Only the witness ranges the
 *     rank reads are uploaded (all of each witness on a rank that needs px).  The size refusals above are decided on
 *     the largest part ANY rank of the shard holds, so every rank returns the same code before anything is enqueued.
 *     A device allocation failure (B200_ENOMEM / B200_ECUDA) while the batch's scratch grows can happen on some ranks only:
 *     those ranks return before the all-gather and their peers wait in it; once the scratch exists, the all-gather runs
 *     whatever else fails.
 *     A witness entry >= r: the ranks that read it return B200_ERANGE, the others B200_OK with proofs that are not
 *     those of the witnesses (the all-gather runs either way).  Scratch: k times the rank's slices, k records and a
 *     gather buffer of world*k records, grown and never shrunk, counted by b200_pk_device_bytes. */
int b200_groth16_prove_witness_batch(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, size_t k,
                                     const uint64_t* r, const uint64_t* s,
                                     uint64_t* pi_a, uint64_t* pi_b, uint64_t* pi_c);
/* b200_groth16_prove_witness_batch from device memory: d_w holds the k witnesses (standard form, witness p at
 * d_w + p*nw*32 bytes), d_out receives k x 48 u64 on `stream`, proof p at d_out + 48p in the PiA | PiC | PiB order of
 * b200_groth16_prove_witness_device.  r and s stay host arrays (k x 4 limbs).  No host synchronisation, except in a
 * call that first meets a given (R1CS, prove context) pair or grows a scratch; a regrowth waits for an event recorded
 * behind the key's previous batch, not for the device.  A witness entry >= r is read as 0 and reported by no call, as
 * in b200_groth16_prove_witness_device; the other errors are those of the host entry. */
int b200_groth16_prove_witness_batch_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                            const uint64_t* r, const uint64_t* s, void* d_out, void* stream);
/* This rank's part of b200_groth16_prove_witness_batch_device on a key shard, for a caller that runs its own collective
 * or emulates the ranks on one GPU: d_parts receives k partial records of 1 KB on `stream`, record p at
 * d_parts + 1024p, in the layout of b200_groth16_prove_device's single record (A @ +0, B1 @ +256, B2 @ +512, the C part
 * with s_p*A_part + r_p*B1_part folded in @ +768; XYZZ; a set the rank does not hold is infinity).
 *   - It never gathers, with or without a communicator.  A world == 1 key gives its k records too (the finalize input
 *     for world = 1).
 *   - Only a rank that holds PowersTauDelta indices (b200_groth16_shard_info needs_px) runs the QAP front end (one
 *     batched front end for the h-direct shape) and reads whole witnesses; a rank that holds no part of A or B1 runs
 *     no blinding products.  Launches: those of the rank's part of one proof, whatever k, plus the documented extras of
 *     b200_msm_device_batch.
 *   - Synchronisation, scratch and the error word as in b200_groth16_prove_witness_batch_device (a witness entry >= r
 *     is read as 0 and reported by no call).
 *   - B200_EINVAL before anything is allocated or enqueued: k = 0, a bad handle or null pointer, nw different from the
 *     key's m or the R1CS's m, or a batch too large for 32-bit indexing on the largest part of ANY rank of the shard
 *     (the same answer on every rank's key).  B200_ERANGE: any r_p or s_p >= r. */
int b200_groth16_prove_witness_batch_partial_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                                    const uint64_t* r, const uint64_t* s, void* d_parts, void* stream);
/* world x k partial records -> k proofs, one launch on `stream` (null: the library stream), no host synchronisation.
 * The record of rank g for proof p is at d_parts + 1024*(g*k + p): what ncclAllGather of k KB per rank leaves.  d_out
 * receives k x 48 u64, proof p at d_out + 48p (PiA | PiC | PiB, Jacobian, standard form); proof p equals what
 * b200_groth16_finalize_device gives for that proof's world records.  pk only names the key (any rank's).
 *   - B200_EINVAL: a bad handle, a null pointer, world < 1, k = 0 or k >= 2^32. */
int b200_groth16_finalize_batch_device(b200_pk_t pk, const void* d_parts, int world, size_t k, void* d_out, void* stream);

/* ---- Pinocchio from device memory, from the witness, and in batches ----------------------------------------------------
 * The twins of the Groth16 entries above for snark.GenerateProofs (snark.go:254-289).  Pinocchio has no blinding, so there
 * is no r or s.  Output layout everywhere: the 7 Jacobian G1 points in the order of b200_pinocchio_prove (PiA, PiAp, PiBp,
 * PiC, PiCp, PiH, PiKp; 84 u64) and PiB (24 u64), standard form; in device memory those 108 u64 are contiguous (the G1
 * block, then PiB).  All of them run on the key's prove context (B200_CFG_PK_CONTEXT); two proofs on keys of ONE context
 * must be ordered by the caller, proofs on keys of contexts 0 and 1 may be in flight together.                           */
/* b200_pinocchio_prove with the witness and px already resident in DEVICE memory (standard form) and the 108-u64 proof
 * left in device memory on `stream`; no host synchronisation.  As in b200_groth16_prove_device, a witness entry or a px
 * coefficient >= r is read as 0, and neither this call nor any later one reports it (nor a proof on another key).
 * B200_EINVAL: a bad handle (a Groth16 key included), a null pointer, nw different from the key's m, len(px) < len(Z),
 * len(hx) > len(G1T).  On a sharded key (b200_pinocchio_pk_load_shard) only the rank that holds G1T reads px; with a
 * matching communicator d_out receives the whole proof on every rank, without one the rank's 2 KB record (the layout of
 * b200_pinocchio_prove_record_device) for b200_pinocchio_finalize_records.                                            */
int b200_pinocchio_prove_device(b200_pk_t pk, const void* d_w, size_t nw, const void* d_px, size_t npx, void* d_out,
                                void* stream);
/* snark.GenerateProofs fed from the witness: the quotient is computed on the device from the resident R1CS and never
 * leaves HBM; otherwise identical to b200_pinocchio_prove with px = CombinePolynomials(w, R1CSToQAP(a, b, c)).  When
 * len(Z) = n + 1 or n and n >= 2 the quotient h = DivisorPolynomial(px, Z) is computed without forming px or C w; any
 * other len(Z) takes px (b200_qap_px) and the key's division.  Like the reference it drops the remainder, so a witness
 * that does not satisfy the R1CS gets the proof b200_pinocchio_prove gives for that witness and its px (which does not
 * verify).  The front end runs on the stream the G1T MSM runs on, beside the seven witness MSMs.  nw must equal the key's
 * m and the R1CS's m.  Unlike b200_pinocchio_prove it waits with the library mutex released, so two host threads proving
 * on keys of contexts 0 and 1 overlap, also when both keys share one R1CS handle.  A witness entry >= r gives B200_ERANGE
 * from the key's own error word; the outputs are left untouched and the next call starts from a clear word.  A sharded
 * key needs a matching communicator (SPMD, the proof is returned on every rank); without one the call returns
 * B200_EINVAL — use b200_pinocchio_prove_witness_device + b200_pinocchio_finalize_records instead.                      */
int b200_pinocchio_prove_witness(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, uint64_t* out_g1,
                                 uint64_t pi_b[24]);
/* b200_pinocchio_prove_witness from a DEVICE-resident witness (m standard-form scalars), the result left in device
 * memory on `stream` as in b200_pinocchio_prove_device.
 *   - No host synchronisation, except on the FIRST call for a given (R1CS, prove context) pair: that call builds the
 *     R1CS's interpolation domains (shared by both contexts) and the context's workspace, and may synchronise.
 *   - Proofs on keys of the two prove contexts may be in flight together on two streams, also on one R1CS handle (each
 *     context has its own workspace on the R1CS, which a Groth16 key of that context shares).
 *   - A witness entry >= r is read as 0 and reported by no call, as in b200_pinocchio_prove_device.
 *   - A bad handle, a null pointer, nw different from the key's m or the R1CS's m, or an R1CS whose quotient does not fit
 *     the key (len(px) = 2n - 1 < len(Z), len(hx) > len(G1T)) returns B200_EINVAL.
 *   - On a sharded key only the rank that holds G1T runs the QAP front end (on the whole witness); every other rank
 *     launches no QAP kernel.  Without a matching communicator d_out receives the rank's 2 KB record.                   */
int b200_pinocchio_prove_witness_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, void* d_out,
                                        void* stream);
/* k witness-fed Pinocchio proofs under one key in one set of launches.  Proof p is the group-element octuple that
 * b200_pinocchio_prove_witness(_device) returns for w_p, satisfied witness or not (compare affine: the Jacobian
 * representatives may differ).  Witness p is at w + p*nw*4 words; outputs: out_g1 k x 84, pi_b k x 24 words.
 *   - Three batched sorts, eight batched bucket phases (b200_msm_device_batch), whatever k.  The scalar vectors of the
 *     seven witness MSMs are the witnesses where they lie: one sort of w_p (stride nw) serves B, Bp, C, Cp, Kp, one of
 *     w_p[NPublic+1..) serves A, Ap, one of the k quotient vectors serves G1T; one kernel writes the k proofs.
 *   - len(Z) = n + 1 or n, n >= 2 (m = n + 2 or n + 1): the k quotients come from one batched front end (for len(Z) = n
 *     one more launch, the k dot products), so a batch issues the launches of a batch of one, plus the documented extras
 *     of b200_msm_device_batch.  Any other len(Z) takes px and the division like the single entry, once per witness:
 *     correct, but not batched.
 *   - Waits with the library mutex released; batches on keys of contexts 0 and 1 may be in flight together, also on one
 *     R1CS handle.
 *   - Scratch: about k times one proof's sort, bucket and front-end scratch.  The key's (counted by b200_pk_device_bytes:
 *     quotient vectors, records, the eight sets' batch sorts and bucket phases) and the R1CS workspace's are allocated on
 *     the first batch and grown (never shrunk) by a larger one, which first waits for the previous batch; the pinned
 *     landing area of this entry holds k*108 + 1 words.
 *   - B200_EINVAL before anything is allocated or enqueued: k = 0, a bad handle or null pointer, the size mismatches of
 *     the single entry, a sharded key without a matching communicator (use
 *     b200_pinocchio_prove_witness_batch_record_device + b200_pinocchio_finalize_records_batch_device around your own
 *     all-gather), or a batch too large for 32-bit indexing: k*ceil(255/c)*terms sort entries (or k times a set's
 *     buckets) of any of the eight sets reaching 2^31, or 3k*2N >= 2^32 transform elements (N = the power of two >= n).
 *   - B200_ERANGE: a witness entry >= r in any witness (the outputs are left untouched, and the next call starts from a
 *     clear error word).
 *   - A sharded key with a matching communicator (b200_comm_init; SPMD, every rank passes the same witnesses): each rank
 *     runs only the sets it owns, one ncclAllGather of k 2 KB records per rank runs on the key's prove-context
 *     communicator, and one launch finalises: every rank returns all k proofs.  The size refusals are decided on every
 *     set of the key, owned or not, so every rank returns the same code; an allocation failure while the scratch grows
 *     can happen on some ranks only, and their peers then wait in the all-gather.  A witness entry >= r: the ranks that
 *     read it return B200_ERANGE, the others B200_OK with proofs that are not those of the witnesses. */
int b200_pinocchio_prove_witness_batch(b200_pk_t pk, b200_r1cs_t r1cs, const uint64_t* w, size_t nw, size_t k,
                                       uint64_t* out_g1, uint64_t* pi_b);
/* b200_pinocchio_prove_witness_batch from device memory: d_w holds the k witnesses (standard form, witness p at
 * d_w + p*nw*32 bytes), d_out receives k x 108 u64 on `stream`, proof p at d_out + 108p.  No host synchronisation, except
 * in a call that first meets a given (R1CS, prove context) pair or grows a scratch; a regrowth waits for an event
 * recorded behind the key's previous batch, not for the device.  A witness entry >= r is read as 0 and reported by no
 * call; the other errors are those of the host entry. */
int b200_pinocchio_prove_witness_batch_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                              void* d_out, void* stream);
/* This rank's part of b200_pinocchio_prove_witness_batch_device on a key shard (b200_pinocchio_pk_load_shard), for a
 * caller that runs its own collective or emulates the ranks on one GPU: d_records receives k records of 2 KB on
 * `stream`, record p at d_records + 2048p, in the layout of b200_pinocchio_prove_record_device's single record (eight
 * XYZZ slots of 256 B: PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp, PiB; a set the rank does not own is infinity).
 *   - It never gathers, with or without a communicator; a world == 1 key gives its k records too.
 *   - Only the sets the rank owns run (whole MSMs are dealt to the ranks); a sort group whose sorting set lives on another
 *     rank is sorted by the first set of the group the rank owns; only the rank that owns G1T runs the QAP front end.
 *   - Synchronisation, scratch and the error word as in b200_pinocchio_prove_witness_batch_device.
 *   - B200_EINVAL before anything is allocated or enqueued: k = 0, a bad handle or null pointer, nw different from the
 *     key's m or the R1CS's m, or a batch too large for 32-bit indexing on any set of the key, owned or not (the same
 *     answer on every rank's key). */
int b200_pinocchio_prove_witness_batch_record_device(b200_pk_t pk, b200_r1cs_t r1cs, const void* d_w, size_t nw, size_t k,
                                                     void* d_records, void* stream);
/* world x k records -> k proofs, one launch on `stream` (null: the library stream), no host synchronisation.  The
 * record of rank g for proof p is at d_records + 2048*(g*k + p): what ncclAllGather of 2k KB per rank leaves.  d_out
 * receives k x 108 u64, proof p at d_out + 108p (the seven G1 points, then PiB); proof p equals what
 * b200_pinocchio_finalize_records gives for that proof's world records.
 *   - B200_EINVAL: a null pointer, world < 1, k = 0 or k >= 2^28. */
int b200_pinocchio_finalize_records_batch_device(const void* d_records, int world, size_t k, void* d_out, void* stream);

/* ---- element-wise group operations, reference formulas (X,Y,Z-exact) ------------------- */
/* bn128.G1.Add / Double / Neg / Affine (bn128/g1.go:32-170) and the G2 twins (bn128/g2.go:32-200), n independent
 * operations per call.  Affine writes (x, y) per point, infinity as (0, 0) like G1.Affine.                            */
int b200_g1_add_batch(const uint64_t* p, const uint64_t* q, size_t n, uint64_t* out);
int b200_g1_double_batch(const uint64_t* p, size_t n, uint64_t* out);
int b200_g1_neg_batch(const uint64_t* p, size_t n, uint64_t* out);
int b200_g1_affine_batch(const uint64_t* p, size_t n, uint64_t* out_xy);
int b200_g2_add_batch(const uint64_t* p, const uint64_t* q, size_t n, uint64_t* out);
int b200_g2_double_batch(const uint64_t* p, size_t n, uint64_t* out);
int b200_g2_neg_batch(const uint64_t* p, size_t n, uint64_t* out);
int b200_g2_affine_batch(const uint64_t* p, size_t n, uint64_t* out_xy);

#ifdef __cplusplus
}
#endif
#endif /* B200SNARK_H */
