// Package b200 is the cgo binding of libb200snark (include/b200snark.h): the marshalling layer a
// maintainer of arnaucube/go-snark-study links under groth16.GenerateProofs / snark.GenerateProofs /
// r1csqap.PolynomialField / bn128.G1,G2 to run the prove path on an H100.
//
// NOT COMPILED IN THIS REPOSITORY: neither the build image nor the GPU box has a Go toolchain
// (`go version`: not found).  The identical marshalling is exercised through ctypes by the Python
// mirror (go-snark-study_b200/_lib.py) in tests/.  See INTEGRATION.md.
package b200

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../go-snark-study_b200/lib -lb200snark
#include <stdlib.h>
#include "b200snark.h"
*/
import "C"

import (
	"crypto/sha256"
	"encoding/binary"
	"errors"
	"hash"
	"math/big"
	"sync"
	"unsafe"
)

// R is the BN254 scalar-field order (bn128/bn128.go:46).
var R, _ = new(big.Int).SetString("21888242871839275222246405745257275088548364400416034343698204186575808495617", 10)

func check(rc C.int) error {
	if rc == 0 {
		return nil
	}
	return errors.New("libb200snark: " + C.GoString(C.b200_last_error()))
}

// limbs appends the 4 little-endian 64-bit limbs of x (0 <= x < 2^256) to dst.
func limbs(dst []uint64, x *big.Int) []uint64 {
	w := x.Bits() // amd64: big.Word is 64-bit, little endian
	for i := 0; i < 4; i++ {
		if i < len(w) {
			dst = append(dst, uint64(w[i]))
		} else {
			dst = append(dst, 0)
		}
	}
	return dst
}

// Scalar is what crosses the ABI for a *big.Int scalar: |e| mod r (the reference's MulScalar
// consumes |e|: fields/fq.go:138-140).  For |e| >= r that is not always the reference's group
// element: its double-and-add meets Add(P, P) = infinity for crafted values such as r + 2.  The
// Python binding's bn128.reduce_scalar has the rule that matches; this function does not have it yet.
func Scalar(e *big.Int) *big.Int { return new(big.Int).Mod(new(big.Int).Abs(e), R) }

// Coeff is what crosses the ABI for a polynomial coefficient: e mod r (Euclidean, like Fq.Add/Mul).
func Coeff(e *big.Int) *big.Int { return new(big.Int).Mod(e, R) }

func FlatFr(v []*big.Int, reduce func(*big.Int) *big.Int) []uint64 {
	out := make([]uint64, 0, 4*len(v))
	for _, x := range v {
		out = limbs(out, reduce(x))
	}
	return out
}
func FlatG1(pts [][3]*big.Int) []uint64 {
	out := make([]uint64, 0, 12*len(pts))
	for _, p := range pts {
		for k := 0; k < 3; k++ {
			out = limbs(out, p[k])
		}
	}
	return out
}
func FlatG2(pts [][3][2]*big.Int) []uint64 {
	out := make([]uint64, 0, 24*len(pts))
	for _, p := range pts {
		for k := 0; k < 3; k++ {
			out = limbs(limbs(out, p[k][0]), p[k][1])
		}
	}
	return out
}
func fromLimbs(w []uint64) *big.Int {
	words := make([]big.Word, len(w))
	for i, x := range w {
		words[i] = big.Word(x)
	}
	return new(big.Int).SetBits(words)
}
func G1FromLimbs(w []uint64) [3]*big.Int {
	return [3]*big.Int{fromLimbs(w[0:4]), fromLimbs(w[4:8]), fromLimbs(w[8:12])}
}
func G2FromLimbs(w []uint64) [3][2]*big.Int {
	var p [3][2]*big.Int
	for k := 0; k < 3; k++ {
		p[k] = [2]*big.Int{fromLimbs(w[8*k : 8*k+4]), fromLimbs(w[8*k+4 : 8*k+8])}
	}
	return p
}
func u64(v []uint64) *C.uint64_t { return (*C.uint64_t)(unsafe.Pointer(&v[0])) }

// Groth16Key is a device-resident proving key (b200_pk_t).
type Groth16Key struct{ h C.b200_pk_t }

// LoadGroth16 uploads groth16.Pk once (b200_groth16_pk_load).
func LoadGroth16(at, b1 [][3]*big.Int, b2 [][3][2]*big.Int, bacDelta, ptd [][3]*big.Int, z []*big.Int,
	alpha1, beta1, delta1 [3]*big.Int, beta2, delta2 [3][2]*big.Int, nVars, nPublic int) (*Groth16Key, error) {
	fa, fb1, fb2, fc, fp := FlatG1(at[:nVars]), FlatG1(b1[:nVars]), FlatG2(b2[:nVars]), FlatG1(bacDelta[:nVars]), FlatG1(ptd)
	fz := FlatFr(z, Coeff)
	a1, be1, d1 := FlatG1([][3]*big.Int{alpha1}), FlatG1([][3]*big.Int{beta1}), FlatG1([][3]*big.Int{delta1})
	be2, d2 := FlatG2([][3][2]*big.Int{beta2}), FlatG2([][3][2]*big.Int{delta2})
	var k Groth16Key
	rc := C.b200_groth16_pk_load(u64(fa), u64(fb1), u64(fb2), u64(fc), C.size_t(nVars), u64(fp), C.size_t(len(ptd)),
		u64(fz), C.size_t(len(z)), u64(a1), u64(be1), u64(d1), u64(be2), u64(d2), C.size_t(nPublic), 0, &k.h)
	return &k, check(rc)
}

// Prove is groth16.GenerateProofs after the randomness has been drawn (groth16.go:231-238).
func (k *Groth16Key) Prove(w, px []*big.Int, r, s *big.Int) (piA [3]*big.Int, piB [3][2]*big.Int, piC [3]*big.Int, err error) {
	fw, fpx := FlatFr(w, Scalar), FlatFr(px, Coeff)
	fr, fs := limbs(nil, r), limbs(nil, s)
	a, b, c := make([]uint64, 12), make([]uint64, 24), make([]uint64, 12)
	rc := C.b200_groth16_prove(k.h, u64(fw), C.size_t(len(w)), u64(fpx), C.size_t(len(px)), u64(fr), u64(fs), u64(a), u64(b), u64(c))
	if err = check(rc); err != nil {
		return
	}
	return G1FromLimbs(a), G2FromLimbs(b), G1FromLimbs(c), nil
}

func (k *Groth16Key) Free() { C.b200_pk_free(k.h) }

// LoadGroth16Pair uploads the same groth16.Pk under the library's two prove contexts (B200_CFG_PK_CONTEXT 0 and 1: own
// tables, scratch, streams).  Two goroutines — one per key — may then call Prove concurrently: a call enqueues under the
// library mutex and waits for its proof with the mutex released, so the sort / bucket-tail / blinding-product chains of one
// proof overlap the bucket accumulation of the other (a proof server's steady state; bench.py `proofs_in_flight`).  cgo releases the goroutine's OS thread for the duration of the call.
func LoadGroth16Pair(at, b1 [][3]*big.Int, b2 [][3][2]*big.Int, bacDelta, ptd [][3]*big.Int, z []*big.Int,
	alpha1, beta1, delta1 [3]*big.Int, beta2, delta2 [3][2]*big.Int, nVars, nPublic int) (keys [2]*Groth16Key, err error) {
	for ctx := 0; ctx < 2; ctx++ {
		if err = check(C.b200_config(C.B200_CFG_PK_CONTEXT, C.int(ctx))); err != nil {
			break
		}
		if keys[ctx], err = LoadGroth16(at, b1, b2, bacDelta, ptd, z, alpha1, beta1, delta1, beta2, delta2, nVars, nPublic); err != nil {
			break
		}
	}
	C.b200_config(C.B200_CFG_PK_CONTEXT, 0)
	return
}

// SetTableWindows sets how many precomputed window rows base sets and proving keys loaded afterwards store
// (B200_CFG_TABLE_WINDOWS): 0 all (the default, fastest), fewer for circuits whose keys do not fit on the GPU otherwise.
func SetTableWindows(t int) error { return check(C.b200_config(C.B200_CFG_TABLE_WINDOWS, C.int(t))) }

// LoadGroth16Windows is LoadGroth16 with t stored window rows per base set (SetTableWindows); the option is 0 again after.
func LoadGroth16Windows(at, b1 [][3]*big.Int, b2 [][3][2]*big.Int, bacDelta, ptd [][3]*big.Int, z []*big.Int,
	alpha1, beta1, delta1 [3]*big.Int, beta2, delta2 [3][2]*big.Int, nVars, nPublic, t int) (key *Groth16Key, err error) {
	if err = SetTableWindows(t); err != nil {
		return nil, err
	}
	key, err = LoadGroth16(at, b1, b2, bacDelta, ptd, z, alpha1, beta1, delta1, beta2, delta2, nVars, nPublic)
	SetTableWindows(0)
	return
}

// DeviceBytes is the device memory the key holds (b200_pk_device_bytes).
func (k *Groth16Key) DeviceBytes() (uint64, error) {
	var b C.size_t
	err := check(C.b200_pk_device_bytes(k.h, &b))
	return uint64(b), err
}

// PolyMul / PolyDiv back r1csqap.PolynomialField.Mul / Div (r1csqap/r1csqap.go:57-84).
func PolyMul(a, b []*big.Int) ([]*big.Int, error) {
	fa, fb := FlatFr(a, Coeff), FlatFr(b, Coeff)
	out := make([]uint64, 4*(len(a)+len(b)-1))
	if err := check(C.b200_poly_mul(u64(fa), C.size_t(len(a)), u64(fb), C.size_t(len(b)), u64(out))); err != nil {
		return nil, err
	}
	res := make([]*big.Int, len(a)+len(b)-1)
	for i := range res {
		res[i] = fromLimbs(out[4*i : 4*i+4])
	}
	return res, nil
}

// Fq12FromLimbs unpacks b200_pairing_batch's 48 words into the reference's [2][3][2]*big.Int (fields/fq12.go).
func Fq12FromLimbs(w []uint64) (r [2][3][2]*big.Int) {
	for h := 0; h < 2; h++ {
		for k := 0; k < 3; k++ {
			for c := 0; c < 2; c++ {
				o := 4 * (6*h + 2*k + c)
				r[h][k][c] = fromLimbs(w[o : o+4])
			}
		}
	}
	return
}

// Pairing backs bn128.Bn128.Pairing (bn128/bn128.go:179-186).
func Pairing(p1 [3]*big.Int, p2 [3][2]*big.Int) ([2][3][2]*big.Int, error) {
	out := make([]uint64, 48)
	g1, g2 := FlatG1([][3]*big.Int{p1}), FlatG2([][3][2]*big.Int{p2})
	err := check(C.b200_pairing_batch(u64(g1), u64(g2), 1, u64(out)))
	return Fq12FromLimbs(out), err
}

// Fq12Mul backs fields.Fq12.Mul in the verification equations (fields/fq12.go:72-84).
func Fq12Mul(a, b [2][3][2]*big.Int) ([2][3][2]*big.Int, error) {
	flat := func(x [2][3][2]*big.Int) []uint64 {
		out := make([]uint64, 0, 48)
		for h := 0; h < 2; h++ {
			for k := 0; k < 3; k++ {
				for c := 0; c < 2; c++ {
					out = limbs(out, x[h][k][c])
				}
			}
		}
		return out
	}
	fa, fb := flat(a), flat(b)
	out := make([]uint64, 48)
	err := check(C.b200_fq12_mul_batch(u64(fa), u64(fb), 1, u64(out)))
	return Fq12FromLimbs(out), err
}

// ---- proving-key cache for the drop-in GenerateProofs(circuit, pk, w, px) form --------------------------------------
// The reference passes Pk BY VALUE (groth16/groth16.go:225), so neither pointer identity nor slice headers identify a
// key across calls (a caller may rebuild an equal Pk, or reuse a backing array for a different one).  The cache key is
// a CONTENT fingerprint: SHA-256 over the array lengths, NVars/NPublic, the three blinding points, Z, and the first
// and last `fpSample` points of every CRS array.  (A maintainer who wants no hashing at all uses the explicit handle
// API instead: LoadGroth16 once, key.Prove per proof.)  At most `cap` keys stay resident; eviction frees device tables.
const fpSample = 8

type fingerprint [32]byte

func hashInt(h hash.Hash, x *big.Int) { h.Write(x.Bytes()); h.Write([]byte{0xff}) }
func hashG1(h hash.Hash, pts [][3]*big.Int) {
	binary.Write(h, binary.LittleEndian, uint64(len(pts)))
	for i, p := range pts {
		if i >= fpSample && i < len(pts)-fpSample {
			continue
		}
		for k := 0; k < 3; k++ {
			hashInt(h, p[k])
		}
	}
}
func hashG2(h hash.Hash, pts [][3][2]*big.Int) {
	binary.Write(h, binary.LittleEndian, uint64(len(pts)))
	for i, p := range pts {
		if i >= fpSample && i < len(pts)-fpSample {
			continue
		}
		for k := 0; k < 3; k++ {
			hashInt(h, p[k][0])
			hashInt(h, p[k][1])
		}
	}
}

// Groth16Fingerprint identifies a groth16.Pk by content (see above).
func Groth16Fingerprint(at, b1 [][3]*big.Int, b2 [][3][2]*big.Int, bacDelta, ptd [][3]*big.Int, z []*big.Int,
	alpha1, beta1, delta1 [3]*big.Int, beta2, delta2 [3][2]*big.Int, nVars, nPublic int) fingerprint {
	h := sha256.New()
	binary.Write(h, binary.LittleEndian, [2]uint64{uint64(nVars), uint64(nPublic)})
	hashG1(h, at)
	hashG1(h, b1)
	hashG2(h, b2)
	hashG1(h, bacDelta)
	hashG1(h, ptd)
	hashG1(h, [][3]*big.Int{alpha1, beta1, delta1})
	hashG2(h, [][3][2]*big.Int{beta2, delta2})
	for _, c := range z {
		hashInt(h, c)
	}
	var f fingerprint
	copy(f[:], h.Sum(nil))
	return f
}

// KeyCache keeps the most recently used device keys (safe for concurrent callers).
type KeyCache struct {
	mu    sync.Mutex
	cap   int
	order []fingerprint
	keys  map[fingerprint]*Groth16Key
}

func NewKeyCache(capacity int) *KeyCache {
	return &KeyCache{cap: capacity, keys: make(map[fingerprint]*Groth16Key)}
}

// Get returns the cached key for fp or loads it with load() and evicts (and frees) the least recently used one.
func (c *KeyCache) Get(fp fingerprint, load func() (*Groth16Key, error)) (*Groth16Key, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	if k, ok := c.keys[fp]; ok {
		for i, f := range c.order {
			if f == fp {
				c.order = append(append(c.order[:i:i], c.order[i+1:]...), fp)
				break
			}
		}
		return k, nil
	}
	k, err := load()
	if err != nil {
		return nil, err
	}
	c.keys[fp] = k
	c.order = append(c.order, fp)
	for len(c.order) > c.cap {
		old := c.order[0]
		c.order = c.order[1:]
		c.keys[old].Free()
		delete(c.keys, old)
	}
	return k, nil
}

// ---- sparse R1CS, witness -> px, witness -> proof (include/b200snark.h: b200_r1cs_load, b200_qap_px, ..) ---------------
// The dense a, b, c [][]*big.Int of r1csqap.R1CSToQAP (r1csqap.go:161) cannot exist at 2^16+ constraints; a caller at
// that size keeps the R1CS in CSR form and calls CombinePolynomials directly on it.
type R1CS struct {
	h    C.b200_r1cs_t
	N, M int
}

// DenseToCSR converts the reference's dense matrix (rows = constraints) to CSR with coefficients mod r.
func DenseToCSR(m [][]*big.Int) (rowptr, col []uint32, val []uint64) {
	rowptr = append(rowptr, 0)
	for _, row := range m {
		for i, x := range row {
			if c := Coeff(x); c.Sign() != 0 {
				col = append(col, uint32(i))
				val = limbs(val, c)
			}
		}
		rowptr = append(rowptr, uint32(len(col)))
	}
	return
}

func u32(v []uint32) *C.uint32_t {
	if len(v) == 0 {
		return nil
	}
	return (*C.uint32_t)(unsafe.Pointer(&v[0]))
}
func u64n(v []uint64) *C.uint64_t {
	if len(v) == 0 {
		return nil
	}
	return u64(v)
}

// LoadR1CS uploads the three matrices (dense reference form) once.
func LoadR1CS(a, b, c [][]*big.Int) (*R1CS, error) {
	ar, ac, av := DenseToCSR(a)
	br, bc, bv := DenseToCSR(b)
	cr, cc, cv := DenseToCSR(c)
	r := &R1CS{N: len(a), M: len(a[0])}
	rc := C.b200_r1cs_load(C.size_t(r.N), C.size_t(r.M), u32(ar), u32(ac), u64n(av), u32(br), u32(bc), u64n(bv),
		u32(cr), u32(cc), u64n(cv), &r.h)
	return r, check(rc)
}

// CombinePolynomials == PolynomialField.CombinePolynomials(w, R1CSToQAP(a, b, c)...) (r1csqap.go:161-210).
func (r *R1CS) CombinePolynomials(w []*big.Int) (ax, bx, cx, px []*big.Int, err error) {
	fw := FlatFr(w, Coeff)
	oa, ob, oc, op := make([]uint64, 4*r.N), make([]uint64, 4*r.N), make([]uint64, 4*r.N), make([]uint64, 4*(2*r.N-1))
	if err = check(C.b200_qap_px(r.h, u64(fw), C.size_t(len(w)), u64(oa), u64(ob), u64(oc), u64(op))); err != nil {
		return
	}
	un := func(v []uint64) []*big.Int {
		out := make([]*big.Int, len(v)/4)
		for i := range out {
			out[i] = fromLimbs(v[4*i : 4*i+4])
		}
		return out
	}
	return un(oa), un(ob), un(oc), un(op), nil
}
func (r *R1CS) Free() { C.b200_r1cs_free(r.h) }

// ProveWitness is GenerateProofs fed from the witness: px never leaves the device (b200_groth16_prove_witness).
func (k *Groth16Key) ProveWitness(r1cs *R1CS, w []*big.Int, r, s *big.Int) (piA [3]*big.Int, piB [3][2]*big.Int, piC [3]*big.Int, err error) {
	fw := FlatFr(w, Scalar)
	fr, fs := limbs(nil, r), limbs(nil, s)
	a, b, c := make([]uint64, 12), make([]uint64, 24), make([]uint64, 12)
	rc := C.b200_groth16_prove_witness(k.h, r1cs.h, u64(fw), C.size_t(len(w)), u64(fr), u64(fs), u64(a), u64(b), u64(c))
	if err = check(rc); err != nil {
		return
	}
	return G1FromLimbs(a), G2FromLimbs(b), G1FromLimbs(c), nil
}

// ProveWitnessBatch is ProveWitness for k witnesses of one circuit in one call (b200_groth16_prove_witness_batch):
// proof p is ProveWitness(r1cs, ws[p], rs[p], ss[p]).  Worth it for small circuits proved many times.  On a
// LoadGroth16Shard key it works after CommInit, SPMD: every rank passes the same witnesses and r, s, computes its part
// of the k proofs, and receives all k proofs after one all-gather.
func (k *Groth16Key) ProveWitnessBatch(r1cs *R1CS, ws [][]*big.Int, rs, ss []*big.Int) (piA [][3]*big.Int, piB [][3][2]*big.Int, piC [][3]*big.Int, err error) {
	n := len(ws)
	if n == 0 || len(rs) != n || len(ss) != n {
		return nil, nil, nil, errors.New("b200: ProveWitnessBatch needs k >= 1 witnesses and k r, s")
	}
	var fw, fr, fs []uint64
	for p := 0; p < n; p++ {
		if len(ws[p]) != len(ws[0]) {
			return nil, nil, nil, errors.New("b200: ProveWitnessBatch: witnesses of different lengths")
		}
		fw = append(fw, FlatFr(ws[p], Scalar)...)
		fr = append(fr, limbs(nil, rs[p])...)
		fs = append(fs, limbs(nil, ss[p])...)
	}
	a, b, c := make([]uint64, 12*n), make([]uint64, 24*n), make([]uint64, 12*n)
	rc := C.b200_groth16_prove_witness_batch(k.h, r1cs.h, u64(fw), C.size_t(len(ws[0])), C.size_t(n), u64(fr), u64(fs), u64(a), u64(b), u64(c))
	if err = check(rc); err != nil {
		return
	}
	for p := 0; p < n; p++ {
		piA = append(piA, G1FromLimbs(a[12*p:12*p+12]))
		piB = append(piB, G2FromLimbs(b[24*p:24*p+24]))
		piC = append(piC, G1FromLimbs(c[12*p:12*p+12]))
	}
	return
}

// ---- snark.GenerateProofs (Pinocchio) fed from the witness -------------------------------------------------------------
// PinocchioKey is a snark.Pk resident on the device (b200_pinocchio_pk_load).
type PinocchioKey struct{ h C.b200_pk_t }

// PinocchioProof is snark.Proof (snark.go:38-47).
type PinocchioProof struct {
	PiA, PiAp, PiBp, PiC, PiCp, PiH, PiKp [3]*big.Int
	PiB                                   [3][2]*big.Int
}

// LoadPinocchio uploads snark.Pk: a, ap, bp, c, cp, kp and b (G2) hold one point per signal.
func LoadPinocchio(a, ap [][3]*big.Int, b [][3][2]*big.Int, bp, c, cp, kp, g1t [][3]*big.Int, z []*big.Int, nPublic int) (*PinocchioKey, error) {
	k := &PinocchioKey{}
	rc := C.b200_pinocchio_pk_load(u64(FlatG1(a)), u64(FlatG1(ap)), u64(FlatG2(b)), u64(FlatG1(bp)), u64(FlatG1(c)),
		u64(FlatG1(cp)), u64(FlatG1(kp)), C.size_t(len(a)), u64(FlatG1(g1t)), C.size_t(len(g1t)), u64(FlatFr(z, Coeff)),
		C.size_t(len(z)), C.size_t(nPublic), 0, &k.h)
	if err := check(rc); err != nil {
		return nil, err
	}
	return k, nil
}

// LoadPinocchioShard loads rank `rank` of a `world`-way shard of a Pinocchio key (b200_pinocchio_pk_load_shard): whole
// MSMs are dealt to the ranks.  After CommInit, ProveWitness and ProveWitnessBatch on it are SPMD calls that return the
// whole proofs on every rank.
func LoadPinocchioShard(a, ap [][3]*big.Int, b [][3][2]*big.Int, bp, c, cp, kp, g1t [][3]*big.Int, z []*big.Int, nPublic,
	rank, world int) (*PinocchioKey, error) {
	k := &PinocchioKey{}
	rc := C.b200_pinocchio_pk_load_shard(u64(FlatG1(a)), u64(FlatG1(ap)), u64(FlatG2(b)), u64(FlatG1(bp)), u64(FlatG1(c)),
		u64(FlatG1(cp)), u64(FlatG1(kp)), C.size_t(len(a)), u64(FlatG1(g1t)), C.size_t(len(g1t)), u64(FlatFr(z, Coeff)),
		C.size_t(len(z)), C.size_t(nPublic), 0, C.int(rank), C.int(world), &k.h)
	if err := check(rc); err != nil {
		return nil, err
	}
	return k, nil
}

func (k *PinocchioKey) Free() { C.b200_pk_free(k.h) }

func pinocchioProof(g1, b []uint64) *PinocchioProof {
	pt := func(i int) [3]*big.Int { return G1FromLimbs(g1[12*i : 12*i+12]) }
	return &PinocchioProof{PiA: pt(0), PiAp: pt(1), PiBp: pt(2), PiC: pt(3), PiCp: pt(4), PiH: pt(5), PiKp: pt(6), PiB: G2FromLimbs(b)}
}

// ProveWitness is snark.GenerateProofs fed from the witness: px never leaves the device (b200_pinocchio_prove_witness).
func (k *PinocchioKey) ProveWitness(r1cs *R1CS, w []*big.Int) (*PinocchioProof, error) {
	fw := FlatFr(w, Scalar)
	g1, b := make([]uint64, 84), make([]uint64, 24)
	rc := C.b200_pinocchio_prove_witness(k.h, r1cs.h, u64(fw), C.size_t(len(w)), u64(g1), u64(b))
	if err := check(rc); err != nil {
		return nil, err
	}
	return pinocchioProof(g1, b), nil
}

// ProveWitnessBatch is ProveWitness for k witnesses of one circuit in one call (b200_pinocchio_prove_witness_batch):
// proof p is ProveWitness(r1cs, ws[p]).  Worth it for small circuits proved many times.  On a LoadPinocchioShard key
// it works after CommInit, SPMD: every rank passes the same witnesses and receives all k proofs after one all-gather.
func (k *PinocchioKey) ProveWitnessBatch(r1cs *R1CS, ws [][]*big.Int) ([]*PinocchioProof, error) {
	n := len(ws)
	if n == 0 {
		return nil, errors.New("b200: ProveWitnessBatch needs k >= 1 witnesses")
	}
	var fw []uint64
	for p := 0; p < n; p++ {
		if len(ws[p]) != len(ws[0]) {
			return nil, errors.New("b200: ProveWitnessBatch: witnesses of different lengths")
		}
		fw = append(fw, FlatFr(ws[p], Scalar)...)
	}
	g1, b := make([]uint64, 84*n), make([]uint64, 24*n)
	rc := C.b200_pinocchio_prove_witness_batch(k.h, r1cs.h, u64(fw), C.size_t(len(ws[0])), C.size_t(n), u64(g1), u64(b))
	if err := check(rc); err != nil {
		return nil, err
	}
	proofs := make([]*PinocchioProof, n)
	for p := range proofs {
		proofs[p] = pinocchioProof(g1[84*p:84*p+84], b[24*p:24*p+24])
	}
	return proofs, nil
}

// ---- multi-GPU: one process per GPU, NCCL inside the library ----------------------------------------------------------
// Rank 0 calls CommUniqueID and hands the 128 bytes to the other ranks (any side channel); every rank calls CommInit after
// choosing its device, loads its shard with LoadGroth16Shard, and then calls key.Prove with the SAME w, px, r, s: the
// proof comes back on every rank.
func CommUniqueID() (id [128]byte, err error) {
	err = check(C.b200_comm_unique_id((*C.uint8_t)(unsafe.Pointer(&id[0]))))
	return
}
func CommInit(id [128]byte, rank, world int) error {
	return check(C.b200_comm_init((*C.uint8_t)(unsafe.Pointer(&id[0])), C.int(rank), C.int(world)))
}
func CommDestroy() error { return check(C.b200_comm_destroy()) }

// TuneShardsForTwoInFlight sets the partition of sharded keys loaded AFTERWARDS the way bench.py does when it keeps two
// proofs in flight (LoadGroth16Pair on every rank): every shard on the batched-affine tree, an A / B1 term 0.85 and a G2
// term 2.75 of a C||PTD term.  The defaults suit one proof at a time.
func TuneShardsForTwoInFlight() error {
	for _, kv := range [][2]C.int{{C.B200_CFG_SHARD_AFFINE_MIN_G1, 1}, {C.B200_CFG_SHARD_AFFINE_MIN_G2, 1},
		{C.B200_CFG_SHARD_W_AB, 85}, {C.B200_CFG_SHARD_W_G2, 275}} {
		if err := check(C.b200_config(kv[0], kv[1])); err != nil {
			return err
		}
	}
	return nil
}

func LoadGroth16Shard(at, b1 [][3]*big.Int, b2 [][3][2]*big.Int, bacDelta, ptd [][3]*big.Int, z []*big.Int,
	alpha1, beta1, delta1 [3]*big.Int, beta2, delta2 [3][2]*big.Int, nVars, nPublic, rank, world int) (*Groth16Key, error) {
	fa, fb1, fb2, fc, fp := FlatG1(at[:nVars]), FlatG1(b1[:nVars]), FlatG2(b2[:nVars]), FlatG1(bacDelta[:nVars]), FlatG1(ptd)
	fz := FlatFr(z, Coeff)
	a1, be1, d1 := FlatG1([][3]*big.Int{alpha1}), FlatG1([][3]*big.Int{beta1}), FlatG1([][3]*big.Int{delta1})
	be2, d2 := FlatG2([][3][2]*big.Int{beta2}), FlatG2([][3][2]*big.Int{delta2})
	var k Groth16Key
	rc := C.b200_groth16_pk_load_shard(u64(fa), u64(fb1), u64(fb2), u64(fc), C.size_t(nVars), u64(fp), C.size_t(len(ptd)),
		u64(fz), C.size_t(len(z)), u64(a1), u64(be1), u64(d1), u64(be2), u64(d2), C.size_t(nPublic), 0,
		C.int(rank), C.int(world), &k.h)
	return &k, check(rc)
}

// ---- trusted setup from the sparse R1CS (b200_groth16_setup, b200_pinocchio_setup) --------------------------------------
// groth16.GenerateTrustedSetup / snark.GenerateTrustedSetup at any size: the dense alphas / betas / gammas they take are
// m x n matrices and cannot exist beyond a few thousand constraints.  Points are affine (x, y, 1) with infinity all zero:
// the same group elements as the reference's for the same toxic values, not its Jacobian representatives.

func g1s(w []uint64) [][3]*big.Int {
	out := make([][3]*big.Int, len(w)/12)
	for i := range out {
		out[i] = G1FromLimbs(w[12*i : 12*i+12])
	}
	return out
}
func g2s(w []uint64) [][3][2]*big.Int {
	out := make([][3][2]*big.Int, len(w)/24)
	for i := range out {
		out[i] = G2FromLimbs(w[24*i : 24*i+24])
	}
	return out
}
func frs(w []uint64) []*big.Int {
	out := make([]*big.Int, len(w)/4)
	for i := range out {
		out[i] = fromLimbs(w[4*i : 4*i+4])
	}
	return out
}

// Groth16Setup holds groth16.Pk and Vk in the shapes LoadGroth16 and the verifier take.
type Groth16Setup struct {
	At, B1, BACDelta, PowersTauDelta, IC [][3]*big.Int
	B2                                   [][3][2]*big.Int
	Z                                    []*big.Int
	Alpha1, Beta1, Delta1                [3]*big.Int
	Beta2, Gamma2, Delta2                [3][2]*big.Int
}

// Groth16Setup is groth16.GenerateTrustedSetup (groth16/groth16.go:94-222) on this R1CS.  toxic = T, Kalpha, Kbeta,
// Kgamma, Kdelta, each < r.
func (r *R1CS) Groth16Setup(nPublic int, toxic [5]*big.Int) (*Groth16Setup, error) {
	var tox []uint64
	for _, t := range toxic {
		tox = limbs(tox, t)
	}
	m := r.M
	at, b1, cd, b2 := make([]uint64, 12*m), make([]uint64, 12*m), make([]uint64, 12*m), make([]uint64, 24*m)
	ptd, z, ic := make([]uint64, 12*(m-1)), make([]uint64, 4*(m-1)), make([]uint64, 12*(nPublic+1))
	a1, be1, d1 := make([]uint64, 12), make([]uint64, 12), make([]uint64, 12)
	be2, g2, d2 := make([]uint64, 24), make([]uint64, 24), make([]uint64, 24)
	rc := C.b200_groth16_setup(r.h, C.size_t(nPublic), u64(tox), u64(at), u64(b1), u64(b2), u64(cd), u64(ptd), u64(z),
		u64(a1), u64(be1), u64(d1), u64(be2), u64(g2), u64(d2), u64(ic))
	if err := check(rc); err != nil {
		return nil, err
	}
	return &Groth16Setup{At: g1s(at), B1: g1s(b1), BACDelta: g1s(cd), PowersTauDelta: g1s(ptd), IC: g1s(ic), B2: g2s(b2),
		Z: frs(z), Alpha1: G1FromLimbs(a1), Beta1: G1FromLimbs(be1), Delta1: G1FromLimbs(d1), Beta2: G2FromLimbs(be2),
		Gamma2: G2FromLimbs(g2), Delta2: G2FromLimbs(d2)}, nil
}

// PinocchioSetup holds snark.Pk and Vk (IC = A[0..nPublic]).
type PinocchioSetup struct {
	A, Ap, Bp, C, Cp, Kp, G1T, IC [][3]*big.Int
	B                             [][3][2]*big.Int
	Z                             []*big.Int
	Vkb, G1Kbg                    [3]*big.Int
	Vka, Vkc, G2Kbg, G2Kg, Vkz    [3][2]*big.Int
}

// PinocchioSetup is snark.GenerateTrustedSetup (snark.go:98-251) on this R1CS.  toxic = T, Ka, Kb, Kc, Kbeta, Kgamma,
// RhoA, RhoB, each < r.
func (r *R1CS) PinocchioSetup(nPublic int, toxic [8]*big.Int) (*PinocchioSetup, error) {
	var tox []uint64
	for _, t := range toxic {
		tox = limbs(tox, t)
	}
	m := r.M
	g1 := make([][]uint64, 6)
	for k := range g1 {
		g1[k] = make([]uint64, 12*m)
	}
	b2, g1t, z := make([]uint64, 24*m), make([]uint64, 12*(m-1)), make([]uint64, 4*(m-1))
	vk1, vk2 := make([]uint64, 24), make([]uint64, 120)
	rc := C.b200_pinocchio_setup(r.h, C.size_t(nPublic), u64(tox), u64(g1[0]), u64(g1[1]), u64(b2), u64(g1[2]), u64(g1[3]),
		u64(g1[4]), u64(g1[5]), u64(g1t), u64(z), u64(vk1), u64(vk2))
	if err := check(rc); err != nil {
		return nil, err
	}
	s := &PinocchioSetup{A: g1s(g1[0]), Ap: g1s(g1[1]), Bp: g1s(g1[2]), C: g1s(g1[3]), Cp: g1s(g1[4]), Kp: g1s(g1[5]),
		G1T: g1s(g1t), B: g2s(b2), Z: frs(z), Vkb: G1FromLimbs(vk1[:12]), G1Kbg: G1FromLimbs(vk1[12:]),
		Vka: G2FromLimbs(vk2[:24]), Vkc: G2FromLimbs(vk2[24:48]), G2Kbg: G2FromLimbs(vk2[48:72]),
		G2Kg: G2FromLimbs(vk2[72:96]), Vkz: G2FromLimbs(vk2[96:])}
	s.IC = s.A[:nPublic+1]
	return s, nil
}

// Groth16Vk holds the verification key of a setup made straight into a resident key: the Vk fields Groth16Setup fills.
type Groth16Vk struct {
	IC                    [][3]*big.Int
	Alpha1                [3]*big.Int
	Beta2, Gamma2, Delta2 [3][2]*big.Int
}

// Groth16SetupKey is Groth16Setup followed by LoadGroth16Shard(.., windowBits, rank, world) in one call
// (b200_groth16_setup_pk): the key is minted on the device straight into its tables and no CRS passes through host
// memory; a rank mints only the part it holds.  Every rank must pass the same toxic values.
func (r *R1CS) Groth16SetupKey(nPublic int, toxic [5]*big.Int, windowBits, rank, world int) (*Groth16Key, Groth16Vk, error) {
	var tox []uint64
	for _, t := range toxic {
		tox = limbs(tox, t)
	}
	a1, be2, g2, d2, ic := make([]uint64, 12), make([]uint64, 24), make([]uint64, 24), make([]uint64, 24), make([]uint64, 12*(nPublic+1))
	var h C.b200_pk_t
	rc := C.b200_groth16_setup_pk(r.h, C.size_t(nPublic), u64(tox), C.int(windowBits), C.int(rank), C.int(world), &h,
		u64(a1), u64(be2), u64(g2), u64(d2), u64(ic))
	if err := check(rc); err != nil {
		return nil, Groth16Vk{}, err
	}
	return &Groth16Key{h}, Groth16Vk{IC: g1s(ic), Alpha1: G1FromLimbs(a1), Beta2: G2FromLimbs(be2), Gamma2: G2FromLimbs(g2),
		Delta2: G2FromLimbs(d2)}, nil
}

// PinocchioVk holds the verification key of a setup made straight into a resident key: the Vk fields PinocchioSetup
// fills (IC = A[0..nPublic]).
type PinocchioVk struct {
	IC                         [][3]*big.Int
	Vkb, G1Kbg                 [3]*big.Int
	Vka, Vkc, G2Kbg, G2Kg, Vkz [3][2]*big.Int
}

// PinocchioSetupKey is PinocchioSetup followed by LoadPinocchioShard(.., windowBits, rank, world) in one call
// (b200_pinocchio_setup_pk).  Every rank must pass the same toxic values.
func (r *R1CS) PinocchioSetupKey(nPublic int, toxic [8]*big.Int, windowBits, rank, world int) (*PinocchioKey, PinocchioVk, error) {
	var tox []uint64
	for _, t := range toxic {
		tox = limbs(tox, t)
	}
	vk1, vk2, ic := make([]uint64, 24), make([]uint64, 120), make([]uint64, 12*(nPublic+1))
	var h C.b200_pk_t
	rc := C.b200_pinocchio_setup_pk(r.h, C.size_t(nPublic), u64(tox), C.int(windowBits), C.int(rank), C.int(world), &h,
		u64(vk1), u64(vk2), u64(ic))
	if err := check(rc); err != nil {
		return nil, PinocchioVk{}, err
	}
	return &PinocchioKey{h}, PinocchioVk{IC: g1s(ic), Vkb: G1FromLimbs(vk1[:12]), G1Kbg: G1FromLimbs(vk1[12:]),
		Vka: G2FromLimbs(vk2[:24]), Vkc: G2FromLimbs(vk2[24:48]), G2Kbg: G2FromLimbs(vk2[48:72]), G2Kg: G2FromLimbs(vk2[72:96]),
		Vkz: G2FromLimbs(vk2[96:])}, nil
}
