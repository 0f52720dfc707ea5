// k2pow.go — cgo bindings for the RandomX k2pow entry points of libb200post.so (include/b200post_k2pow.h).
// SOURCE-ONLY (no Go toolchain in the build image); mirrors go-spacemesh_b200/k2pow.py, which the tests exercise.
// Where it stands in the reference: the proof-of-work the post-service computes before the proving scan
// (activation/nipost.go:171, PostProvingOpts.RandomXMode activation/post.go:64-81) and the check inside
// verifying.ProofVerifier.Verify (activation/post_verifier.go:159).
package b200post

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../.. -lb200post -Wl,-rpath,${SRCDIR}/../..
#include <stdlib.h>
#include <string.h>
#include "b200post_k2pow.h"
*/
import "C"

import (
	"context"
	"sync/atomic"
	"unsafe"
)

// K2powNotFound is returned as the nonce when no pow in the searched range meets the difficulty.
const K2powNotFound = ^uint64(0)

// K2powParams names one search: pow[0:7] ‖ nonce_group ‖ challenge[0:8] ‖ node_id is hashed under CacheKey
// (nil = "spacemesh-randomx-cache-key") and compared with Difficulty (already divided by the number of units).
type K2powParams struct {
	CacheKey   []byte
	NonceGroup uint8
	Challenge8 [8]byte
	NodeID     [32]byte
	Difficulty [32]byte
}

// ScaleDifficulty = PowDifficulty / numUnits as 256-bit big-endian integers (activation/post_types.go:11-38 holds the
// configured value; the division by units is post-rs's).
func ScaleDifficulty(powDifficulty [32]byte, numUnits uint32) (out [32]byte) {
	C.b200post_k2pow_scale_difficulty((*C.uint8_t)(unsafe.Pointer(&powDifficulty[0])), C.uint32_t(numUnits),
		(*C.uint8_t)(unsafe.Pointer(&out[0])))
	return out
}

// cParams builds the C struct in C memory: it holds a pointer (cache_key), and the cgo rules forbid passing Go memory
// that itself contains Go pointers.  The caller frees with the returned func.
func (p *K2powParams) cParams() (*C.b200post_k2pow_params, func()) {
	c := (*C.b200post_k2pow_params)(C.calloc(1, C.size_t(unsafe.Sizeof(C.b200post_k2pow_params{}))))
	var key unsafe.Pointer
	if len(p.CacheKey) > 0 {
		key = C.CBytes(p.CacheKey)
		c.cache_key, c.cache_key_len = (*C.uint8_t)(key), C.size_t(len(p.CacheKey))
	}
	c.nonce_group = C.uint8_t(p.NonceGroup)
	C.memcpy(unsafe.Pointer(&c.challenge8[0]), unsafe.Pointer(&p.Challenge8[0]), 8)
	C.memcpy(unsafe.Pointer(&c.node_id[0]), unsafe.Pointer(&p.NodeID[0]), 32)
	C.memcpy(unsafe.Pointer(&c.difficulty[0]), unsafe.Pointer(&p.Difficulty[0]), 32)
	return c, func() {
		if key != nil {
			C.free(key)
		}
		C.free(unsafe.Pointer(c))
	}
}

// cancelFlag returns a C int that becomes 1 when ctx is done (the library polls it between device batches, the way
// Initialize polls ctx at activation/post.go:301-304) and a func that stops the watcher and frees the flag.
func cancelFlag(ctx context.Context) (*C.int, func()) {
	flag := (*C.int)(C.calloc(1, C.size_t(unsafe.Sizeof(C.int(0)))))
	done := make(chan struct{})
	stopped := make(chan struct{})
	go func() {
		defer close(stopped)
		select {
		case <-ctx.Done():
			atomic.StoreInt32((*int32)(unsafe.Pointer(flag)), 1) // the library reads the flag as `const volatile int *`
			<-done
		case <-done:
		}
	}()
	return flag, func() { close(done); <-stopped; C.free(unsafe.Pointer(flag)) }
}

// K2powSearch looks for the smallest valid pow in [start, start+count) on the given providers (one device: the range
// is walked in device batches; several: batches are interleaved over the devices, no collective — nonces are
// independent).  Returns K2powNotFound if the range holds none, and the number of hashes computed.
func K2powSearch(ctx context.Context, providers []uint32, p *K2powParams, start, count uint64) (pow uint64, hashes uint64, err error) {
	if len(providers) == 0 {
		return K2powNotFound, 0, ErrNoProvider
	}
	cp, free := p.cParams()
	defer free()
	flag, stop := cancelFlag(ctx)
	defer stop()
	var found, done C.uint64_t
	provs := (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&providers[0])), 4*len(providers))))
	defer C.free(unsafe.Pointer(provs))
	err = statusErr(checked(func() C.int {
		if len(providers) == 1 {
			return C.b200post_k2pow_search(C.uint32_t(providers[0]), cp, C.uint64_t(start), C.uint64_t(count), &found, &done, flag)
		}
		return C.b200post_k2pow_search_multi(provs, C.int(len(providers)), cp, C.uint64_t(start), C.uint64_t(count), &found, &done, flag)
	}))
	if err != nil {
		return K2powNotFound, uint64(done), err
	}
	return uint64(found), uint64(done), nil
}

// K2powSearchGroups is what a prover needs: the smallest valid pow of every nonce group 0..groups-1
// (Nonces/16 groups, activation/post.go:64-81), all groups sharing device batches.
func K2powSearchGroups(ctx context.Context, provider uint32, p *K2powParams, groups uint32, maxNoncesPerGroup uint64) ([]uint64, error) {
	if groups == 0 {
		return nil, nil
	}
	cp, free := p.cParams()
	defer free()
	flag, stop := cancelFlag(ctx)
	defer stop()
	pows := (*C.uint64_t)(C.calloc(C.size_t(groups), 8))
	defer C.free(unsafe.Pointer(pows))
	if err := statusErr(checked(func() C.int {
		return C.b200post_k2pow_search_groups(C.uint32_t(provider), cp, C.uint32_t(groups), C.uint64_t(maxNoncesPerGroup), pows, nil, flag)
	})); err != nil {
		return nil, err
	}
	out := make([]uint64, groups)
	copy(out, unsafe.Slice((*uint64)(unsafe.Pointer(pows)), groups))
	return out, nil
}

// K2powSearchGroupsOn is K2powSearchGroups over several devices (repeats allowed): windows of nonces go to the devices
// from one shared cursor, and the result is exactly the one-device result (the smallest valid pow of every group).
func K2powSearchGroupsOn(ctx context.Context, providers []uint32, p *K2powParams, groups uint32, maxNoncesPerGroup uint64) ([]uint64, error) {
	if len(providers) == 0 {
		return nil, ErrNoProvider
	}
	if groups == 0 {
		return nil, nil
	}
	cp, free := p.cParams()
	defer free()
	flag, stop := cancelFlag(ctx)
	defer stop()
	provs := (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&providers[0])), 4*len(providers))))
	defer C.free(unsafe.Pointer(provs))
	pows := (*C.uint64_t)(C.calloc(C.size_t(groups), 8))
	defer C.free(unsafe.Pointer(pows))
	if err := statusErr(checked(func() C.int {
		return C.b200post_k2pow_search_groups_multi(provs, C.int(len(providers)), cp, C.uint32_t(groups), C.uint64_t(maxNoncesPerGroup), pows, nil, flag)
	})); err != nil {
		return nil, err
	}
	out := make([]uint64, groups)
	copy(out, unsafe.Slice((*uint64)(unsafe.Pointer(pows)), groups))
	return out, nil
}

// K2powVerify is the verifier's check of one proof's pow (the batched verifier does the same for a whole batch in one
// device launch; this entry point is for callers that hold a single pow).
func K2powVerify(provider uint32, p *K2powParams, pow uint64) (bool, error) {
	cp, free := p.cParams()
	defer free()
	var valid C.int
	if err := statusErr(checked(func() C.int {
		return C.b200post_k2pow_verify(C.uint32_t(provider), cp, C.uint64_t(pow), &valid)
	})); err != nil {
		return false, err
	}
	return valid != 0, nil
}

// RandomxHash computes RandomX hashes of equally long inputs under key (RandomX's published vectors run through it).
func RandomxHash(provider uint32, key []byte, inputs [][]byte) ([][32]byte, error) {
	if len(inputs) == 0 {
		return nil, nil
	}
	n, l := len(inputs), len(inputs[0])
	flat := make([]byte, 0, n*l)
	for _, in := range inputs {
		if len(in) != l {
			return nil, ErrUnsupported // one launch hashes inputs of one length
		}
		flat = append(flat, in...)
	}
	ck, ci := C.CBytes(key), C.CBytes(flat)
	defer C.free(ck)
	defer C.free(ci)
	out := C.calloc(C.size_t(n), 32)
	defer C.free(out)
	if err := statusErr(checked(func() C.int {
		return C.b200post_randomx_hash(C.uint32_t(provider), (*C.uint8_t)(ck), C.size_t(len(key)), (*C.uint8_t)(ci), C.size_t(l), C.size_t(n), (*C.uint8_t)(out))
	})); err != nil {
		return nil, err
	}
	res := make([][32]byte, n)
	copy(unsafe.Slice((*byte)(unsafe.Pointer(&res[0])), 32*n), unsafe.Slice((*byte)(out), 32*n))
	return res, nil
}

// K2powJob is one k2pow of a job search: any identity, challenge and nonce group, with its own difficulty (the
// PowDifficulty divided by that identity's NumUnits, ScaleDifficulty).
type K2powJob struct {
	NodeID     [32]byte
	Challenge8 [8]byte
	NonceGroup uint8
	Difficulty [32]byte
}

// K2powSearchJobs runs several identities' k2pows in one search (b200post_k2pow_search_jobs): their windows of
// nonces share device batches.  pows[j] is job j's smallest valid pow below maxNoncesPerJob (0 = the whole nonce space)
// or K2powNotFound, whatever the other jobs and the device list (repeats allowed).  ctx cancels between windows.
func K2powSearchJobs(ctx context.Context, providers []uint32, cacheKey []byte, jobs []K2powJob, maxNoncesPerJob uint64) (pows []uint64, hashes uint64, err error) {
	if len(providers) == 0 {
		return nil, 0, ErrNoProvider
	}
	if len(jobs) == 0 {
		return nil, 0, nil
	}
	cj := (*C.b200post_k2pow_job)(C.calloc(C.size_t(len(jobs)), C.size_t(unsafe.Sizeof(C.b200post_k2pow_job{}))))
	defer C.free(unsafe.Pointer(cj))
	for i, j := range jobs {
		x := &unsafe.Slice(cj, len(jobs))[i]
		C.memcpy(unsafe.Pointer(&x.node_id[0]), unsafe.Pointer(&j.NodeID[0]), 32)
		C.memcpy(unsafe.Pointer(&x.challenge8[0]), unsafe.Pointer(&j.Challenge8[0]), 8)
		x.nonce_group = C.uint8_t(j.NonceGroup)
		C.memcpy(unsafe.Pointer(&x.difficulty[0]), unsafe.Pointer(&j.Difficulty[0]), 32)
	}
	var key unsafe.Pointer
	if cacheKey != nil {
		key = C.CBytes(cacheKey)
		defer C.free(key)
	}
	provs := (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&providers[0])), 4*len(providers))))
	defer C.free(unsafe.Pointer(provs))
	out := (*C.uint64_t)(C.calloc(C.size_t(len(jobs)), 8))
	defer C.free(unsafe.Pointer(out))
	flag, stop := cancelFlag(ctx)
	defer stop()
	var done C.uint64_t
	if err := statusErr(checked(func() C.int {
		return C.b200post_k2pow_search_jobs(provs, C.int(len(providers)), (*C.uint8_t)(key), C.size_t(len(cacheKey)), C.size_t(len(jobs)), cj,
			C.uint64_t(maxNoncesPerJob), out, &done, flag)
	})); err != nil {
		return nil, uint64(done), err
	}
	pows = make([]uint64, len(jobs))
	copy(pows, unsafe.Slice((*uint64)(unsafe.Pointer(out)), len(jobs)))
	return pows, uint64(done), nil
}
