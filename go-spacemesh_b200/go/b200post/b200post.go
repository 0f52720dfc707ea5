// Package b200post binds libb200post.so (include/b200post.h) for go-spacemesh.
//
// SOURCE-ONLY DELIVERABLE: this image has no Go toolchain (`go version` -> not found), so this file has
// never been compiled here.  It is the cgo stub a maintainer adds next to activation/; the C ABI below it
// is exercised end-to-end from tests/ through ctypes with the same call sequence.
//
// It provides what the POST label path of the reference consumes from github.com/spacemeshos/post:
//   - Providers / Benchmark            (activation/post_supervisor.go:105-127)
//   - Initializer.Initialize batches   (activation/post.go:295, 355-361)
//   - label recomputation for Verify   (activation/post_verifier.go:159)
//   - VerifyVRFNonce                   (activation/validation.go:261-282)
package b200post

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../.. -lb200post -Wl,-rpath,${SRCDIR}/../..
#include <stdlib.h>
#include "b200post.h"
*/
import "C"

import (
	"context"
	"errors"
	"fmt"
	"runtime"
	"sync/atomic"
	"unsafe"
)

// Provider mirrors initialization.Provider (ID, Model, DeviceType) — activation/post.go:24.
type Provider struct {
	ID         uint32
	Model      string
	DeviceType int // 2 = GPU; this library never reports a CPU provider
	HBMBytes   uint64
}

// ErrReferenceLabelMismatch-style sentinel errors the activation package switches on.
var (
	ErrNoDevice    = errors.New("b200post: no usable CUDA device")
	ErrUnsupported = errors.New("b200post: provider not served (no CPU path in this library)")
	ErrCancelled   = context.Canceled
)

// checked runs ONE C call and, if it failed, reads b200post_last_error() before the goroutine can move: the error text
// is thread-local in C, and without LockOSThread a second cgo call may land on another OS thread and read a stale or
// empty message.  Every call whose error text matters goes through here.
func checked(call func() C.int) (C.int, string) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	rc := call()
	if rc == C.B200POST_OK {
		return rc, ""
	}
	return rc, C.GoString(C.b200post_last_error())
}

func statusErr(rc C.int, msg string) error {
	switch rc {
	case C.B200POST_OK:
		return nil
	case C.B200POST_ERR_NO_DEVICE:
		return ErrNoDevice
	case C.B200POST_ERR_UNSUPPORTED:
		return ErrUnsupported
	case C.B200POST_ERR_CANCELLED:
		return ErrCancelled
	default:
		return fmt.Errorf("b200post: status %d: %s", int(rc), msg)
	}
}

// Providers lists the GPUs — drop-in for initialization.OpenCLProviders().
func Providers() ([]Provider, error) {
	n := int(C.b200post_providers(nil, 0))
	if n == 0 {
		return nil, nil
	}
	raw := make([]C.b200post_provider, n)
	n = int(C.b200post_providers(&raw[0], C.int(n)))
	out := make([]Provider, n)
	for i := 0; i < n; i++ {
		out[i] = Provider{ID: uint32(raw[i].id), Model: C.GoString(&raw[i].model[0]), DeviceType: int(raw[i].device_class), HBMBytes: uint64(raw[i].hbm_bytes)}
	}
	return out, nil
}

// Benchmark returns labels ("hashes") per second — drop-in for initialization.Benchmark.
func Benchmark(provider uint32, scryptN uint64) (int, error) {
	var v C.double
	if err := statusErr(checked(func() C.int { return C.b200post_benchmark(C.uint32_t(provider), C.uint64_t(scryptN), 2.0, &v) })); err != nil {
		return 0, err
	}
	return int(v), nil
}

// CommitmentBytes = blake3(nodeID || commitmentATX) (oracle.CommitmentBytes upstream).
func CommitmentBytes(nodeID, commitmentAtxID []byte) [32]byte {
	var out [32]byte
	C.b200post_commitment((*C.uint8_t)(unsafe.Pointer(&nodeID[0])), (*C.uint8_t)(unsafe.Pointer(&commitmentAtxID[0])), (*C.uint8_t)(unsafe.Pointer(&out[0])))
	return out
}

// VRFNonce is the result of the arg-min scan over a range.
type VRFNonce struct {
	Index   uint64
	Label32 [32]byte
}

// InitializeRange computes labels [start, start+count) into out (16 bytes per label; nil = discard) and,
// when difficulty != nil, the VRF nonce candidate of the range.  ctx cancellation is polled between layers
// (mirrors the `errors.Is(err, context.Canceled)` branch at activation/post.go:301).
func InitializeRange(ctx context.Context, provider uint32, commitment [32]byte, scryptN, start, count uint64, out []byte, difficulty []byte) (*VRFNonce, error) {
	if out != nil && uint64(len(out)) < 16*count {
		return nil, errors.New("b200post: output buffer too small")
	}
	var cancel int32
	done := make(chan struct{})
	defer close(done)
	go func() {
		select {
		case <-ctx.Done():
			atomic.StoreInt32(&cancel, 1)
		case <-done:
		}
	}()
	var outPtr *C.uint8_t
	if out != nil && count > 0 {
		outPtr = (*C.uint8_t)(unsafe.Pointer(&out[0]))
	}
	var diffPtr *C.uint8_t
	var nonce C.b200post_vrf_nonce
	noncePtr := (*C.b200post_vrf_nonce)(nil)
	if difficulty != nil {
		diffPtr = (*C.uint8_t)(unsafe.Pointer(&difficulty[0]))
		noncePtr = &nonce
	}
	rc, msg := checked(func() C.int {
		return C.b200post_labels_range(C.uint32_t(provider), (*C.uint8_t)(unsafe.Pointer(&commitment[0])), C.uint64_t(scryptN),
		C.uint64_t(start), C.uint64_t(count), outPtr, diffPtr, noncePtr, (*C.int)(unsafe.Pointer(&cancel)))
	})
	if err := statusErr(rc, msg); err != nil {
		return nil, err
	}
	if difficulty == nil || nonce.found == 0 {
		return nil, nil
	}
	res := &VRFNonce{Index: uint64(nonce.index)}
	copy(res.Label32[:], C.GoBytes(unsafe.Pointer(&nonce.label32[0]), 32))
	return res, nil
}

// LabelsGather recomputes labels at scattered (commitment, index) pairs — the K2/K3 label recomputation
// inside verifying.ProofVerifier.Verify.  commitments is n x 32 bytes.
func LabelsGather(provider uint32, commitments []byte, indices []uint64, scryptN uint64) ([]byte, error) {
	n := len(indices)
	if len(commitments) != 32*n {
		return nil, errors.New("b200post: commitments must be 32 bytes per index")
	}
	out := make([]byte, 16*n)
	if n == 0 {
		return out, nil
	}
	rc, msg := checked(func() C.int {
		return C.b200post_labels_gather(C.uint32_t(provider), C.size_t(n), (*C.uint8_t)(unsafe.Pointer(&commitments[0])),
		(*C.uint64_t)(unsafe.Pointer(&indices[0])), C.uint64_t(scryptN), (*C.uint8_t)(unsafe.Pointer(&out[0])))
	})
	return out, statusErr(rc, msg)
}

// LabelsGatherIndexed is LabelsGather for items that share few commitments (one identity checked at K2
// indices): commitments is m x 32 bytes and item i uses row rows[i].
func LabelsGatherIndexed(provider uint32, commitments []byte, rows []uint32, indices []uint64, scryptN uint64) ([]byte, error) {
	n := len(indices)
	if len(rows) != n || len(commitments)%32 != 0 {
		return nil, errors.New("b200post: one row per index and 32 bytes per commitment")
	}
	out := make([]byte, 16*n)
	if n == 0 {
		return out, nil
	}
	if len(commitments) == 0 {
		return nil, errors.New("b200post: no commitments")
	}
	rc, msg := checked(func() C.int {
		return C.b200post_labels_gather_indexed(C.uint32_t(provider), C.size_t(n), C.size_t(len(commitments)/32),
		(*C.uint8_t)(unsafe.Pointer(&commitments[0])), (*C.uint32_t)(unsafe.Pointer(&rows[0])),
		(*C.uint64_t)(unsafe.Pointer(&indices[0])), C.uint64_t(scryptN), (*C.uint8_t)(unsafe.Pointer(&out[0])))
	})
	return out, statusErr(rc, msg)
}

// VerifyVRFNonce is the drop-in for verifying.VerifyVRFNonce (activation/validation.go:277).
func VerifyVRFNonce(provider uint32, nonce uint64, nodeID, commitmentAtxID []byte, numUnits uint32, labelsPerUnit, scryptN uint64) (bool, error) {
	var valid C.int
	rc, msg := checked(func() C.int {
		return C.b200post_verify_vrf_nonce(C.uint32_t(provider), C.uint64_t(nonce), (*C.uint8_t)(unsafe.Pointer(&nodeID[0])),
		(*C.uint8_t)(unsafe.Pointer(&commitmentAtxID[0])), C.uint32_t(numUnits), C.uint64_t(labelsPerUnit), C.uint64_t(scryptN), &valid)
	})
	return valid != 0, statusErr(rc, msg)
}
