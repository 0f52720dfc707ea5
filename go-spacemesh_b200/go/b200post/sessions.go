// sessions.go — cgo bindings for the setup manager, the batched verifier and the prover of libb200post.so.
// SOURCE-ONLY (no Go toolchain in the build image); mirrors the ctypes layer the tests exercise
// (go-spacemesh_b200/setup.py, verify.py, prove.py).
package b200post

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../.. -lb200post -Wl,-rpath,${SRCDIR}/../..
#include <stdlib.h>
#include "b200post_setup.h"
#include "b200post_verify.h"
#include "b200post_prove.h"
*/
import "C"

import (
	"context"
	"errors"
	"fmt"
	"sync/atomic"
	"unsafe"
)

// ---------------------------------------------------------------------------------------------------------
// PostSetupManager backend (activation/post.go:185-449; interface postSetupProvider, interface.go:114-119)
// ---------------------------------------------------------------------------------------------------------

// PostSetupState has the reference's values (activation/post.go:128-137).
type PostSetupState int32

const (
	PostSetupStateNotStarted PostSetupState = 1 + iota
	PostSetupStatePrepared
	PostSetupStateInProgress
	PostSetupStateStopped
	PostSetupStateComplete
	PostSetupStateError
)

var (
	ErrNotPrepared      = errors.New("post session not prepared")        // activation/post.go:277
	ErrSessionInProgess = errors.New("post setup session in progress")   // activation/post.go:345
	ErrNoProvider       = errors.New("no provider specified")            // activation/post_test.go:113
	ErrLabelMismatch    = errors.New("reference label mismatch")         // initialization.ErrReferenceLabelMismatch
	ErrConfigMismatch   = errors.New("post data belongs to another identity or configuration")
	ErrInvalidPow       = errors.New("invalid k2pow")
)

type SetupConfig struct { // PostConfig (activation/post.go:27-38)
	MinNumUnits, MaxNumUnits uint32
	LabelsPerUnit            uint64
	K1, K2, K3               uint32
	PowDifficulty            [32]byte
}

type SetupOpts struct { // PostSetupOpts (activation/post.go:53-61)
	DataDir          string
	NumUnits         uint32
	MaxFileSize      uint64
	ProviderID       *uint32 // nil = not specified; use AllProviders for every GPU of the box
	ScryptN          uint64
	ComputeBatchSize uint64
}

const AllProviders = ^uint32(1) // maps to B200POST_PROVIDER_ALL

type SetupManager struct{ h *C.b200post_setup_manager }

func setupErr(rc C.int, msg string) error {
	switch rc {
	case C.B200POST_OK:
		return nil
	case C.B200POST_ERR_CANCELLED:
		return context.Canceled
	case C.B200POST_ERR_NO_PROVIDER:
		return ErrNoProvider
	case C.B200POST_ERR_LABEL_MISMATCH:
		return ErrLabelMismatch
	case C.B200POST_ERR_CONFIG_MISMATCH:
		return fmt.Errorf("%w: %s", ErrConfigMismatch, msg)
	case C.B200POST_ERR_STATE:
		// msg was read on the OS thread that made the failing call (checked): safe to compare
		switch msg {
		case ErrNotPrepared.Error():
			return ErrNotPrepared
		case ErrSessionInProgess.Error():
			return ErrSessionInProgess
		}
		return errors.New(msg)
	default:
		return statusErr(rc, msg)
	}
}

func NewSetupManager(cfg SetupConfig) (*SetupManager, error) {
	var c C.b200post_post_config
	c.min_num_units, c.max_num_units = C.uint32_t(cfg.MinNumUnits), C.uint32_t(cfg.MaxNumUnits)
	c.labels_per_unit = C.uint64_t(cfg.LabelsPerUnit)
	c.k1, c.k2, c.k3 = C.uint32_t(cfg.K1), C.uint32_t(cfg.K2), C.uint32_t(cfg.K3)
	C.memcpy(unsafe.Pointer(&c.pow_difficulty[0]), unsafe.Pointer(&cfg.PowDifficulty[0]), 32)
	m := &SetupManager{}
	if err := setupErr(checked(func() C.int { return C.b200post_setup_manager_new(&c, &m.h) })); err != nil {
		return nil, err
	}
	return m, nil
}

// PrepareInitializer: the commitment ATX is chosen by the caller (activation/post.go:373-435 stays in Go).
func (m *SetupManager) PrepareInitializer(opts SetupOpts, nodeID, commitmentAtxID []byte) error {
	dir := C.CString(opts.DataDir)
	defer C.free(unsafe.Pointer(dir))
	var o C.b200post_setup_opts
	C.b200post_default_setup_opts(&o)
	o.data_dir = dir
	o.num_units = C.uint32_t(opts.NumUnits)
	o.max_file_size = C.uint64_t(opts.MaxFileSize)
	o.scrypt_n, o.scrypt_r, o.scrypt_p = C.uint64_t(opts.ScryptN), 1, 1
	o.compute_batch_size = C.uint64_t(opts.ComputeBatchSize)
	switch {
	case opts.ProviderID == nil:
		o.provider_id = C.B200POST_PROVIDER_UNSET
	case *opts.ProviderID == AllProviders:
		o.provider_id = C.B200POST_PROVIDER_ALL
	default:
		o.provider_id = C.int64_t(*opts.ProviderID)
	}
	return setupErr(checked(func() C.int {
		return C.b200post_setup_prepare_initializer(m.h, &o, (*C.uint8_t)(unsafe.Pointer(&nodeID[0])), (*C.uint8_t)(unsafe.Pointer(&commitmentAtxID[0])))
	}))
}

// StartSession blocks until the data is complete, ctx is cancelled (context.Canceled, state Stopped) or an error.
func (m *SetupManager) StartSession(ctx context.Context) error {
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
	return setupErr(checked(func() C.int {
		return C.b200post_setup_start_session(m.h, (*C.int)(unsafe.Pointer(&cancel)))
	}))
}

func (m *SetupManager) Status() (PostSetupState, uint64) {
	var st C.b200post_setup_status
	C.b200post_setup_get_status(m.h, &st)
	return PostSetupState(st.state), uint64(st.num_labels_written)
}

func (m *SetupManager) Reset() error { return setupErr(checked(func() C.int { return C.b200post_setup_reset(m.h) })) }
func (m *SetupManager) Close()       { C.b200post_setup_manager_free(m.h) }

// ---------------------------------------------------------------------------------------------------------
// PostVerifier backend (activation/interface.go:26-29; replaces offloadingPostVerifier + its worker pool)
// ---------------------------------------------------------------------------------------------------------

// ErrInvalidIndex mirrors verifying.ErrInvalidIndex (activation/handler_v1.go:228, handler_v2.go:639).
type ErrInvalidIndex struct{ Index int }

func (e *ErrInvalidIndex) Error() string { return fmt.Sprintf("invalid index: %d", e.Index) }

var ErrVerifierClosed = errors.New("verifier is closed") // activation/post_verifier.go:338,346

type Proof struct { // shared.Proof
	Nonce   uint32
	Indices []byte
	Pow     uint64
}
type ProofMetadata struct { // shared.ProofMetadata (activation/validation.go:193-199)
	NodeId, CommitmentAtxId, Challenge []byte
	NumUnits                           uint32
	LabelsPerUnit                      uint64
}
type VerifyOptions struct {
	Prioritized   bool   // PrioritizedCall()
	SubsetK3      uint32 // verifying.Subset(k3, seed) when > 0
	SubsetSeed    []byte
	SelectedIndex *int // verifying.SelectedIndex(i)
}

type Verifier struct{ h *C.b200post_verifier }

// VerifierOptions: the k2pow policy is explicit.  The zero value runs the RandomX pow check of
// verifying.ProofVerifier.Verify (activation/post_verifier.go:150-160) on the device; SkipPow must be asked for.
type VerifierOptions struct {
	SkipPow        bool
	MaxBatchProofs uint32
}

// NewVerifier = NewPostVerifier (activation/post_verifier.go:191-221) with the builtin k2pow check.
func NewVerifier(provider uint32) (*Verifier, error) { return NewVerifierWith(provider, VerifierOptions{}) }

func NewVerifierWith(provider uint32, o VerifierOptions) (*Verifier, error) {
	v := &Verifier{}
	var co C.b200post_verifier_opts // C struct without Go pointers: may be passed by address
	co.max_batch_proofs = C.uint32_t(o.MaxBatchProofs)
	co.pow_mode = C.B200POST_POW_BUILTIN
	if o.SkipPow {
		co.pow_mode = C.B200POST_POW_SKIP
	}
	if err := statusErr(checked(func() C.int { return C.b200post_verifier_new(C.uint32_t(provider), &co, &v.h) })); err != nil {
		return nil, err
	}
	return v, nil
}

// NewVerifierOn builds one verifier over several GPUs: a worker per device drains the same queue.
func NewVerifierOn(providers []uint32) (*Verifier, error) {
	if len(providers) == 0 {
		return nil, errors.New("b200post: no providers")
	}
	v := &Verifier{}
	rc, msg := checked(func() C.int {
		return C.b200post_verifier_new_multi((*C.uint32_t)(unsafe.Pointer(&providers[0])), C.int(len(providers)), nil, &v.h)
	})
	if err := statusErr(rc, msg); err != nil {
		return nil, err
	}
	return v, nil
}

func (v *Verifier) Verify(p *Proof, m *ProofMetadata, k1, k2 uint32, powDifficulty [32]byte, scryptN uint64, o VerifyOptions) error {
	if len(p.Indices) == 0 {
		return errors.New("proof indices are empty")
	}
	// cgo pointer rules: a Go-allocated struct passed to C must not contain Go pointers, so the variable-length inputs
	// (packed indices, subset seed) are copied into C memory for the duration of the call.
	cidx := C.CBytes(p.Indices)
	defer C.free(cidx)
	cp := C.b200post_proof{nonce: C.uint32_t(p.Nonce), indices: (*C.uint8_t)(cidx), indices_len: C.size_t(len(p.Indices)), pow: C.uint64_t(p.Pow)}
	var cm C.b200post_proof_metadata
	C.memcpy(unsafe.Pointer(&cm.node_id[0]), unsafe.Pointer(&m.NodeId[0]), 32)
	C.memcpy(unsafe.Pointer(&cm.commitment_atx_id[0]), unsafe.Pointer(&m.CommitmentAtxId[0]), 32)
	C.memcpy(unsafe.Pointer(&cm.challenge[0]), unsafe.Pointer(&m.Challenge[0]), 32)
	cm.num_units, cm.labels_per_unit = C.uint32_t(m.NumUnits), C.uint64_t(m.LabelsPerUnit)
	cq := C.b200post_verify_params{k1: C.uint32_t(k1), k2: C.uint32_t(k2), scrypt_n: C.uint64_t(scryptN)}
	var co C.b200post_verify_options
	switch {
	case o.SelectedIndex != nil:
		co.mode, co.selected_index = C.B200POST_VERIFY_SELECTED_INDEX, C.uint32_t(*o.SelectedIndex)
	case o.SubsetK3 > 0:
		co.mode, co.k3 = C.B200POST_VERIFY_SUBSET, C.uint32_t(o.SubsetK3)
		if len(o.SubsetSeed) > 0 {
			cseed := C.CBytes(o.SubsetSeed)
			defer C.free(cseed)
			co.seed, co.seed_len = (*C.uint8_t)(cseed), C.size_t(len(o.SubsetSeed))
		}
	}
	if o.Prioritized {
		co.prioritized = 1
	}
	C.memcpy(unsafe.Pointer(&cq.pow_difficulty[0]), unsafe.Pointer(&powDifficulty[0]), 32)
	var bad C.uint64_t
	rc, msg := checked(func() C.int { return C.b200post_verifier_verify(v.h, &cp, &cm, &cq, &co, &bad) })
	switch rc {
	case C.B200POST_OK:
		return nil
	case C.B200POST_ERR_INVALID_PROOF:
		if uint64(bad) == ^uint64(0) {
			return ErrInvalidPow // the k2pow, not a label
		}
		// Index = POSITION in the proof's K2 index list: handler_v1.go:248 stores it as InvalidPostIndexProof.InvalidIdx,
		// malfeasance.go:165 re-verifies it with verifying.SelectedIndex(int(InvalidIdx))
		return &ErrInvalidIndex{Index: int(bad)}
	case C.B200POST_ERR_CLOSED:
		return ErrVerifierClosed
	case C.B200POST_ERR_EMPTY_PROOF:
		return errors.New("proof indices are empty")
	default:
		return statusErr(rc, msg)
	}
}

func (v *Verifier) Close() error { C.b200post_verifier_close(v.h); return nil }

// ---------------------------------------------------------------------------------------------------------
// Proof generation scan (the AES half of PostClient.Proof, activation/interface.go:204-207)
// ---------------------------------------------------------------------------------------------------------

// GenerateProof = PostClient.Proof for data on this host: the k2pow search of every nonce group (RandomX, on the device)
// followed by the proving scan.  It stands where the RPC to the post-service stands (activation/nipost.go:171).
func GenerateProof(provider uint32, dataDir string, challenge []byte, cfg SetupConfig, nonces uint32) (*Proof, error) {
	dir := C.CString(dataDir)
	defer C.free(unsafe.Pointer(dir))
	var c C.b200post_post_config
	c.labels_per_unit, c.k1, c.k2 = C.uint64_t(cfg.LabelsPerUnit), C.uint32_t(cfg.K1), C.uint32_t(cfg.K2)
	C.memcpy(unsafe.Pointer(&c.pow_difficulty[0]), unsafe.Pointer(&cfg.PowDifficulty[0]), 32)
	o := C.b200post_prove_opts{provider: C.uint32_t(provider), nonces: C.uint32_t(nonces)}
	var out C.b200post_proof_out
	if err := statusErr(checked(func() C.int {
		return C.b200post_generate_proof(dir, (*C.uint8_t)(unsafe.Pointer(&challenge[0])), &c, &o, &out, nil, nil)
	})); err != nil {
		return nil, err
	}
	return &Proof{Nonce: uint32(out.nonce), Pow: uint64(out.pow), Indices: C.GoBytes(unsafe.Pointer(&out.indices[0]), C.int(out.indices_len))}, nil
}
