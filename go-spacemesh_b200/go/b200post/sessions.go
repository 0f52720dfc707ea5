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
	"runtime"
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

func setupOpts(opts SetupOpts, dir *C.char) C.b200post_setup_opts {
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
	return o
}

// PrepareInitializer: the commitment ATX is chosen by the caller (activation/post.go:373-435 stays in Go).
func (m *SetupManager) PrepareInitializer(opts SetupOpts, nodeID, commitmentAtxID []byte) error {
	dir := C.CString(opts.DataDir)
	defer C.free(unsafe.Pointer(dir))
	o := setupOpts(opts, dir)
	return setupErr(checked(func() C.int {
		return C.b200post_setup_prepare_initializer(m.h, &o, (*C.uint8_t)(unsafe.Pointer(&nodeID[0])), (*C.uint8_t)(unsafe.Pointer(&commitmentAtxID[0])))
	}))
}

// PrepareFiles is PrepareInitializer restricted to postdata files [fromFile, toFile] (toFile -1 = the last file), for one
// POST initialised on several machines (postcli -fromFile/-toFile).  Without a nonce in the metadata it marks the data
// VrfScanPending: merge every range's files with one metadata file, then SearchVRFNonce (or run a full session).
func (m *SetupManager) PrepareFiles(opts SetupOpts, nodeID, commitmentAtxID []byte, fromFile uint64, toFile int64) error {
	dir := C.CString(opts.DataDir)
	defer C.free(unsafe.Pointer(dir))
	o := setupOpts(opts, dir)
	return setupErr(checked(func() C.int {
		return C.b200post_setup_prepare_files(m.h, &o, (*C.uint8_t)(unsafe.Pointer(&nodeID[0])), (*C.uint8_t)(unsafe.Pointer(&commitmentAtxID[0])),
			C.uint64_t(fromFile), C.int64_t(toFile))
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

// VRFCheck is shared.VRFNonceMetadata plus the nonce (activation/validation.go:261-285).
type VRFCheck struct {
	NodeId, CommitmentAtxId []byte
	Nonce                   uint64
	NumUnits                uint32
	LabelsPerUnit           uint64
	ScryptN                 uint64
	Prioritized             bool // PrioritizedCall(); used by Verifier.VerifyVRFNonce
}

// VRFResult is one check's outcome.  Valid is label32 < floor(2^256 / numLabels): the UNPINNED rule of
// b200post_verify_vrf_nonce, which real network data contradicts as a universal rule (include/b200post.h).  Label is
// the label32 at the nonce, for the rule the network uses.  Err is set for a malformed check only.
type VRFResult struct {
	Valid bool
	Label [32]byte
	Err   error
}

func (c *VRFCheck) cCheck() (cc C.b200post_vrf_check, err error) {
	if len(c.NodeId) != 32 || len(c.CommitmentAtxId) != 32 {
		return cc, errors.New("b200post: node id and commitment ATX id must be 32 bytes")
	}
	C.memcpy(unsafe.Pointer(&cc.node_id[0]), unsafe.Pointer(&c.NodeId[0]), 32)
	C.memcpy(unsafe.Pointer(&cc.commitment_atx_id[0]), unsafe.Pointer(&c.CommitmentAtxId[0]), 32)
	cc.nonce, cc.num_units, cc.labels_per_unit, cc.scrypt_n = C.uint64_t(c.Nonce), C.uint32_t(c.NumUnits), C.uint64_t(c.LabelsPerUnit), C.uint64_t(c.ScryptN)
	if c.Prioritized {
		cc.prioritized = 1
	}
	return cc, nil
}

// VerifyVRFNonce = Validator.VRFNonce / VRFNonceV2 through the verifier's dispatcher: blocking, safe for concurrent
// use, coalesced with concurrent proofs into one GPU gather.  See VRFResult for what valid and label mean.
func (v *Verifier) VerifyVRFNonce(c *VRFCheck) (valid bool, label [32]byte, err error) {
	cc, err := c.cCheck()
	if err != nil {
		return false, label, err
	}
	var ok C.int
	var cl [32]C.uint8_t
	rc, msg := checked(func() C.int { return C.b200post_verifier_verify_vrf_nonce(v.h, &cc, &ok, &cl[0]) })
	switch rc {
	case C.B200POST_OK:
		for i := range label {
			label[i] = byte(cl[i])
		}
		return ok != 0, label, nil
	case C.B200POST_ERR_CLOSED:
		return false, label, ErrVerifierClosed
	default:
		return false, label, statusErr(rc, msg)
	}
}

// VerifyVRFNonces runs many checks in one GPU batch on the calling goroutine, split over `providers` in contiguous
// runs (one device: []uint32{id}).  Results are in the order of `checks`; a malformed check (numLabels 0 or above
// 2^64-1, scrypt N not a power of two in [2, 2^20]) gets its own Err and leaves the others alone.
func VerifyVRFNonces(providers []uint32, checks []VRFCheck) ([]VRFResult, error) {
	if len(providers) == 0 {
		return nil, errors.New("b200post: no providers")
	}
	n := len(checks)
	out := make([]VRFResult, n)
	cs := make([]C.b200post_vrf_check, n+1) // C structs without Go pointers; one spare so that &cs[0] exists for n == 0
	for i := range checks {
		cc, err := checks[i].cCheck()
		if err != nil {
			return nil, err
		}
		cs[i] = cc
	}
	statuses, valid := make([]C.int, n+1), make([]C.int, n+1)
	labels := make([]byte, 32*(n+1))
	rc, msg := checked(func() C.int {
		return C.b200post_verify_vrf_nonces_multi((*C.uint32_t)(unsafe.Pointer(&providers[0])), C.int(len(providers)), C.size_t(n),
			&cs[0], &statuses[0], &valid[0], (*C.uint8_t)(unsafe.Pointer(&labels[0])))
	})
	if err := statusErr(rc, msg); err != nil {
		return nil, err
	}
	for i := range out {
		out[i].Valid = valid[i] != 0
		copy(out[i].Label[:], labels[32*i:32*i+32])
		if statuses[i] != C.B200POST_OK {
			out[i].Err = statusErr(statuses[i], "malformed VRF check (num_units * labels_per_unit or scrypt N)")
		}
	}
	return out, nil
}

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

// GenerateProofOn is GenerateProof over several devices (repeats allowed): the k2pow windows and contiguous shards of
// the label scan are spread over the list, and the proof is byte-identical to the one-device proof.  ctx cancels the
// call (polled between k2pow windows and per scan chunk).  A read error in any shard fails the call, even past the
// point where a one-device scan would already have found its proof.
func GenerateProofOn(ctx context.Context, providers []uint32, dataDir string, challenge []byte, cfg SetupConfig, nonces uint32) (*Proof, error) {
	if len(providers) == 0 {
		return nil, ErrNoProvider
	}
	dir := C.CString(dataDir)
	defer C.free(unsafe.Pointer(dir))
	var c C.b200post_post_config
	c.labels_per_unit, c.k1, c.k2 = C.uint64_t(cfg.LabelsPerUnit), C.uint32_t(cfg.K1), C.uint32_t(cfg.K2)
	C.memcpy(unsafe.Pointer(&c.pow_difficulty[0]), unsafe.Pointer(&cfg.PowDifficulty[0]), 32)
	o := C.b200post_prove_opts{nonces: C.uint32_t(nonces)}
	provs := (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&providers[0])), 4*len(providers))))
	defer C.free(unsafe.Pointer(provs))
	flag, stop := cancelFlag(ctx)
	defer stop()
	var out C.b200post_proof_out
	if err := statusErr(checked(func() C.int {
		return C.b200post_generate_proof_multi(dir, (*C.uint8_t)(unsafe.Pointer(&challenge[0])), &c, &o, provs, C.int(len(providers)), &out, nil, flag)
	})); err != nil {
		return nil, err
	}
	return &Proof{Nonce: uint32(out.nonce), Pow: uint64(out.pow), Indices: C.GoBytes(unsafe.Pointer(&out.indices[0]), C.int(out.indices_len))}, nil
}

// ProveCheck is what GenerateProofChecked found: scan hits recomputed, distinct damaged label indices among them (a
// lower bound on the damage), the lowest 64 of those ascending, and whether the proof passed the library's verifier.
type ProveCheck struct {
	LabelsRechecked uint64
	Damaged         uint64
	DamagedIndex    []uint64
	ProofVerified   bool
	Rounds          uint32
}

// GenerateProofChecked is GenerateProofOn over stored data that may be damaged (b200post_generate_proof_checked): a
// stored label is a hit only when it also equals its recomputed label, and the proof passes the library's verifier
// before it is returned.  On clean data the proof equals GenerateProofOn's.  Damage is not an error: a non-empty
// report means the data needs `b200postcli -verify -fraction 100` and the damaged file a repair.
func GenerateProofChecked(ctx context.Context, providers []uint32, dataDir string, challenge []byte, cfg SetupConfig, nonces uint32) (*Proof, *ProveCheck, error) {
	if len(providers) == 0 {
		return nil, nil, ErrNoProvider
	}
	dir := C.CString(dataDir)
	defer C.free(unsafe.Pointer(dir))
	var c C.b200post_post_config
	c.labels_per_unit, c.k1, c.k2 = C.uint64_t(cfg.LabelsPerUnit), C.uint32_t(cfg.K1), C.uint32_t(cfg.K2)
	C.memcpy(unsafe.Pointer(&c.pow_difficulty[0]), unsafe.Pointer(&cfg.PowDifficulty[0]), 32)
	o := C.b200post_prove_opts{nonces: C.uint32_t(nonces)}
	provs := (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&providers[0])), 4*len(providers))))
	defer C.free(unsafe.Pointer(provs))
	flag, stop := cancelFlag(ctx)
	defer stop()
	var out C.b200post_proof_out
	var chk C.b200post_prove_check
	if err := statusErr(checked(func() C.int {
		return C.b200post_generate_proof_checked(dir, (*C.uint8_t)(unsafe.Pointer(&challenge[0])), &c, &o, provs, C.int(len(providers)), &out, nil, &chk, flag)
	})); err != nil {
		return nil, nil, err
	}
	rep := &ProveCheck{LabelsRechecked: uint64(chk.labels_rechecked), Damaged: uint64(chk.damaged), ProofVerified: chk.proof_verified != 0,
		Rounds: uint32(chk.rounds)}
	for i := 0; i < int(chk.n_reported); i++ {
		rep.DamagedIndex = append(rep.DamagedIndex, uint64(chk.damaged_index[i]))
	}
	return &Proof{Nonce: uint32(out.nonce), Pow: uint64(out.pow), Indices: C.GoBytes(unsafe.Pointer(&out.indices[0]), C.int(out.indices_len))}, rep, nil
}

// ---------------------------------------------------------------------------------------------------------
// The initial proof (BuildInitialPost's PostClient.Proof(ctx, nodeID, shared.ZeroChallenge, nil), activation/activation.go:350-403)
// ---------------------------------------------------------------------------------------------------------

// RequestInitialProof asks the prepared session (the whole POST, not a file range) for the initial proof: the proof
// for the zero challenge, computed from the labels as StartSession writes them and stored in initial_post.json in the
// data dir.  The k2pow runs on the session's devices (builtin RandomX search) before the first label batch.  Call it
// between PrepareInitializer and StartSession; K1, K2 and the pow difficulty are the manager's SetupConfig.
func (m *SetupManager) RequestInitialProof(nonces uint32) error {
	o := C.b200post_prove_opts{nonces: C.uint32_t(nonces), pow_mode: C.B200POST_POW_BUILTIN}
	return setupErr(checked(func() C.int { return C.b200post_setup_request_initial_proof(m.h, &o) }))
}

// InitialProof returns the initial proof of the completed session.  ErrInvalidProof-class errors (the status text
// gives the reason) mean no nonce reached K2 or the verifier refused the proof: the post-service then proves from the
// stored data.
func (m *SetupManager) InitialProof() (*Proof, error) {
	var out C.b200post_proof_out
	if err := setupErr(checked(func() C.int { return C.b200post_setup_initial_proof(m.h, &out, nil) })); err != nil {
		return nil, err
	}
	return &Proof{Nonce: uint32(out.nonce), Pow: uint64(out.pow), Indices: C.GoBytes(unsafe.Pointer(&out.indices[0]), C.int(out.indices_len))}, nil
}

// LoadInitialProof is the post-service's answer to the ZeroChallenge without a scan: the proof a setup session stored
// in dataDir, if it was made for this POST's metadata, cfg and nonce count.  An absent or stale proof is an error
// ("no initial proof"); fall back to GenerateProofChecked.
func LoadInitialProof(dataDir string, cfg SetupConfig, nonces uint32) (*Proof, error) {
	dir := C.CString(dataDir)
	defer C.free(unsafe.Pointer(dir))
	var c C.b200post_post_config
	c.labels_per_unit, c.k1, c.k2 = C.uint64_t(cfg.LabelsPerUnit), C.uint32_t(cfg.K1), C.uint32_t(cfg.K2)
	C.memcpy(unsafe.Pointer(&c.pow_difficulty[0]), unsafe.Pointer(&cfg.PowDifficulty[0]), 32)
	var out C.b200post_proof_out
	if err := setupErr(checked(func() C.int { return C.b200post_load_initial_proof(dir, &c, C.uint32_t(nonces), &out, nil) })); err != nil {
		return nil, err
	}
	return &Proof{Nonce: uint32(out.nonce), Pow: uint64(out.pow), Indices: C.GoBytes(unsafe.Pointer(&out.indices[0]), C.int(out.indices_len))}, nil
}

// ---------------------------------------------------------------------------------------------------------
// Checking stored POST data (postcli -verify; verifying.VerifyPos, recalled, unpinned)
// ---------------------------------------------------------------------------------------------------------

type VerifyPosOpts struct {
	ProviderID uint32  // CUDA ordinal or AllProviders
	Fraction   float64 // percent of each file's labels, (0, 100]; 100 = every label
	FromFile   uint64
	ToFile     int64   // inclusive; -1 = the last file
	Seed       uint64  // 0 = drawn from the OS (returned in the result)
	Progress   *uint64 // optional: labels checked so far (read it with atomic.LoadUint64)
}

type VerifyPosResult struct {
	FilesChecked, LabelsChecked, Mismatches, Seed uint64
	NonceOK, ArgminChecked, ArgminOK             bool
	BadIndices                                   []uint64 // lowest mismatching global label indices, ascending (<= 64)
}

// VerifyPos recomputes a share of each file's labels on the GPU and compares them with the stored bytes.  Invalid data
// returns the result together with ErrLabelMismatch; matching labels without a VRF nonce in the metadata return the
// result and an error saying initialisation has not finished; a cancelled ctx returns the partial result and
// context.Canceled.  Progress needs Go 1.21 (runtime.Pinner).
func VerifyPos(ctx context.Context, dataDir string, o VerifyPosOpts) (*VerifyPosResult, error) {
	dir := C.CString(dataDir)
	defer C.free(unsafe.Pointer(dir))
	var co C.b200post_verify_pos_opts
	C.b200post_default_verify_pos_opts(&co)
	if o.ProviderID == AllProviders {
		co.provider_id = C.B200POST_PROVIDER_ALL
	} else {
		co.provider_id = C.int64_t(o.ProviderID)
	}
	co.fraction, co.from_file, co.to_file, co.seed = C.double(o.Fraction), C.uint64_t(o.FromFile), C.int64_t(o.ToFile), C.uint64_t(o.Seed)
	if o.Progress != nil {
		// co is passed to C, so the Go pointer it holds must be pinned for the call (cgo pointer-passing rules)
		var pin runtime.Pinner
		pin.Pin(o.Progress)
		defer pin.Unpin()
		co.progress = (*C.uint64_t)(unsafe.Pointer(o.Progress))
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
	var out C.b200post_verify_pos_result
	rc, msg := checked(func() C.int { return C.b200post_verify_pos(dir, &co, &out, (*C.int)(unsafe.Pointer(&cancel))) })
	r := &VerifyPosResult{FilesChecked: uint64(out.files_checked), LabelsChecked: uint64(out.labels_checked),
		Mismatches: uint64(out.mismatches), Seed: uint64(out.seed), NonceOK: out.nonce_ok != 0,
		ArgminChecked: out.argmin_checked != 0, ArgminOK: out.argmin_ok != 0}
	for i := 0; i < int(out.n_reported); i++ {
		r.BadIndices = append(r.BadIndices, uint64(out.bad_index[i]))
	}
	switch rc {
	case C.B200POST_OK, C.B200POST_ERR_LABEL_MISMATCH, C.B200POST_ERR_STATE, C.B200POST_ERR_CANCELLED:
		return r, setupErr(rc, msg)
	}
	return nil, setupErr(rc, msg)
}

// ---------------------------------------------------------------------------------------------------------
// The VRF nonce from stored labels (postcli -searchForNonce, recalled, unpinned)
// ---------------------------------------------------------------------------------------------------------

type VRFSearchOpts struct {
	ProviderID       uint32  // CUDA ordinal or AllProviders (scan on the first GPU, past-the-end search on all)
	ComputeBatchSize uint64  // batch of the past-the-end search; 0 = 2^20 (use the init's batch for the same nonce)
	ChunkLabels      uint64  // labels per H2D chunk; 0 = 2^22
	Progress         *uint64 // optional: labels scanned (read it with atomic.LoadUint64)
}

// SearchVRFNonce finds the VRF nonce of the complete POST in dataDir from its stored labels and writes Nonce,
// NonceValue and LastPosition to the metadata as one uninterrupted init would have.  Damaged data returns
// ErrLabelMismatch (the error text names the index) and leaves the metadata as it was.
func SearchVRFNonce(ctx context.Context, dataDir string, o VRFSearchOpts) (nonce uint64, label [32]byte, err error) {
	dir := C.CString(dataDir)
	defer C.free(unsafe.Pointer(dir))
	var co C.b200post_vrf_search_opts
	C.b200post_default_vrf_search_opts(&co)
	if o.ProviderID == AllProviders {
		co.provider_id = C.B200POST_PROVIDER_ALL
	} else {
		co.provider_id = C.int64_t(o.ProviderID)
	}
	co.compute_batch_size, co.chunk_labels = C.uint64_t(o.ComputeBatchSize), C.uint64_t(o.ChunkLabels)
	if o.Progress != nil {
		var pin runtime.Pinner
		pin.Pin(o.Progress)
		defer pin.Unpin()
		co.progress = (*C.uint64_t)(unsafe.Pointer(o.Progress))
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
	var out C.b200post_vrf_nonce
	rc, msg := checked(func() C.int { return C.b200post_search_vrf_nonce(dir, &co, &out, (*C.int)(unsafe.Pointer(&cancel))) })
	if rc == C.B200POST_ERR_LABEL_MISMATCH {
		return 0, label, fmt.Errorf("%w: %s", ErrLabelMismatch, msg)
	}
	if err := setupErr(rc, msg); err != nil {
		return 0, label, err
	}
	C.memcpy(unsafe.Pointer(&label[0]), unsafe.Pointer(&out.label32[0]), 32)
	return uint64(out.index), label, nil
}
