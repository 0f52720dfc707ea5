// metrics.h — process-wide counters of the label engine, the analogue of the reference's Prometheus metrics for
// this path: activation/metrics/metrics.go (post_verification_waiting_total :40-44, post_verification_seconds
// histogram with buckets 1 s x 2^k :46-52, post_duration) and metrics/public/public.go:19-21.
#pragma once
#include <atomic>
#include <cstdint>

namespace b200post {

struct Metrics {
    std::atomic<uint64_t> labels_range_total{0};      // labels produced by init-style range calls
    std::atomic<uint64_t> labels_gather_total{0};     // labels recomputed for verification
    std::atomic<uint64_t> range_calls_total{0}, gather_calls_total{0};
    std::atomic<uint64_t> device_ns_total{0};         // device time of all label calls (CUDA events), ns
    std::atomic<uint64_t> verify_proofs_total{0}, verify_invalid_total{0}, verify_batches_total{0};
    std::atomic<uint64_t> verify_prepare_us_total{0}, verify_gather_judge_us_total{0};   // host unpack/key stage, device stage (wall)
    std::atomic<int64_t> verify_waiting{0};           // PostVerificationQueue gauge: callers inside Verify()
    // PostVerificationLatency: cumulative histogram, upper bounds 1 s x 2^k (k = 0..9), last = +Inf
    std::atomic<uint64_t> verify_seconds_bucket[11];
    std::atomic<uint64_t> verify_seconds_sum_us{0};
    std::atomic<uint64_t> prove_labels_scanned_total{0}, proofs_generated_total{0};
    std::atomic<uint64_t> prove_passes_total{0};   // b200post_generate_proof[_multi|_checked]: one per read of the data
    std::atomic<uint64_t> prove_labels_rechecked_total{0}, prove_damaged_labels_total{0};   // b200post_generate_proof_checked
    std::atomic<uint64_t> setup_sessions_total{0}, setup_label_mismatch_total{0};
    std::atomic<uint64_t> post_data_labels_verified_total{0}, post_data_label_mismatch_total{0};   // b200post_verify_pos
    // block checksums: blocks hashed and compared (check_sums, write_sums), found damaged, rewritten by a repair
    std::atomic<uint64_t> sums_blocks_checked_total{0}, sums_blocks_bad_total{0}, sums_blocks_repaired_total{0};
    // b200post_generate_proof_sums: digest ranges the scan hashed and compared, found bad, recomputed and scanned
    std::atomic<uint64_t> prove_sum_blocks_checked_total{0}, prove_sum_blocks_bad_total{0}, prove_sum_blocks_healed_total{0};
    // gathers that rode a range job's layers (DeviceEngine riders): calls, labels computed in shared layers, and the
    // calls' wait from enqueue to done, a cumulative histogram with upper bounds 1 ms x 2^k (k = 0..14), last = +Inf
    std::atomic<uint64_t> rider_calls_total{0}, rider_labels_total{0};
    std::atomic<uint64_t> rider_wait_bucket[16];
    std::atomic<uint64_t> rider_wait_sum_us{0};
};
Metrics &metrics();
void observe_verify_seconds(double s);
void observe_rider_wait_seconds(double s);

}  // namespace b200post
