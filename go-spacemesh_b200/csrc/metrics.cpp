// metrics.cpp — see metrics.h; b200post_metrics_text() renders the counters in the Prometheus text format.
#include "metrics.h"

#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/b200post.h"

namespace b200post {

Metrics &metrics() { static Metrics m; return m; }

void observe_verify_seconds(double s) {
    Metrics &m = metrics();
    double bound = 1.0;
    for (int k = 0; k < 10; k++, bound *= 2)
        if (s <= bound) m.verify_seconds_bucket[k]++;
    m.verify_seconds_bucket[10]++;   // +Inf
    m.verify_seconds_sum_us += (uint64_t)(s * 1e6);
}

void observe_rider_wait_seconds(double s) {
    Metrics &m = metrics();
    double bound = 0.001;
    for (int k = 0; k < 15; k++, bound *= 2)
        if (s <= bound) m.rider_wait_bucket[k]++;
    m.rider_wait_bucket[15]++;   // +Inf
    m.rider_wait_sum_us += (uint64_t)(s * 1e6);
}

}  // namespace b200post

using namespace b200post;

extern "C" size_t b200post_metrics_text(char *buf, size_t cap) {
    Metrics &m = metrics();
    std::string o;
    auto line = [&](const char *name, const char *help, const char *type, uint64_t v) {
        o += std::string("# HELP ") + name + " " + help + "\n# TYPE " + name + " " + type + "\n" + name + " " + std::to_string(v) + "\n";
    };
    line("b200post_labels_range_total", "POST labels computed over contiguous ranges (initialisation)", "counter", m.labels_range_total);
    line("b200post_labels_gather_total", "POST labels recomputed at scattered indices (verification)", "counter", m.labels_gather_total);
    line("b200post_range_calls_total", "labels_range calls", "counter", m.range_calls_total);
    line("b200post_gather_calls_total", "labels_gather calls", "counter", m.gather_calls_total);
    line("b200post_device_seconds_total_us", "device time of label calls in microseconds", "counter", m.device_ns_total / 1000);
    line("b200post_post_verification_waiting_total", "callers currently inside Verify (post_verification_waiting_total)", "gauge", (uint64_t)m.verify_waiting.load());
    line("b200post_verify_proofs_total", "proofs verified", "counter", m.verify_proofs_total);
    line("b200post_verify_invalid_total", "proofs rejected with an invalid index or pow", "counter", m.verify_invalid_total);
    line("b200post_verify_batches_total", "GPU batches dispatched by the verifier", "counter", m.verify_batches_total);
    line("b200post_verify_prepare_us_total", "host time spent unpacking indices and deriving keys (wall, microseconds)", "counter", m.verify_prepare_us_total);
    line("b200post_verify_gather_judge_us_total", "time spent in the label gather and the judge kernel incl. copies (wall, microseconds)", "counter", m.verify_gather_judge_us_total);
    o += "# HELP b200post_post_verification_seconds Verify latency (post_verification_seconds)\n# TYPE b200post_post_verification_seconds histogram\n";
    double bound = 1.0;
    for (int k = 0; k < 10; k++, bound *= 2)
        o += "b200post_post_verification_seconds_bucket{le=\"" + std::to_string((int)bound) + "\"} " + std::to_string(m.verify_seconds_bucket[k].load()) + "\n";
    o += "b200post_post_verification_seconds_bucket{le=\"+Inf\"} " + std::to_string(m.verify_seconds_bucket[10].load()) + "\n";
    o += "b200post_post_verification_seconds_sum " + std::to_string(m.verify_seconds_sum_us.load() / 1e6) + "\n";
    o += "b200post_post_verification_seconds_count " + std::to_string(m.verify_seconds_bucket[10].load()) + "\n";
    line("b200post_prove_labels_scanned_total", "stored labels streamed through the proving scan", "counter", m.prove_labels_scanned_total);
    line("b200post_proofs_generated_total", "proofs generated", "counter", m.proofs_generated_total);
    line("b200post_prove_passes_total", "reads of the stored POST data by the prover (one per pass of nonce windows)", "counter", m.prove_passes_total);
    line("b200post_prove_labels_rechecked_total", "proving-scan hits recomputed and compared with their stored bytes (checked proofs)", "counter", m.prove_labels_rechecked_total);
    line("b200post_prove_damaged_labels_total", "proving-scan hits whose stored bytes differed from their recomputation (checked proofs)", "counter", m.prove_damaged_labels_total);
    line("b200post_setup_sessions_total", "setup sessions started", "counter", m.setup_sessions_total);
    line("b200post_setup_label_mismatch_total", "reference-label cross-check failures", "counter", m.setup_label_mismatch_total);
    line("b200post_post_data_labels_verified_total", "stored POST labels recomputed and compared (verify_pos)", "counter", m.post_data_labels_verified_total);
    line("b200post_post_data_label_mismatch_total", "stored POST labels that differed from their recomputation (verify_pos)", "counter", m.post_data_label_mismatch_total);
    line("b200post_sums_blocks_checked_total", "1 MiB label blocks hashed and compared with their checksums (check_sums, write_sums)", "counter", m.sums_blocks_checked_total);
    line("b200post_sums_blocks_bad_total", "label blocks whose stored bytes differed from their checksum or recomputation", "counter", m.sums_blocks_bad_total);
    line("b200post_sums_blocks_repaired_total", "damaged label blocks recomputed and written back (check_sums -repair)", "counter", m.sums_blocks_repaired_total);
    line("b200post_prove_sum_blocks_checked_total", "label blocks the proving scan hashed and compared with their checksums (checksummed proofs)", "counter", m.prove_sum_blocks_checked_total);
    line("b200post_prove_sum_blocks_bad_total", "label blocks of checksummed proofs whose stored digest differed from their checksum", "counter", m.prove_sum_blocks_bad_total);
    line("b200post_prove_sum_blocks_healed_total", "bad label blocks a checksummed proof recomputed and scanned from the recomputation", "counter", m.prove_sum_blocks_healed_total);
    line("b200post_engine_rider_calls_total", "gather calls that rode a running range job's ROMix layers instead of waiting for it", "counter", m.rider_calls_total);
    line("b200post_engine_rider_labels_total", "labels of rider calls computed in a range job's layers", "counter", m.rider_labels_total);
    o += "# HELP b200post_engine_rider_wait_seconds rider calls from enqueue to done\n# TYPE b200post_engine_rider_wait_seconds histogram\n";
    bound = 0.001;
    for (int k = 0; k < 15; k++, bound *= 2) {
        char le[32];
        snprintf(le, sizeof le, "%g", bound);
        o += std::string("b200post_engine_rider_wait_seconds_bucket{le=\"") + le + "\"} " + std::to_string(m.rider_wait_bucket[k].load()) + "\n";
    }
    o += "b200post_engine_rider_wait_seconds_bucket{le=\"+Inf\"} " + std::to_string(m.rider_wait_bucket[15].load()) + "\n";
    o += "b200post_engine_rider_wait_seconds_sum " + std::to_string(m.rider_wait_sum_us.load() / 1e6) + "\n";
    o += "b200post_engine_rider_wait_seconds_count " + std::to_string(m.rider_wait_bucket[15].load()) + "\n";
    if (buf && cap) {
        const size_t n = o.size() < cap - 1 ? o.size() : cap - 1;
        memcpy(buf, o.data(), n);
        buf[n] = 0;
    }
    return o.size();
}
