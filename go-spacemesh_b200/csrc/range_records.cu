// range_records.cu — b200post_merge_range_records (include/b200post_prove.h, DESIGN.md §3c, §3e): the VRF nonce and the
// initial proof of a POST whose files were written by file-range sessions with records, from the records alone.
//
// Why the records suffice.  The ranges are disjoint and tile [0, numLabels), so the POST's arg-min of label32 under
// (label32, index) is the least of the ranges' arg-mins below the common starting threshold; only the threshold test
// and the past-the-end search are POST-wide, and settle_nonce applies them as the stored search does.  Each record's
// hit lists are a ProveRule shard scanned to its end (first K2 hits per nonce inside the range), and the rule merges
// shards in order: the first K2 hits of a nonce over the POST are the first K2 of the concatenation.  So the winner,
// its indices and its pow are those of one session's scan of [0, numLabels).
#include <dirent.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200post_prove.h"
#include "engine.h"
#include "host_hash.h"
#include "initial_proof.h"
#include "postdata_io.h"
#include "prove_internal.h"
#include "setup_internal.h"

namespace b200post {
namespace {

std::string span(uint64_t lo, uint64_t hi) { return "[" + std::to_string(lo) + ", " + std::to_string(hi) + ")"; }

// The initial proof from the records (in range order), or the reason there is none: STATE when they hold no common
// proof scan, INVALID_PROOF when no nonce reached K2 or the gate refused.  Other codes are errors of the call.
int merged_proof(const std::vector<std::unique_ptr<InitialProofScan>> &recs, const b200post_post_metadata &md, const Layout &lay,
                 const b200post_post_config &cfg, uint32_t gate_dev, b200post_proof_out *out, b200post_proof_metadata *pm) {
    InitialProofScan &first = *recs[0];
    for (const auto &rp : recs) {
        InitialProofScan &r = *rp;
        const std::string name = r.state_path();   // read back, a record has no directory
        if (!r.has_proof()) return fail(B200POST_ERR_STATE, name + " holds no initial-proof scan (VRF only)");
        if (r.proof_part() != first.proof_part())
            return fail(B200POST_ERR_STATE, name + " was scanned under other K1, K2, nonces, nonce windows, pow difficulty, pow mode or cache key");
        if (r.pows() != first.pows()) return fail(B200POST_ERR_STATE, name + " was scanned with other pows than the first range");
    }
    const b200post_post_config &rc_cfg = first.cfg();
    if (rc_cfg.k1 != cfg.k1 || rc_cfg.k2 != cfg.k2 || memcmp(rc_cfg.pow_difficulty, cfg.pow_difficulty, 32))
        return fail(B200POST_ERR_STATE, "the records were scanned under another K1, K2 or pow difficulty than asked for");
    const uint32_t nonces = first.opts().nonces, windows = first.windows();
    std::vector<std::pair<uint64_t, uint64_t>> ranges;
    for (const auto &r : recs) ranges.emplace_back(r->range().lo, r->range().hi);
    ProveRule rule(ranges, 0, nonces, windows, cfg.k2);
    for (size_t s = 0; s < recs.size(); s++) {
        HitBook &book = rule.book(s);
        for (const auto &kv : recs[s]->hits().lists())
            for (const KeptHit &k : kv.second) book.add(kv.first, k.index, nullptr);
        book.advance(ranges[s].second - ranges[s].first);   // the shard is whole
    }
    uint32_t nonce = 0;
    std::vector<uint64_t> idx;
    int rc;
    if (!rule.decide(&nonce, &idx, &rc)) return rc ? rc : no_proof(windows, nonces);
    if ((rc = write_proof(lay.num_labels, nonce, idx, first.pows().data(), 0, lay.num_labels, out))) return rc;
    memset(pm, 0, sizeof *pm);
    memcpy(pm->node_id, md.node_id, 32);
    memcpy(pm->commitment_atx_id, md.commitment_atx_id, 32);
    pm->num_units = md.num_units; pm->labels_per_unit = md.labels_per_unit;   // the challenge is the zero one
    return gate_proof(gate_dev, cfg, md.scrypt_n, first.opts(), *pm, out);
}

}  // namespace
}  // namespace b200post

using namespace b200post;

extern "C" int b200post_merge_range_records(const char *data_dir, const b200post_post_config *cfg, const b200post_merge_opts *o,
                                            b200post_merge_result *out, const volatile int *cancel) {
    if (!data_dir || !cfg || !o || !out) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid argument");
    if (o->provider_id < 0 && o->provider_id != B200POST_PROVIDER_ALL) return fail(B200POST_ERR_INVALID_ARGUMENT, "invalid provider id");
    memset(out, 0, sizeof *out);
    const std::string dir = data_dir;

    // ---- the host checks, in order; nothing is written until they all pass
    b200post_post_metadata md;
    if (int rc = load_post_metadata(dir, &md)) return rc;
    if (cfg->labels_per_unit != md.labels_per_unit) return fail(B200POST_ERR_CONFIG_MISMATCH, "`LabelsPerUnit` mismatch with the metadata in DataDir");
    const Layout lay(md);   // checked with the files, below
    std::vector<std::string> names;
    if (DIR *d = opendir(dir.c_str())) {
        while (struct dirent *e = readdir(d)) {
            bool tmp;
            if (post_file_kind(e->d_name, &tmp) == PostFile::kRangeRecord && !tmp) names.push_back(e->d_name);
        }
        closedir(d);
    }
    std::sort(names.begin(), names.end());
    std::vector<std::unique_ptr<InitialProofScan>> recs;
    for (const std::string &name : names) {
        const std::string path = join(dir, name);
        std::string bytes;
        if (!read_file(path, &bytes)) return fail(B200POST_ERR_IO, "range record " + path + " cannot be read");
        recs.emplace_back(new InitialProofScan);
        InitialProofScan &r = *recs.back();
        if (!r.read_record(bytes)) return fail(B200POST_ERR_IO, "range record " + path + " is damaged");
        const b200post_post_metadata &rm = r.md();
        if (memcmp(rm.node_id, md.node_id, 32) || memcmp(rm.commitment_atx_id, md.commitment_atx_id, 32) || rm.num_units != md.num_units ||
            rm.labels_per_unit != md.labels_per_unit || rm.max_file_size != md.max_file_size || rm.scrypt_n != md.scrypt_n)
            return fail(B200POST_ERR_CONFIG_MISMATCH, "range record " + path + " was made for another POST (identity, NumUnits, LabelsPerUnit, "
                                                      "MaxFileSize or Scrypt.N)");
    }
    std::sort(recs.begin(), recs.end(), [](const std::unique_ptr<InitialProofScan> &a, const std::unique_ptr<InitialProofScan> &b) {
        return a->range().lo < b->range().lo;
    });
    std::string gaps;
    uint64_t covered = 0;
    for (size_t i = 0; i < recs.size(); i++) {
        const RangeSpec &r = recs[i]->range();
        if (r.lo < covered)
            return fail(B200POST_ERR_STATE, "range records overlap: labels " + span(r.lo, std::min(covered, r.hi)) + " are in two records");
        if (r.lo > covered) gaps += (gaps.empty() ? "" : ", ") + span(covered, r.lo);
        covered = r.hi;
    }
    if (covered < lay.num_labels) gaps += (gaps.empty() ? "" : ", ") + span(covered, lay.num_labels);
    if (!gaps.empty()) return fail(B200POST_ERR_STATE, "the range records do not cover labels " + gaps + ": those ranges have no record");
    for (const auto &r : recs)
        if (r->upto() != r->range().hi)
            return fail(B200POST_ERR_STATE, "range record " + r->state_path() + " is incomplete: it covers labels " + span(r->range().lo, r->upto()) +
                                                " of " + span(r->range().lo, r->range().hi) + "; finish its range session first");
    if (int rc = check_layout(md)) return rc;
    if (int rc = check_post_files(dir, lay, 0, lay.n_files - 1)) return rc;
    std::vector<uint32_t> devs;
    if (int rc = provider_devices(o->provider_id, &devs)) return rc;
    const uint32_t dev = devs[0];
    if (int rc = device_engine(dev)) return rc;
    out->ranges = (uint32_t)recs.size();

    // ---- the nonce: the least of the ranges' bests under (label32, index), then the rule of an init
    uint8_t best32[32];
    memset(best32, 0xff, 32);   // none below the threshold: never below it either
    uint64_t best_index = 0;
    bool any = false;
    for (const auto &r : recs) {
        const b200post_vrf_nonce &v = r->vrf();
        if (!v.found) continue;
        if (!any || vrf_less(v.label32, v.index, best32, best_index)) { memcpy(best32, v.label32, 32); best_index = v.index; any = true; }
    }
    bool past_end = false;
    if (int rc = settle_nonce(dir, &md, best_index, best32, o->provider_id, o->compute_batch_size ? o->compute_batch_size : 1ull << 20,
                              &out->nonce, &past_end, cancel))
        return rc;
    out->past_end = past_end;

    // ---- the initial proof, once the nonce is settled (as in a full session); a stale file must not answer
    b200post_proof_metadata pm{};
    int rc = merged_proof(recs, md, lay, *cfg, dev, &out->proof, &pm);
    if (rc == B200POST_OK) {
        if ((rc = save_initial_proof_file(dir, pm, *cfg, recs[0]->opts().nonces, recs[0]->windows(), out->proof))) return rc;
    } else if (rc == B200POST_ERR_STATE || rc == B200POST_ERR_INVALID_PROOF) {
        snprintf(out->proof_reason, sizeof out->proof_reason, "%s", last_error());
        memset(&out->proof, 0, sizeof out->proof);
        unlink(join(dir, kInitialProofFile).c_str());
    } else {
        return rc;
    }
    out->proof_rc = rc;
    set_error("");
    return B200POST_OK;
}
