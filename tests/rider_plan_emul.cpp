// rider_plan_emul.cpp — csrc/rider_plan.cpp's layer plan driven the way DeviceEngine::run_job drives it, behind a flat C
// interface, for tests/test_rider_plan_host.py.
#include <cstdint>
#include <vector>

#include "../go-spacemesh_b200/csrc/rider_plan.h"

using namespace b200post;

// A range job of range_total labels in layers of S slots; rider r (of items[r] items) joins the queue before layer
// arrive[r] is planned (riders arriving at the same layer queue in index order).  A rider leaves the queue once every
// item of it is in a layer.  Outputs, at most cap rows each:
//   layers (4 x u64 per layer): range_off, n_range, range_slots, n_slots
//   chunks (5 x u64 per chunk, in plan order): layer, rider, item_off, n, slot
//   placed (per rider): its items that some layer took (the rest would run as an ordinary call)
//   counts: layers, chunks
// Returns 0, or -1 when a table would exceed cap.
extern "C" int emul_run(uint32_t S, uint64_t range_total, uint32_t n_riders, const uint64_t *items, const uint64_t *arrive, uint64_t cap,
                        uint64_t *layers, uint64_t *chunks, uint64_t *placed, uint64_t *counts) {
    std::vector<RiderLoad> load(n_riders);
    for (uint32_t r = 0; r < n_riders; r++) load[r].items = items[r];
    std::vector<uint32_t> queue;   // rider ids, FIFO
    uint64_t off = 0, n_layers = 0, n_chunks = 0;
    for (uint64_t m = 0; off < range_total; m++) {
        for (uint32_t r = 0; r < n_riders; r++)
            if (arrive[r] == m) queue.push_back(r);
        std::vector<RiderLoad *> q;
        for (uint32_t r : queue) q.push_back(&load[r]);
        const LayerPlan p = plan_layer(S, off, range_total, q);
        if (n_layers >= cap) return -1;
        uint64_t *L = layers + 4 * n_layers++;
        L[0] = p.range_off; L[1] = p.n_range; L[2] = p.range_slots; L[3] = p.n_slots;
        for (const RiderChunk &c : p.chunks) {
            if (n_chunks >= cap) return -1;
            uint64_t *C = chunks + 5 * n_chunks++;
            C[0] = m; C[1] = queue[c.rider]; C[2] = c.item_off; C[3] = c.n; C[4] = c.slot;
        }
        std::vector<uint32_t> keep;
        for (uint32_t r : queue)
            if (load[r].placed < load[r].items) keep.push_back(r);
        queue = keep;
        off += p.n_range;
    }
    for (uint32_t r = 0; r < n_riders; r++) placed[r] = load[r].placed;
    counts[0] = n_layers; counts[1] = n_chunks;
    return 0;
}

extern "C" uint32_t emul_cap(uint32_t S) { return rider_cap(S); }
