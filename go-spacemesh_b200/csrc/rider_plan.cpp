// rider_plan.cpp — see rider_plan.h.
#include "rider_plan.h"

#include <algorithm>

namespace b200post {

static inline uint64_t warps_of(uint64_t n) { return (n + 31) / 32 * 32; }

uint32_t rider_cap(uint32_t layer_slots) { return layer_slots / 2 / 32 * 32; }

LayerPlan plan_layer(uint32_t layer_slots, uint64_t range_off, uint64_t range_total, const std::vector<RiderLoad *> &queue) {
    LayerPlan p;
    p.range_off = range_off;
    const uint32_t cap = rider_cap(layer_slots);
    uint32_t used = 0;   // rider slots taken, relative to the rider segment
    for (size_t q = 0; q < queue.size() && used < cap; q++) {
        RiderLoad &r = *queue[q];
        if (r.placed >= r.items) continue;   // every item is in a layer already; it waits for them to retire
        const uint32_t take = (uint32_t)std::min<uint64_t>(r.items - r.placed, cap - used);
        p.chunks.push_back(RiderChunk{q, r.placed, take, used});
        r.placed += take;
        used += (uint32_t)warps_of(take);
    }
    p.n_range = (uint32_t)std::min<uint64_t>(range_total - range_off, layer_slots - used);
    p.range_slots = (uint32_t)warps_of(p.n_range);
    for (RiderChunk &c : p.chunks) c.slot += p.range_slots;
    p.n_slots = p.range_slots + used;
    return p;
}

}  // namespace b200post
