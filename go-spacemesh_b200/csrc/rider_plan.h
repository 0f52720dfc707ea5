// rider_plan.h — how one layer of a range job is shared with queued gathers ("riders", DeviceEngine in engine.cu).
// Plain C++17, so that it can be tested on the CPU.
//
// A layer of S slots is two segments: [0, range_slots) holds the range job's next n_range labels (start + slot, the
// shared commitment), [range_slots, n_slots) the riders' chunks, each a run of one rider's items from a slot that is a
// multiple of 32, so every chunk has whole warps of K3 and its own words of a compare job's mismatch bitmap.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace b200post {

// A queued gather as the plan sees it: its item count and how many of its items earlier layers took.
struct RiderLoad { uint64_t items = 0, placed = 0; };

// Items [item_off, item_off + n) of queue entry `rider`, in layer slots [slot, slot + n)
struct RiderChunk { size_t rider; uint64_t item_off; uint32_t n, slot; };

struct LayerPlan {
    uint64_t range_off = 0;      // the range job's first label of this layer, relative to its start
    uint32_t n_range = 0;        // range labels in the layer
    uint32_t range_slots = 0;    // n_range rounded up to whole warps: where the rider segment begins
    uint32_t n_slots = 0;        // slots the layer's ROMix launch covers (a multiple of 32)
    std::vector<RiderChunk> chunks;   // rider chunks, ascending slots
};

// Riders may take at most this many slots of a layer of `layer_slots`: half of it, in whole warps
uint32_t rider_cap(uint32_t layer_slots);

// The next layer of a range job of range_total labels whose first range_off are already in earlier layers (< range_total).
// Riders are taken in queue order, each from its first unplaced item, into at most rider_cap(layer_slots) slots, a chunk
// taking its item count rounded up to 32 slots; a rider that does not fit whole takes what fits and continues in the next
// layer, and no later rider goes before it.  The range job fills the rest of the layer (at most layer_slots minus the
// rider slots), so its labels of a layer drop by exactly the rider slots.  `placed` of every rider the layer takes is
// advanced.  layer_slots is a multiple of 32.
LayerPlan plan_layer(uint32_t layer_slots, uint64_t range_off, uint64_t range_total, const std::vector<RiderLoad *> &queue);

}  // namespace b200post
