// unc_stream_logic.hpp -- host-side bookkeeping of one channel of the streaming path: which of
// Mapper::new_read(Chunk&) / add_chunk / request_reset applies to an arriving chunk, and what
// Mapper::map_chunk concludes once the chunk's events are mapped (reference src/mapper.cpp:210-218,
// 281-299, 381-431; src/read_buffer.cpp:249-296; src/realtime_pool.cpp:108-139).
// Pure C++, __host__ __device__ under nvcc: one copy for unc_stream_step (host), the device replay of
// unc_stream_replay (unc_replay.cuh, thread 0 of a CTA) and the CPU emulator harness of the tests.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/unc_b200.h"

#ifdef __CUDACC__
#define UNC_HD __host__ __device__
#else
#define UNC_HD
#endif

struct HostChan {
    int state = UNC_STREAM_INACTIVE;
    uint32_t chunk_count = 0;
    uint64_t raw_len = 0;
    int ended = 0;
    int max_events_hit = 0;      // event_i_ reached max_events with the chunk fully mapped: map_chunk has not looked yet
    unc_paf_rec rec;
    uint64_t n_children = 0, n_sources = 0, n_occ_blocks = 0, n_sa_steps = 0, n_seeds = 0;
    UNC_HD HostChan() { memset(&rec, 0, sizeof(rec)); rec.rid = -1; }
};

// Returns true when the chunk must be processed on the device.
static UNC_HD inline bool stream_admit(HostChan &h, const unc_chunk_desc &c, uint32_t max_chunks) {
    if (c.new_read) {                                   // Mapper::new_read(Chunk&) -> ReadBuffer(Chunk&)
        h = HostChan();
        h.state = UNC_STREAM_MAPPING; h.chunk_count = 1; h.raw_len = c.n_samples;
        return true;
    }
    if (h.state != UNC_STREAM_MAPPING) return false;    // finished or inactive: the chunk is dropped
    if (c.n_samples == 0) {                             // request_reset -> map_chunk: set_failed + set_ended
        h.state = UNC_STREAM_FAILURE; h.ended = 1;
        return false;
    }
    if (h.chunk_count >= max_chunks) {                  // Mapper::add_chunk, chunks_maxed: set_failed ...
        h.state = UNC_STREAM_FAILURE;
        if (h.max_events_hit) h.ended = 1;              // ... and the next map_chunk's first test adds set_ended (:384-390)
        return false;
    }
    h.chunk_count++; h.raw_len += c.n_samples;          // ReadBuffer::add_chunk
    return true;
}

// After the device mapped the chunk's events: `r` is the mapper's record of this step.
static UNC_HD inline void stream_settle(HostChan &h, const unc_paf_rec &r, uint32_t total_events, uint32_t max_events,
                                 uint32_t max_chunks) {
    h.n_children += r.n_children; h.n_sources += r.n_sources; h.n_occ_blocks += r.n_occ_blocks;
    h.n_sa_steps += r.n_sa_steps; h.n_seeds += r.n_seeds;
    const uint32_t chunk_events = r.n_events;            // unmasked events this chunk pushed into the normaliser
    const uint32_t prev_used = h.rec.events_used;        // event_i_ before this chunk (0 for a new read)
    h.rec = r;
    h.rec.n_events = total_events;
    if (r.status != 0) h.state = UNC_STREAM_FAILURE;
    else if (r.mapped) h.state = UNC_STREAM_SUCCESS;                                   // map_next -> SUCCESS
    else if (r.events_used >= max_events) {
        // map_chunk tests event_i_ >= max_events at its NEXT call (:384-390).  If the chunk's events ran out exactly when
        // event_i_ got there, the chunk is fully mapped and the channel first sees try_add_chunk: the next chunk is still
        // accepted and goes through the detector and the normaliser (no event of it is mapped) before the read fails.
        if (!h.max_events_hit && prev_used < max_events && prev_used + chunk_events == r.events_used) h.max_events_hit = 1;
        else { h.state = UNC_STREAM_FAILURE; h.ended = 1; }
    }
    // map_chunk right after process_chunk: nothing to map, chunk processed, chunks maxed -> set_failed (:392-403).
    // (When the chunk did produce events, the next thing the channel sees after mapping them is try_add_chunk.)
    else if (chunk_events == 0 && h.chunk_count >= max_chunks) h.state = UNC_STREAM_FAILURE;
}

static UNC_HD inline void stream_result(const HostChan &h, float bp_per_samp, unc_stream_result *o) {
    o->state = h.state; o->ended = h.ended; o->chunks = h.chunk_count; o->pad_ = 0;
    o->rec = h.rec;
    o->rec.n_children = h.n_children; o->rec.n_sources = h.n_sources; o->rec.n_occ_blocks = h.n_occ_blocks;
    o->rec.n_sa_steps = h.n_sa_steps; o->rec.n_seeds = h.n_seeds;
    if (!o->rec.mapped) o->rec.rd_len = (uint64_t) (h.raw_len * bp_per_samp);          // ReadBuffer::set_raw_len
}
