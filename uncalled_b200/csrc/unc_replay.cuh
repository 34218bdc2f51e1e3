// unc_replay.cuh -- the device replay of whole reads (unc_stream_replay, `map-ord`): what MapPoolOrd::update
// (reference src/map_pool_ord.cpp:61-121) does to one channel, step after step, until the channel's reads of
// the window are finished -- without returning to the host between one chunk and the next.
//
// One CTA takes one CHANNEL at a time from a queue (the host lists them longest signal first) and runs its
// reads in order.  Per step, thread 0 builds the front read's next chunk (ReadBuffer::get_chunk,
// src/read_buffer.cpp:302-315: the last chunk may be partial, past the end the chunk is empty) and puts it
// through stream_admit, the bookkeeping unc_stream_step runs on the host (unc_stream_logic.hpp).  An admitted
// chunk is detected, profiled and normalised by thread 0 (unc_stream_chunk), its events are mapped by the whole
// CTA in the channel's workspace slot (unc_k2_map_read<STREAM>), and thread 0 settles the step
// (stream_settle).  A read that is no longer MAPPING is appended to the output and the next read starts at the
// next step.  Per-channel state is where unc_stream_step keeps it: DevChanSig, the normaliser ring, DevMapState,
// one workspace slot per channel, and the channel's HostChan (copied to the device for the call).
//
// Items of the DevBatch are indexed by CHANNEL (B.chan is the identity), so the mapper finds the chunk's events,
// scale/shift and record at the channel's position and its state at mstate[channel].
#pragma once
#include "unc_stream.cuh"
#include "unc_stream_logic.hpp"

struct DevReplay {
    const unc_replay_read *reads;    // the window's reads, grouped by channel in per-channel order
    const u32 *read_idx;             // their positions in the caller's array
    const u32 *chans;                // the window's channels, in the order the CTAs take them
    const u32 *first, *count;        // per listed channel: its reads in `reads`
    u32 n_chans;
    u32 chunk_len, max_chunks, max_events;
    float bp_per_samp;
    HostChan *hc;                    // n_channels: the stream's per-channel bookkeeping
    u64 *step;                       // n_channels: steps taken so far by each channel
    DevReadDesc *desc;               // n_channels: the chunk in progress (B.reads aliases it)
    unc_replay_result *out;          // one entry per read, in the order reads finish on the device
    u32 *n_out, *queue, *overflow;
};

// thread 0: the read at reads[rd] is finished at `step`
UNC_DEV void unc_replay_emit(const DevReplay &R, u32 rd, const HostChan &h, u64 step, u32 kind) {
    unc_replay_result &o = R.out[d_atomic_add(R.n_out, 1u)];
    o.read = R.read_idx[rd];
    o.number = R.reads[rd].number;
    o.step = step;
    o.kind = kind;
    o.pad_ = 0;
    stream_result(h, R.bp_per_samp, &o.res);
    if (o.res.rec.status != 0) d_atomic_add(R.overflow, 1u);
}

// Persistent CTA body.  ctl: two broadcast words in shared memory (the channel; go | new_read << 1).
template <bool EXACT>
UNC_DEV void unc_replay_cta_main(const DevIndex &ix, const DevParams &p, const DevBatch &B, const DevWork &W0,
                                 const DevWorkStrides &S, const DevStream &St, const DevReplay &R, K2Shared *sh,
                                 volatile u32 *ctl) {
    unc_k2_cta_setup(ix, p, sh);
    const bool t0 = c_tid() == 0;
    u32 rd = 0, rd_end = 0, kind = 1;                   // thread 0's cursor: front read, end of the channel's reads
    u64 ci = 0, step = 0;                              // chunk index of the front read, the channel's step count
    for (;;) {
        if (t0) {
            const u32 k = d_atomic_add(R.queue, 1u);
            u32 ch = 0xFFFFFFFFu;
            if (k < R.n_chans) {
                ch = R.chans[k];
                rd = R.first[k]; rd_end = rd + R.count[k]; ci = 0;
                step = R.step[ch];
                sh->work = unc_work_slot(W0, S, ch);    // published by unc_k2_map_read's first barrier
            }
            ctl[0] = ch;
        }
        c_sync();
        const u32 ch = ctl[0];
        if (ch == 0xFFFFFFFFu) break;
        for (;;) {
            if (t0) {
                HostChan &h = R.hc[ch];
                u32 go = 0;
                while (rd < rd_end) {                   // MapPoolOrd::update for this channel, until a chunk needs the device
                    const unc_replay_read &q = R.reads[rd];
                    const u64 st = ci * R.chunk_len;
                    unc_chunk_desc c;
                    c.channel = ch; c.new_read = ci == 0 ? 1u : 0u; c.dtype = q.dtype;
                    c.offset = q.offset + st;
                    c.n_samples = st >= q.n_samples ? 0u : (u32) (q.n_samples - st < R.chunk_len ? q.n_samples - st : R.chunk_len);
                    c.cal_range = q.cal_range; c.cal_offset = q.cal_offset; c.cal_digit = q.cal_digit;
                    kind = c.n_samples ? 1u : 0u;
                    const u64 s = step++;
                    if (stream_admit(h, c, R.max_chunks)) {
                        DevReadDesc &d = R.desc[ch];
                        d.offset = c.offset; d.n_samples = c.n_samples; d.dtype = c.dtype;
                        d.cal_range = c.cal_range; d.cal_offset = c.cal_offset; d.cal_digit = c.cal_digit; d.pad = 0;
                        go = 1u | c.new_read << 1;
                        ci++;
                        break;
                    }
                    // not admitted: "no more signal" or chunks maxed -- the read is finished
                    unc_replay_emit(R, rd, h, s, kind);
                    rd++; ci = 0;
                }
                if (!go) R.step[ch] = step;
                ctl[1] = go;
            }
            c_sync();
            const u32 go = ctl[1];
            if (!go) break;
            if (t0) {
                unc_stream_chunk(B, p, St, ch, go >> 1);
                B.k1_flags[ch] = St.sig[ch].evdt.total_events;   // EventDetector::total_events_ so far
            }
            c_sync();
            unc_k2_map_read<true, EXACT, true>(ix, p, B, sh->work, sh, ch);
            if (t0) {
                HostChan &h = R.hc[ch];
                stream_settle(h, *(const unc_paf_rec *) &B.out[ch], B.k1_flags[ch], R.max_events, R.max_chunks);
                if (h.state != UNC_STREAM_MAPPING) {
                    unc_replay_emit(R, rd, h, step - 1, kind);
                    rd++; ci = 0;
                }
            }
        }
    }
}
