// oracle/_ref shim: a C-ABI window onto the UNMODIFIED reference mapping path.
//
// TEST INFRASTRUCTURE ONLY.  This file is compiled together with the reference's own
// sources where they lie under /root/reference (src/mapper.cpp, event_detector.cpp,
// normalizer.cpp, seed_tracker.cpp, range.cpp, read_buffer.cpp, chunk.cpp,
// event_profiler.cpp and the vendored submods/bwa C files) by oracle/ref_build/Makefile
// into oracle/_ref/libuncalled_ref.so.  Nothing of the reference is copied into this
// repository; this translation unit only *calls* it:
//   Mapper::new_read / Mapper::map_read      (reference src/mapper.cpp:188-207)
//   EventDetector::get_means / get_events    (reference src/event_detector.cpp:114-145)
//   Normalizer::set_signal / pop             (reference src/normalizer.cpp:31-44,120-129)
//   PoreModel::match_prob                    (reference src/pore_model.hpp:163-165)
//   BwaIndex::get_neighbor/get_kmer_range/sa (reference src/bwa_index.hpp:158-178)
//   BwaIndex::create -> bwa_idx_build        (reference src/bwa_index.hpp:92-101)
// Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference)
// may load the resulting library.
#include <algorithm>
#include <array>
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <fstream>
#include <iostream>
#include <map>
#include <mutex>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>
#include <cmath>
#include <chrono>
#include <cassert>
#include "pdqsort.h"
#include <climits>
#include <utility>
#include <exception>

// The shim needs to read Paf's coordinates and Mapper's event counter, which the
// reference keeps private.  Access control does not change object layout.
#define private public
#include "mapper.hpp"
#undef private
#include "self_align_ref.hpp"
#include "model_r94.inl"
#include "dtw.hpp"

extern "C" {

typedef struct {
    int32_t mapped, fwd, rid;
    uint32_t n_events;     // events detected over the whole signal
    uint32_t events_used;  // Mapper::event_i_ when map_read returned
    uint32_t matches;
    uint64_t rd_len, rd_st, rd_en, rf_st, rf_en, rf_len;
    float map_ms;
} ref_paf_rec;

static std::vector<std::pair<std::string, u64>> g_seqs;

int ref_load(const char *bwa_prefix, const char *preset) {
    if (Mapper::fmi.is_loaded()) return 1;  // static index: one load per process
    Mapper::PRMS.bwa_prefix = bwa_prefix;
    Mapper::PRMS.idx_preset = preset ? preset : "default";
    Mapper m;  // triggers Mapper::load_static()
    g_seqs = Mapper::fmi.get_seqs();
    return 0;
}

// The reference's DTW classes (src/dtw.hpp:188-232) on one problem; path = get_path() as (first, second) pairs.
int ref_dtw(int cost_kind, int subseq, float dw, float hw, float vw, const float *means, uint32_t n_cols, const uint16_t *kmers,
            uint32_t n_rows, uint64_t *path, uint64_t *path_len, float *score, float *mean_score) {
    std::vector<float> m(means, means + n_cols);
    std::vector<u16> k(kmers, kmers + n_rows);
    DTWParams prm = {subseq == 1 ? DTWSubSeq::ROW : (subseq == 2 ? DTWSubSeq::COL : DTWSubSeq::NONE), dw, hw, vw};
    std::vector<std::pair<u64, u64>> p;
    if (cost_kind == 0) { DTWr94p d(m, k, prm); p = d.get_path(); *score = d.score(); *mean_score = d.mean_score(); }
    else { DTWr94d d(m, k, prm); p = d.get_path(); *score = d.score(); *mean_score = d.mean_score(); }
    for (size_t i = 0; i < p.size(); i++) { path[2 * i] = p[i].first; path[2 * i + 1] = p[i].second; }
    *path_len = p.size();
    return 0;
}

// The reference's SeedTracker alone, seed by seed (src/seed_tracker.cpp:129-143,157-232); out as orc_tracker_run (oracle/unc_oracle.c).
int ref_tracker_run(uint32_t min_map_len, float min_mean_conf, float min_top_conf, const uint64_t *ref_en, const uint32_t *ref_len,
                    const uint32_t *evt, uint32_t n, uint32_t *out) {
    SeedTracker::Params prm = {min_map_len, min_mean_conf, min_top_conf};
    SeedTracker t(prm);
    for (uint32_t i = 0; i < n; i++) {
        t.add_seed(ref_en[i], ref_len[i], evt[i]);
        SeedCluster f = t.get_final();
        out[6 * i + 0] = (uint32_t) t.seed_clusters_.size();
        out[6 * i + 1] = t.max_map_.total_len_;
        out[6 * i + 2] = (uint32_t) t.max_map_.ref_en_.start_;
        out[6 * i + 3] = t.max_map_.evt_en_;
        out[6 * i + 4] = f.is_valid() ? f.total_len_ : 0u;
        out[6 * i + 5] = (uint32_t) t.all_lens_.size();
    }
    return 0;
}

void ref_set_max_events(uint32_t v) { Mapper::PRMS.max_events = v; }
void ref_set_max_paths(uint32_t v) { Mapper::PRMS.max_paths = v; }
uint32_t ref_get_max_events() { return Mapper::PRMS.max_events; }

uint64_t ref_fmi_size() { return Mapper::fmi.size(); }
uint64_t ref_sa(uint64_t i) { return Mapper::fmi.sa(i); }
void ref_kmer_range(uint16_t kmer, uint64_t *st, uint64_t *en) {
    Range r = Mapper::fmi.get_kmer_range(kmer);
    *st = r.start_; *en = r.end_;
}
void ref_get_neighbor(uint64_t st, uint64_t en, uint8_t base, uint64_t *ost, uint64_t *oen) {
    Range r = Mapper::fmi.get_neighbor(Range(st, en), base);
    *ost = r.start_; *oen = r.end_;
}
float ref_prob_thresh(int bin) { return Mapper::prob_threshes_[bin]; }
float ref_match_prob(float samp, uint16_t kmer) { return Mapper::model.match_prob(samp, kmer); }
float ref_model_mean() { return Mapper::model.get_means_mean(); }
float ref_model_stdv() { return Mapper::model.get_means_stdv(); }
int ref_n_seqs() { return (int) g_seqs.size(); }
const char *ref_seq_name(int i) { return g_seqs[i].first.c_str(); }
uint64_t ref_seq_len(int i) { return g_seqs[i].second; }

// EventDetector over a whole signal.  means/starts/lens must hold n entries.
uint32_t ref_get_events(const float *raw, uint32_t n, float *means, uint32_t *starts,
                        uint32_t *lens, float *mean_event_len) {
    EventDetector ed;
    std::vector<float> sig(raw, raw + n);
    std::vector<Event> ev = ed.get_events(sig);
    for (size_t i = 0; i < ev.size(); i++) {
        means[i] = ev[i].mean; starts[i] = ev[i].start; lens[i] = ev[i].length;
    }
    if (mean_event_len) *mean_event_len = ed.mean_event_len();
    return (uint32_t) ev.size();
}

// Offline normaliser as Mapper::map_read drives it (set_signal then pop()).
void ref_normalize(const float *events, uint32_t n, float *out) {
    if (n == 0) return;  // the reference divides by zero here (normalizer.cpp:123)
    Normalizer norm(Mapper::model.get_means_mean(), Mapper::model.get_means_stdv());
    std::vector<float> ev(events, events + n);
    norm.set_signal(ev);
    for (uint32_t i = 0; i < n; i++) out[i] = norm.pop();
}

static void fill_rec(Mapper &m, Paf &p, uint32_t n_events, ref_paf_rec *out) {
    memset(out, 0, sizeof(*out));
    out->mapped = p.is_mapped_;
    out->fwd = p.fwd_;
    out->rid = -1;
    if (p.is_mapped_) {
        for (size_t i = 0; i < g_seqs.size(); i++)
            if (g_seqs[i].first == p.rf_name_) { out->rid = (int32_t) i; break; }
    }
    out->n_events = n_events;
    out->events_used = m.event_i_;
    out->matches = p.matches_;
    out->rd_len = p.rd_len_; out->rd_st = p.rd_st_; out->rd_en = p.rd_en_;
    out->rf_st = p.rf_st_; out->rf_en = p.rf_en_; out->rf_len = p.rf_len_;
    out->map_ms = p.float_tags_.empty() ? 0.f : p.float_tags_.back().second;
}

static void map_one(Mapper &m, const float *sig, uint32_t n, ref_paf_rec *out) {
    uint32_t n_events;
    {
        EventDetector ed;
        std::vector<float> s(sig, sig + n);
        n_events = (uint32_t) ed.get_means(s).size();
    }
    ReadBuffer rb;
    rb.id_ = "r";
    rb.channel_idx_ = 0;
    rb.number_ = 0;
    rb.start_sample_ = 0;
    rb.chunk_processed_ = false;
    rb.full_signal_.assign(sig, sig + n);
    rb.loc_ = Paf(rb.id_, 1, 0);
    rb.set_raw_len(n);
    if (n_events == 0) {  // reference would SIGFPE (normalizer.cpp:123); report unmapped
        fill_rec(m, rb.loc_, 0, out);
        out->events_used = 0;
        return;
    }
    m.new_read(rb);
    Paf p = m.map_read();
    fill_rec(m, p, n_events, out);
}

// One read through a FRESH Mapper (no state carried from earlier reads).
int ref_map_read(const float *sig, uint32_t n, ref_paf_rec *out) {
    Mapper m;
    map_one(m, sig, n, out);
    return 0;
}

// Many reads over n_threads worker threads, one long-lived Mapper per thread exactly as
// MapPool::MapperThread keeps one (reference src/map_pool.cpp:104-158).  Used for timing.
int ref_map_batch_mt(const float *samples, const uint64_t *offsets, const uint32_t *lens,
                     uint32_t n_reads, int n_threads, ref_paf_rec *out) {
    if (n_threads < 1) n_threads = 1;
    std::atomic<uint32_t> next(0);
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; t++) {
        th.emplace_back([&]() {
            Mapper m;
            for (;;) {
                uint32_t i = next.fetch_add(1);
                if (i >= n_reads) break;
                map_one(m, samples + offsets[i], lens[i], out + i);
            }
        });
    }
    for (auto &t : th) t.join();
    return 0;
}

// ---- streaming path (reference src/mapper.cpp:281-431, realtime_pool.cpp:108-139,349-356) -------------
// One read fed chunk by chunk through the reference's own Mapper::new_read(Chunk&) /
// process_chunk / map_chunk / add_chunk, in the order RealtimePool's worker loop and
// try_add_chunk impose: a chunk is converted to events and pushed into the streaming normaliser
// (process_chunk), mapped in batches of evt_batch_size events (map_chunk), and the next chunk is
// accepted only once the previous one is fully mapped (chunk_mapped()).  Wall-clock limits
// (evt_timeout, chunk_timeout) are disabled so that the result is a function of the input only.
// Chunks are cut by the reference's own ReadBuffer::get_chunks (full chunks only).
static void stream_one(Mapper &m, const float *sig, uint32_t n, uint32_t number, ref_paf_rec *out,
                       uint32_t *n_chunks_used, int32_t *ended) {
    ReadBuffer full;
    full.id_ = "r"; full.channel_idx_ = 0; full.number_ = number; full.start_sample_ = 0;
    full.full_signal_.assign(sig, sig + n);
    std::vector<Chunk> chunks;
    full.get_chunks(chunks, true, 0);
    memset(out, 0, sizeof(*out));
    out->rid = -1;
    if (n_chunks_used) *n_chunks_used = 0;
    if (ended) *ended = 0;
    if (chunks.empty()) return;
    m.new_read(chunks[0]);
    uint32_t used = 1;
    size_t next = 1;
    for (;;) {
        m.process_chunk();
        if (m.map_chunk()) break;
        if (m.chunk_mapped()) {
            if (next < chunks.size()) { if (m.add_chunk(chunks[next])) { next++; used++; } }
            else m.request_reset();       // try_add_chunk with an empty chunk: no more signal for this read
        }
    }
    Paf p = m.get_read().loc_;
    fill_rec(m, p, (uint32_t) m.evdt_.total_events_, out);
    if (n_chunks_used) *n_chunks_used = used;
    if (ended) *ended = p.ended_ ? 1 : 0;
    m.deactivate();                       // RealtimePool::update after collecting the result (:166)
}

int ref_stream_read(const float *sig, uint32_t n, float chunk_time, uint32_t max_chunks, ref_paf_rec *out,
                    uint32_t *n_chunks_used, int32_t *ended) {
    Mapper::PRMS.evt_timeout = 1e30f;
    Mapper::PRMS.chunk_timeout = 1e30f;
    float old_ct = ReadBuffer::PRMS.chunk_time;
    u32 old_mc = ReadBuffer::PRMS.max_chunks;
    ReadBuffer::PRMS.chunk_time = chunk_time;
    ReadBuffer::PRMS.max_chunks = max_chunks;
    Mapper m;
    stream_one(m, sig, n, 1, out, n_chunks_used, ended);
    ReadBuffer::PRMS.chunk_time = old_ct; ReadBuffer::PRMS.max_chunks = old_mc;
    return 0;
}

// Several reads one after the other through ONE Mapper, as the reads of one channel reach a
// RealtimePool (the Mapper's streaming normaliser and sources_added_ persist between reads).
// norm_state (optional, 4 per read): the Mapper's streaming Normalizer after the read, (mean_, varsum_, n_, wr_)
// (src/normalizer.hpp:76-78), read directly from its members.
int ref_stream_channel_norm(const float *samples, const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads,
                            float chunk_time, uint32_t max_chunks, ref_paf_rec *out, uint32_t *n_chunks_used, int32_t *ended,
                            double *norm_state) {
    Mapper::PRMS.evt_timeout = 1e30f;
    Mapper::PRMS.chunk_timeout = 1e30f;
    float old_ct = ReadBuffer::PRMS.chunk_time;
    u32 old_mc = ReadBuffer::PRMS.max_chunks;
    ReadBuffer::PRMS.chunk_time = chunk_time;
    ReadBuffer::PRMS.max_chunks = max_chunks;
    Mapper m;
    for (uint32_t i = 0; i < n_reads; i++) {
        stream_one(m, samples + offsets[i], lens[i], i + 1, out + i, n_chunks_used ? n_chunks_used + i : nullptr,
                   ended ? ended + i : nullptr);
        if (norm_state) {
            double *s = norm_state + (size_t) 4 * i;
            s[0] = m.norm_.mean_; s[1] = m.norm_.varsum_; s[2] = m.norm_.n_; s[3] = m.norm_.wr_;
        }
    }
    ReadBuffer::PRMS.chunk_time = old_ct; ReadBuffer::PRMS.max_chunks = old_mc;
    return 0;
}

int ref_stream_channel(const float *samples, const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads,
                       float chunk_time, uint32_t max_chunks, ref_paf_rec *out, uint32_t *n_chunks_used, int32_t *ended) {
    return ref_stream_channel_norm(samples, offsets, lens, n_reads, chunk_time, max_chunks, out, n_chunks_used, ended, nullptr);
}

// A flow cell's worth of channels on n_threads worker threads: read i sits on channel i % n_channels, the reads of a
// channel follow each other through that channel's ONE Mapper (RealtimePool keeps one Mapper per channel and hands the
// channels to its threads, reference src/realtime_pool.cpp:38-72).  Used for timing the streaming path's CPU arm.
int ref_stream_channels_mt(const float *samples, const uint64_t *offsets, const uint32_t *lens, uint32_t n_reads,
                           uint32_t n_channels, float chunk_time, uint32_t max_chunks, int n_threads, ref_paf_rec *out,
                           uint32_t *n_chunks_used, int32_t *ended) {
    Mapper::PRMS.evt_timeout = 1e30f;
    Mapper::PRMS.chunk_timeout = 1e30f;
    float old_ct = ReadBuffer::PRMS.chunk_time;
    u32 old_mc = ReadBuffer::PRMS.max_chunks;
    ReadBuffer::PRMS.chunk_time = chunk_time;
    ReadBuffer::PRMS.max_chunks = max_chunks;
    if (n_threads < 1) n_threads = 1;
    std::atomic<uint32_t> next(0);
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; t++) {
        th.emplace_back([&]() {
            for (;;) {
                uint32_t c = next.fetch_add(1);
                if (c >= n_channels) break;
                Mapper m;
                uint32_t number = 0;
                for (uint32_t i = c; i < n_reads; i += n_channels)
                    stream_one(m, samples + offsets[i], lens[i], ++number, out + i, n_chunks_used ? n_chunks_used + i : nullptr,
                               ended ? ended + i : nullptr);
            }
        });
    }
    for (auto &t : th) t.join();
    ReadBuffer::PRMS.chunk_time = old_ct; ReadBuffer::PRMS.max_chunks = old_mc;
    return 0;
}

// self_align (reference src/self_align_ref.cpp:34-91) as `uncalled index` calls it: FM range lengths along
// the reference from deterministically sampled start positions.  Returns the number of paths; a second call
// with buffers copies them out (CSR: offsets[n+1], values[offsets[n]]).
static std::vector<std::vector<u64>> g_self_align;
uint64_t ref_self_align(const char *bwa_prefix, uint32_t sample_dist, uint64_t *n_values) {
    g_self_align = self_align(bwa_prefix, sample_dist);
    uint64_t tot = 0;
    for (auto &v : g_self_align) tot += v.size();
    if (n_values) *n_values = tot;
    return g_self_align.size();
}
void ref_self_align_copy(uint64_t *offsets, uint64_t *values) {
    uint64_t o = 0;
    for (size_t i = 0; i < g_self_align.size(); i++) {
        offsets[i] = o;
        for (u64 x : g_self_align[i]) values[o++] = x;
    }
    offsets[g_self_align.size()] = o;
}

// pdqsort itself -- the vendored submods/pdqsort/pdqsort.h, the call of src/mapper.cpp:531 -- over 16-byte sort keys under
// the comparison of PathBuffer's operator< (src/mapper.cpp:866-871 with Range's, src/range.cpp:112-119).  A user-defined
// comparison on a non-arithmetic type takes the header's non-branchless code path, as PathBuffer does.  Pins
// uncalled_b200/csrc/unc_pdqsort.cuh (and the oracle's restatement) to the real header on arbitrary arrays, including the
// patterns that drive it into its heapsort fallback, which mapping data never does.
struct RefSortKey { uint32_t start, end; float prob; uint32_t tag; };
void ref_pdqsort_keys(RefSortKey *k, uint32_t n) {
    pdqsort(k, k + n, [](const RefSortKey &a, const RefSortKey &b) {
        const bool range_lt = a.start < b.start || (a.start == b.start && a.end < b.end);
        const bool range_eq = a.start == b.start && a.end == b.end;
        return range_lt || (range_eq && a.prob < b.prob);
    });
}

// pdqsort's fallback after log2(n) highly unbalanced partitions (pdqsort.h:464-468): libstdc++'s make_heap + sort_heap.
// Mapping data never gets there, so the restatement of that routine is pinned on its own.
void ref_heapsort_keys(RefSortKey *k, uint32_t n) {
    auto lt = [](const RefSortKey &a, const RefSortKey &b) {
        const bool range_lt = a.start < b.start || (a.start == b.start && a.end < b.end);
        const bool range_eq = a.start == b.start && a.end == b.end;
        return range_lt || (range_eq && a.prob < b.prob);
    };
    std::make_heap(k, k + n, lt);
    std::sort_heap(k, k + n, lt);
}

// bwa index build exactly as `uncalled index` performs it (bwa_idx_build).
int ref_index_build(const char *fasta, const char *prefix) {
    BwaIndex<KLEN>::create(fasta, prefix);
    return 0;
}

}  // extern "C"
