/* include/unc_b200.h -- C-ABI of the H100-native `uncalled map` hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types, no
 * exceptions or abort() across it, every call returns 0 or a negative unc_status.
 * The library (uncalled_b200/libunc_b200.so) contains ONLY the CUDA path; there is no
 * CPU fallback -- if no CUDA device is usable every compute entry point fails with
 * UNC_E_CUDA / UNC_E_NO_DEVICE.
 *
 * Each entry point names the reference interface it replaces (paths under the reference
 * tree, skovaka/UNCALLED v2.3.0):
 *
 *   unc_index_load      Mapper::load_static            src/mapper.cpp:109-159
 *                       BwaIndex::load_index           src/bwa_index.hpp:116-135
 *   unc_index_build     BwaIndex::create -> bwa_idx_build
 *                                                      src/bwa_index.hpp:92-101
 *   unc_index_build_device  the same files, built on the GPU
 *   unc_params_default  Mapper::PRMS and sub-structs   src/mapper.cpp:29-52,
 *                       seed_tracker.cpp:28-32, event_detector.cpp:17-26,
 *                       read_buffer.cpp:26-32          (what Conf binds, src/conf.hpp:57-95)
 *   unc_pool_create     MapPool::MapPool(Conf&)        src/map_pool.cpp:28-43
 *   unc_map_batch       MapPool::update -> MapperThread::run -> Mapper::new_read/map_read
 *                                                      src/map_pool.cpp:45-69,130-158,
 *                                                      src/mapper.cpp:188-207
 *   unc_map_batch_ordered  one MapperThread's loop with its long-lived Mapper (`-t 1`)
 *                                                      src/map_pool.cpp:104-158, src/mapper.cpp:88,216-246
 *   unc_pool_set_tie_order / unc_stream_set_tie_order
 *                       pdqsort(next_paths_...) as it is  src/mapper.cpp:531,866-871, submods/pdqsort/pdqsort.h
 *   unc_events_batch    EventDetector::get_means + Normalizer::set_signal/pop
 *                                                      src/event_detector.cpp:133-145,
 *                                                      src/normalizer.cpp:31-44,114-129
 *   unc_events_*        EventDetector::get_events, EventProfiler::get_full_mask, PoreModel::match_prob
 *                       (the `events` command; see the section below)
 *   unc_pool_free       MapPool::stop                  src/map_pool.cpp:71-82
 */
#ifndef UNC_B200_H
#define UNC_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    UNC_OK = 0,
    UNC_E_ARG = -1,          /* bad argument */
    UNC_E_IO = -2,           /* index file missing / unreadable / inconsistent */
    UNC_E_CUDA = -3,         /* CUDA runtime error (see unc_last_error) */
    UNC_E_NO_DEVICE = -4,    /* no usable CUDA device */
    UNC_E_TOO_LARGE = -5,    /* index or batch exceeds what the device image supports */
    UNC_E_NOMEM = -6,
    UNC_E_OVERFLOW = -7      /* a per-read device workspace overflowed (record status says which) */
} unc_status;

/* Mirror of the reference's process-global parameter structs (Conf binds references to
 * them, src/conf.hpp:66-72); snapshot by value at unc_pool_create. */
typedef struct {
    /* Mapper::PRMS, src/mapper.cpp:29-52 */
    uint32_t seed_len;        /* 22; the device image supports seed_len == 22 only */
    uint32_t min_rep_len;     /* 0 */
    uint32_t max_rep_copy;    /* 50 */
    uint32_t max_paths;       /* 10000 (<= 32767) */
    uint32_t max_consec_stay; /* 8 */
    uint32_t max_events;      /* 30000 */
    float max_stay_frac;      /* 0.5 */
    float min_seed_prob;      /* -3.75 */
    /* SeedTracker::PRMS_DEF, src/seed_tracker.cpp:28-32 */
    uint32_t min_map_len;     /* 25 */
    float min_mean_conf;      /* 6.00 */
    float min_top_conf;       /* 1.85 */
    /* EventDetector::PRMS_DEF, src/event_detector.cpp:17-26 (window lengths 3/6 are fixed
     * in the device image) */
    uint32_t window_length1, window_length2;
    float threshold1, threshold2, peak_height, min_mean, max_mean;
    /* ReadBuffer::PRMS, src/read_buffer.cpp:26-32 */
    float bp_per_sec, sample_rate;
} unc_params;

/* One read of a batch.  `offset` counts samples (not bytes) from the start of `samples`. */
typedef struct {
    uint64_t offset;
    uint32_t n_samples;
    uint32_t dtype; /* UNC_DTYPE_F32: calibrated pA; UNC_DTYPE_I16: raw DAC values calibrated on
                       the device as src/read_buffer.cpp:239-242 does (u16 reinterpretation) */
    float cal_range, cal_offset, cal_digit; /* used for UNC_DTYPE_I16 only */
} unc_read_desc;

#define UNC_DTYPE_F32 0
#define UNC_DTYPE_I16 1

/* What Paf::set_mapped / set_read_len receive (src/read_buffer.cpp:133-155) plus counters. */
typedef struct {
    int32_t mapped;       /* Paf::is_mapped_ */
    int32_t fwd;          /* '+' / '-' */
    int32_t rid;          /* index into the .ann sequences, -1 when unmapped / untranslatable */
    int32_t status;       /* 0, or UNC_E_OVERFLOW when a device workspace overflowed for this read */
    uint32_t n_events;    /* valid events detected over the whole (possibly truncated) signal */
    uint32_t events_used; /* Mapper::event_i_ when mapping stopped */
    uint32_t matches;
    uint32_t n_clusters;
    uint64_t rd_len, rd_st, rd_en, rf_st, rf_en, rf_len;
    /* exact work counters (algorithmic bytes of the roofline, DESIGN.md) */
    uint64_t n_children, n_sources, n_occ_blocks, n_sa_steps, n_seeds;
} unc_paf_rec;

typedef struct {
    float h2d_ms, k1_ms, k2_ms, d2h_ms, total_ms; /* CUDA events on the pool's stream */
    uint32_t kernel_launches;                      /* launches of this library's kernels */
    uint64_t h2d_bytes, d2h_bytes;
    float k1_events_ms;                            /* the event-detection kernel alone (k1_ms also covers the
                                                      serial-redo and normaliser-statistics launches) */
    float pad_;
} unc_timing;

typedef struct {
    uint64_t n_rows;  /* FM-index length (fwd + revcomp) */
    int32_t n_seqs;
    int32_t device;
    uint64_t device_bytes;  /* the index's device tables; 4 (n_rows + 1) of them are the expanded suffix array when
                               the load built it */
    uint32_t n_kmer_groups;
} unc_index_info;

typedef struct unc_index unc_index;
typedef struct unc_pool unc_pool;

const char *unc_strerror(int status);
const char *unc_last_error(void); /* thread-local detail of the last failure */
int unc_device_count(void);
/* Select the CUDA device used by subsequent unc_index_load / unc_pool_create calls of
 * this process (one process per GPU). */
int unc_init(int device);
/* End of use in this process: waits for the selected device to go idle and forgets the device selection and
 * error text.  Objects the caller still holds (indexes, pools, streams) stay valid until freed; the CUDA context
 * is NOT reset, because the host application (e.g. PyTorch in bench.py) may share it. */
int unc_shutdown(void);

int unc_params_default(unc_params *p);

/* Parses <prefix>.bwt/.sa/.ann/.amb and the <preset> line of <prefix>.uncl on the host,
 * builds the device image (Occ blocks, u32 sampled SA, 1024 k-mer FM ranges, pore model,
 * thresholds) and uploads it.  model_path == NULL selects the built-in r9.4 5-mer model
 * table file given by model_table_path (1024 x {mean, stdv} f32, template order). */
int unc_index_load(const char *bwa_prefix, const char *preset, const char *model_table_path,
                   unc_index **out);
int unc_index_get_info(const unc_index *idx, unc_index_info *info);
int unc_index_seq(const unc_index *idx, int rid, const char **name, uint64_t *len);
/* Host-side copies of device tables, for parity tests. */
int unc_index_kmer_range(const unc_index *idx, uint32_t kmer, uint64_t *start, uint64_t *end);
int unc_index_thresholds(const unc_index *idx, float out[64]);
void unc_index_free(unc_index *idx);

/* bwa-compatible FM-index construction (.pac .ann .amb .bwt .sa), host C++.  UNC_E_TOO_LARGE when 2 x the
 * reference length + 1 reaches 0x7FFFFFF0 (its suffix array is int32). */
int unc_index_build(const char *fasta_path, const char *prefix);
/* The same five files, byte for byte, with the suffix sort and the BWT / Occ / SA construction on the device selected
 * by unc_init.  Accepts every reference whose seq_len = 2 x length is below 0xFFFFFF00 (what unc_index_load accepts):
 * UNC_E_TOO_LARGE above, UNC_E_NO_DEVICE without a device, UNC_E_NOMEM when the device's free memory is below what
 * the build needs; in each of these cases nothing is written.  Device memory: at most 16.4 bytes per FM row plus a sort
 * workspace (DESIGN.md section 4, "FM-index build").
 * unc_index_build_device_last_times: CUDA-event time of the last successful call's phases, ms[0..2] = initial sort
 * (with the upload of the text), doubling rounds, BWT / Occ / SA output (with the copy back); *rounds = doubling rounds;
 * *peak_bytes = the most device memory the build held at once.  unc_index_build_device_last_active: the active rows
 * (rows of groups not yet sorted) of each doubling round, up to cap of them; returns the number of rounds. */
int unc_index_build_device(const char *fasta_path, const char *prefix);
void unc_index_build_device_last_times(float ms[3], uint32_t *rounds, uint64_t *peak_bytes);
uint32_t unc_index_build_device_last_active(uint64_t *active, uint32_t cap);

/* Device workspace for batches of at most max_reads reads / max_samples samples in total. */
int unc_pool_create(const unc_index *idx, const unc_params *prm, uint32_t max_reads,
                    uint64_t max_samples, unc_pool **out);
void unc_pool_free(unc_pool *pool);

/* Whole path over a batch held in HOST memory (pinned or pageable): H2D of the samples,
 * event detection + normalisation kernel, mapping kernel, D2H of the records.  Synchronous. */
int unc_map_batch(unc_pool *pool, const unc_read_desc *reads, uint32_t n_reads, const void *samples,
                  unc_paf_rec *out);
/* Same, with the samples already resident in device memory (`d_samples` is a device
 * pointer on the pool's device); descriptors and results stay on the host. */
int unc_map_batch_device(unc_pool *pool, const unc_read_desc *reads, uint32_t n_reads,
                         const void *d_samples, unc_paf_rec *out);

/* Order of children that compare equal in the per-event child sort (reference src/mapper.cpp:531, pdqsort under
 * operator< :866-871; only the LAST child of a run of equal FM ranges survives, :569-572).  mode 0 (default): emission
 * order -- a stable parallel sort; what the reference computes with its sort made stable, and what it computes itself on
 * 99.7 % of reads.  mode 1: the reference's own pdqsort reproduced step by step (one thread per CTA sorts the event's
 * keys serially, kernel k2_map_exact), so that equal children land exactly where the reference's land: results are then
 * those of the unmodified reference on every read, several times slower on reads that run at the max_paths cap.
 * Applies to the batch calls of this pool; unc_stream_set_tie_order is the streaming path's switch. */
int unc_pool_set_tie_order(unc_pool *pool, int mode);

/* The batch mapped as ONE long-lived Mapper maps its reads one after the other -- what `uncalled map -t 1` prints
 * for a multi-read input.  Replaces a MapPool thread's loop over its reads (reference src/map_pool.cpp:104-158):
 * Mapper::reset (src/mapper.cpp:216-246) keeps the sources_added_ flags (:88), so a read starts with the flags its
 * predecessor left set.  unc_map_batch gives every read a clear set (the reference's result for a read that is
 * first on its thread); this call resolves the chain instead: all reads are mapped in one launch, then only those
 * whose predecessor ended with other flags than they were mapped from are mapped again, until nothing changes
 * (uncalled_b200/csrc/unc_ordered_logic.hpp).  carry[32] (k-mer k = bit k&31 of word k>>5): in, the flags before
 * reads[0] (all zero for a new Mapper); out, the flags after the last read -- pass it on to the next batch.
 * n_remapped / n_rounds (optional): reads mapped a second time, extra launches. */
int unc_map_batch_ordered(unc_pool *pool, const unc_read_desc *reads, uint32_t n_reads, const void *samples,
                          int samples_on_device, uint32_t carry[32], unc_paf_rec *out, uint32_t *n_remapped,
                          uint32_t *n_rounds);

/* The same work as two calls, so that batches on DIFFERENT pools overlap: submit queues the copies and both
 * kernels on the pool's stream and returns; wait blocks until they are done and hands the records over.  Reads
 * differ widely in cost (one that never maps takes ~6x one that does), so the last reads of a batch leave CTAs
 * idle; with two pools used alternately the next batch's CTAs fill the SMs the previous batch's tail frees -- what
 * the reference's thread pool gets by handing every idle thread the next read (src/map_pool.cpp:45-69).
 * `samples` (and, for host samples, the buffer they live in) must stay untouched until the matching wait; a pool
 * holds at most one submitted batch. */
int unc_map_batch_submit(unc_pool *pool, const unc_read_desc *reads, uint32_t n_reads, const void *samples,
                         int samples_on_device);
int unc_map_batch_wait(unc_pool *pool, unc_paf_rec *out);
/* Device-side timing of work spread over several pools: record marks event `slot` (0 or 1) at the current end of
 * the pool's stream; elapsed waits for both events and returns the milliseconds from the first to the second (they
 * may belong to different pools of the same device). */
int unc_pool_record(unc_pool *pool, int slot);
int unc_pool_elapsed(unc_pool *from, int from_slot, unc_pool *to, int to_slot, float *ms);

/* Event detection + normalisation alone.  events/normed hold `stride` floats per read
 * (stride >= the longest read's n_samples); n_events, mean_event_len one entry per read. */
int unc_events_batch(unc_pool *pool, const unc_read_desc *reads, uint32_t n_reads, const void *samples,
                     uint32_t stride, float *events, float *normed, uint32_t *n_events,
                     float *mean_event_len);

/* pore-model log-probabilities of one normalised event against all 1024 k-mers, computed
 * on the device with the mapper's own routine (parity probe). */
int unc_match_probs(const unc_index *idx, float event, float out[1024]);
/* FM probes computed on the device by the mapper's own routines (parity probes).
 *   unc_fm_step       the mapper's backward step, per entry i: rows start[i]-1 and end[i] (1 <= start <= n_rows + 1,
 *                     end <= n_rows); ns[4i+c] = L2[c] + Occ(start-1, c) + 1 and ne[4i+c] = L2[c] + Occ(end, c) for
 *                     all four bases, and valid[i] bit c set iff bit c of want[i] is and ns <= ne.
 *   unc_fm_neighbors  the same step for one base per entry (BwaIndex::get_neighbor): an empty range reads
 *                     start = end + 1 as there.
 *   unc_fm_sa         bwt_sa at rows 0..n_rows as the mapper reads it: from the expanded suffix array when the index
 *                     load built one (it does not when device memory is short or UNC_NO_SA_EXPAND is set), by the LF
 *                     walk over the sampled array otherwise. */
int unc_fm_step(const unc_index *idx, uint32_t n, const uint64_t *start, const uint64_t *end, const uint8_t *want,
                uint64_t *ns, uint64_t *ne, uint8_t *valid);
int unc_fm_neighbors(const unc_index *idx, uint32_t n, const uint64_t *start, const uint64_t *end,
                     const uint8_t *base, uint64_t *ostart, uint64_t *oend);
int unc_fm_sa(const unc_index *idx, uint32_t n, const uint64_t *rows, uint64_t *out);

int unc_pool_last_timing(const unc_pool *pool, unc_timing *t);
/* Counters of the event-detection kernel over the last batch: tiles processed, speculative-FSM
 * re-run rounds, lanes re-run, reads redone by the serial routine (exactness condition failed). */
int unc_pool_k1_stats(const unc_pool *pool, uint32_t out[4]);

/* ---- streaming path (chunks of many channels, persistent per-channel state on the device) ----------
 *   unc_stream_create   RealtimePool::RealtimePool(Conf&): one Mapper per channel  src/realtime_pool.cpp:38-60
 *   unc_stream_step     RealtimePool::add_chunk / try_add_chunk + MapperThread::run ->
 *                       Mapper::new_read(Chunk&) / add_chunk / process_chunk / map_chunk
 *                                                      src/realtime_pool.cpp:74-139,316-360, src/mapper.cpp:210-431
 *   unc_stream_free     RealtimePool::stop_all         src/realtime_pool.cpp:286-297
 * One step hands each listed channel its next chunk and maps ALL of the chunk's events (the reference maps
 * them evt_batch_size at a time and accepts the next chunk only when the previous one is fully mapped, so
 * the results are the same; its wall-clock limits evt_timeout / chunk_timeout do not exist here). */
typedef struct {
    uint32_t channel;     /* 0-based channel index */
    uint32_t new_read;    /* 1: this chunk starts a new read on the channel (Mapper::new_read) */
    uint64_t offset;      /* in samples from `samples` */
    uint32_t n_samples;   /* 0 (with new_read == 0): no more signal for the read in progress */
    uint32_t dtype;       /* UNC_DTYPE_F32 / UNC_DTYPE_I16 */
    float cal_range, cal_offset, cal_digit;
} unc_chunk_desc;

#define UNC_STREAM_INACTIVE 0
#define UNC_STREAM_MAPPING 1
#define UNC_STREAM_SUCCESS 2   /* rec holds the mapping */
#define UNC_STREAM_FAILURE 3   /* gave up: max_events / max_chunks / no more signal (ended = 1 like Paf::set_ended) */

typedef struct {
    int32_t state, ended;
    uint32_t chunks;      /* chunks of the read consumed so far */
    uint32_t pad_;
    unc_paf_rec rec;      /* n_events = events detected so far, events_used = Mapper::event_i_ */
} unc_stream_result;

typedef struct unc_stream unc_stream;
int unc_stream_create(const unc_index *idx, const unc_params *prm, uint32_t n_channels, uint32_t max_chunk_len,
                      uint32_t max_chunks, unc_stream **out);
int unc_stream_step(unc_stream *st, const unc_chunk_desc *chunks, uint32_t n, const void *samples,
                    unc_stream_result *out);
/* Tie order of the per-event child sort for this stream's steps: see unc_pool_set_tie_order (1 = the reference's pdqsort
 * reproduced; applies from the next step on, the per-channel state is unaffected). */
int unc_stream_set_tie_order(unc_stream *st, int mode);
/* Mapper::PRMS.chunk_timeout (src/mapper.cpp:40,384-390; default there 4000 ms, FLT_MAX for `uncalled map` / sim,
 * conf.hpp:89-90): a read whose chunk has been with the mapper for longer fails and is marked ended.  Here a chunk is with
 * the mapper for the duration of the step that maps it, so the test is made once per step on the step's wall-clock time
 * (off until set).  The reference's evt_timeout only makes a thread yield and has no counterpart.  unc_stream_last_step_ms:
 * wall-clock time of the last step, copies included (the per-chunk decision latency a ReadUntil client sees). */
int unc_stream_set_chunk_timeout(unc_stream *st, float ms);
float unc_stream_last_step_ms(const unc_stream *st);
/* The channel's streaming normaliser (Mapper::norm_, src/normalizer.hpp:76-78) as the last step left it: mean_ and
 * varsum_ (Normalizer::get_mean = mean, get_stdv = sqrt(varsum / n)), n_ (events in the window, at most 6000) and the
 * ring cursor wr_.  Read-only; for inspection and tests. */
int unc_stream_channel_norm(const unc_stream *st, uint32_t channel, double *mean, double *varsum, uint32_t *n, uint32_t *wr);
void unc_stream_free(unc_stream *st);

/* ---- offline replay of whole reads (`uncalled_map_ord`) on a stream ---------------------------------
 *   unc_stream_replay   MapPoolOrd::update -> RealtimePool::try_add_chunk / is_read_finished / update, until every
 *                       read of the window is finished      src/map_pool_ord.cpp:61-121, src/realtime_pool.cpp:108-139
 * A window is a list of whole reads of any subset of the stream's channels; the reads of one channel are listed in the
 * order they follow each other on it (reads of different channels may interleave).  Each channel steps through its
 * reads on the device exactly as the lockstep loop of MapPoolOrd would: one step hands the front read its next chunk
 * (chunk i = samples [i*max_chunk_len, ...), the last one possibly partial), or, past the end of the signal, the empty
 * chunk that means "no more signal"; a read that finishes is replaced by the next one at the following step.  No host
 * round trip happens between the chunks of a channel.  The records depend only on the channel's earlier reads (the
 * reference accepts a channel's next chunk only once the previous one is mapped, and MAP_ORD has no timeouts), so a
 * run cut into several windows gives the records of one window.  The stream's chunk timeout does not apply.
 * Every descriptor is validated before any channel's state changes.  out[] receives one entry per read, in completion
 * order: by step, then kind, then channel, which is the order a lockstep loop over unc_stream_step returns them in.
 * UNC_E_OVERFLOW: a channel overflowed its seed-cluster workspace (that read's rec.status != 0; out[] is complete).
 * MapPoolOrd's min_active_reads is applied by the caller on the steps (api.MapPoolOrd, DESIGN.md section 4). */
typedef struct {
    uint32_t channel;     /* 0-based channel index */
    uint32_t number;      /* read number (ReadBuffer::number_), reported back */
    uint64_t offset;      /* in samples from `samples` */
    uint64_t n_samples;   /* > 0 */
    uint32_t dtype;       /* UNC_DTYPE_F32 / UNC_DTYPE_I16, one per window */
    float cal_range, cal_offset, cal_digit;
} unc_replay_read;

typedef struct {
    uint32_t read;        /* index of the read in the window */
    uint32_t number;      /* its read number */
    uint64_t step;        /* the channel's replay step that finished it (counted from 0 over all of the stream's
                             replays; a read that finishes at step s is followed by the next one at s + 1) */
    uint32_t kind;        /* 0: finished by the "no more signal" chunk, 1: by a chunk with samples */
    uint32_t pad_;
    unc_stream_result res;   /* as unc_stream_step reports the read's last step */
} unc_replay_result;

int unc_stream_replay(unc_stream *st, const unc_replay_read *reads, uint32_t n, const void *samples,
                      unc_replay_result *out);

/* ---- `uncalled index` after the BWA build ----------------------------------------------------------
 *   unc_self_align      self_align(bwa_prefix, sample_dist) -> vector<vector<u64>>
 *                                                      src/self_align_ref.cpp:34-91 (Python: src/pybinder.cpp:59,
 *                                                      called by IndexParameterizer, uncalled/index.py:82)
 * For every sampled reference position (glibc srand(0); rand() % sample_dist == 0, one draw per position) the
 * FM range lengths of the search that follows the reference until the range is unique.  Loads <prefix>.bwt /
 * .sa / .ann / .pac itself (no .uncl exists yet).  Result in CSR form: path i = (*values)[(*offsets)[i] ..
 * (*offsets)[i+1]), (*offsets) has *n_paths + 1 entries.  Both arrays are allocated by the library; release
 * each with unc_free. */
int unc_self_align(const char *bwa_prefix, uint32_t sample_dist, uint64_t *n_paths, uint64_t **offsets,
                   uint64_t **values);
void unc_free(void *p);

/* ---- DTW of event means against reference k-mers (analysis; SURVEY section 8(f) rank 4) ----------------------
 *   unc_dtw_batch       DTWr94p(means, kmers, prms) / DTWr94d(...) + get_path() / score()
 *                                                      src/dtw.hpp:31-183 (DTW<float, u16, Func>), :188-232 (the two
 *                                                      instances), bound at src/pybinder.cpp:75-91
 * Rows = k-mers, columns = event means.  cost_kind 0 = DTWr94p (cost = -match_prob of the r9.4 TEMPLATE model), 1 = DTWr94d
 * (cost = abs(e - mean_k) as the reference compiles it: int abs(int), the difference truncated towards zero first).
 * model_means_stdvs = the 1024 (mean, stdv) pairs of src/model_r94.inl (uncalled_b200/data/r94_5mer_template.f32).
 * unc_dtw_params = DTWParams (subseq: DTWSubSeq NONE 0 / ROW 1 / COL 2; dw, hw, vw).  Problem p: event means
 * means[mean_off[p] .. mean_off[p+1]), k-mers kmers[kmer_off[p] .. kmer_off[p+1]).  Out, per problem: get_path() as
 * (column, row) u64 pairs from the end cell back to the start at path[2*path_off[p] ...] (path_off[p+1] - path_off[p] >=
 * rows + columns), their number in path_len[p], score() in score[p]; mean_score() = score / path_len.  The matrices of
 * one call (one byte per cell) must fit the device memory: UNC_E_NOMEM otherwise. */
typedef struct { int32_t subseq; float dw, hw, vw; } unc_dtw_params;
int unc_dtw_batch(const float *model_means_stdvs, int cost_kind, const unc_dtw_params *prm, uint32_t n_problems,
                  const float *means, const uint64_t *mean_off, const uint16_t *kmers, const uint64_t *kmer_off,
                  uint64_t *path, const uint64_t *path_off, uint64_t *path_len, float *score);
/* unc_dtw_batch_banded: unc_dtw_batch restricted to a band of rows around the diagonal (the recurrence of
 * src/dtw.hpp:51-120, its traceback unchanged), for subseq NONE only (else UNC_E_ARG; band = 0 is UNC_E_ARG too).  Column
 * j of an R x C problem holds rows max(0, c - We) .. min(R-1, c + We), c = floor(j (R-1) / (C-1)) (0 when C = 1), We =
 * max(band, ceil((R-1) / (C-1))) (R - 1 when C = 1); a predecessor outside the band scores FLT_MAX / 2, as one outside the
 * matrix does.  Same outputs as unc_dtw_batch.  The score is never below the full sweep's and equals it whenever the full
 * path lies in the band; band >= R gives unc_dtw_batch's results.  The workspace holds one byte per in-band cell. */
int unc_dtw_batch_banded(const float *model_means_stdvs, int cost_kind, const unc_dtw_params *prm, uint32_t n_problems,
                         const float *means, const uint64_t *mean_off, const uint16_t *kmers, const uint64_t *kmer_off,
                         uint64_t *path, const uint64_t *path_off, uint64_t *path_len, float *score, uint32_t band);
/* The device workspace of unc_dtw_batch is kept between calls and grown on demand; unc_dtw_release (also called by
 * unc_shutdown) frees it.  unc_dtw_last_kernel_ms: CUDA-event time of the last call's sweep kernel. */
void unc_dtw_release(void);
float unc_dtw_last_kernel_ms(void);

/* ---- signal-level alignment of reads to reference spans (the reference's dtw_test driver) ---------------------
 *   unc_dtw_aligner_create  BwaIndex<KLEN> idx(prefix); idx.load_pacseq(); pmodel_r94_template
 *                                                      src/dtw_test.cpp:74-81 (host only: the device copy of the .pac is
 *                                                      made by the first batch)
 *   unc_dtw_aligner_contig  BwaIndex::coord_to_pacseq's contig lookup by name    src/bwa_index.hpp:226-233
 *   unc_dtw_align_batch     the loop body of dtw_test per query, for many reads at once   src/dtw_test.cpp:94-175:
 *                           EventDetector::get_events over the signal (no max_events cap), EventProfiler::get_full_mask
 *                           and the unmasked means, BwaIndex::get_kmers(rf_name, rf_st, rf_en) (+ kmers_revcomp unless
 *                           fwd), Normalizer(read_mean, read_stdv) from the span's template model means, the > 50 000
 *                           means skip, DTWr94d(means, kmers, {NONE, 1, 1, 1}) and mean_score()
 *   unc_dtw_align_path      DTW::get_path() of one aligned query of the last batch   src/dtw.hpp:124-126
 * reads[i] is the signal of query i: samples [rd_st, rd_en) of the read, as unc_map_batch takes them (one dtype per batch).
 * Every query gets a status: UNC_DTW_ALIGN_OK, or the reason it was skipped (the other queries are unaffected).  The
 * sweep runs in launches whose breadcrumb matrices (one byte per cell) and work arrays fit the budget (default: the free
 * device memory less 128 MiB); a query whose matrix alone exceeds it is skipped with UNC_DTW_ALIGN_TOO_LARGE.  Queries
 * skipped by the host checks (unknown contig, span past the contig's end or shorter than 5 bases, empty signal) never
 * reach the device: a batch made only of them does not touch it.  With keep_paths, unc_dtw_align_path copies query i's
 * path, path_len (column = event index, row = k-mer index) u64 pairs from the end cell back to the start, as
 * unc_dtw_batch returns them, and (each optional) its n_kept normalised means and its n_kmers = rf_en - rf_st - 4 k-mers.  unc_dtw_align_last_times: CUDA-event times of the last batch in ms (H2D, stages (a)-(e)
 * of unc_dtw_align.cuh, the sweep launches, total), the number of sweep launches and of matrix cells. */
#define UNC_DTW_ALIGN_OK 0
#define UNC_DTW_ALIGN_TOO_MANY_MEANS 1   /* more than 50 000 means after the mask (dtw_test.cpp:156-159) */
#define UNC_DTW_ALIGN_NO_EVENTS 2        /* no event left after the mask */
#define UNC_DTW_ALIGN_TOO_LARGE 3        /* the matrix alone exceeds the workspace budget */
#define UNC_DTW_ALIGN_UNKNOWN_CONTIG 4
#define UNC_DTW_ALIGN_SPAN_PAST_END 5    /* rf_en past the contig's end (or rf_st > rf_en) */
#define UNC_DTW_ALIGN_SPAN_SHORT 6       /* fewer than 5 bases: no k-mer */
#define UNC_DTW_ALIGN_EMPTY_SIGNAL 7
typedef struct unc_dtw_aligner unc_dtw_aligner;
typedef struct { int32_t rid; uint32_t fwd; uint64_t rf_st, rf_en; } unc_dtw_query;
typedef struct {
    int32_t status;
    uint32_t n_events, n_kept;       /* events detected; means left after the mask */
    float score, mean_score;
    uint32_t pad;
    uint64_t path_len;
} unc_dtw_align_result;
int unc_dtw_aligner_create(const char *bwa_prefix, const char *model_table_path, unc_dtw_aligner **out);
void unc_dtw_aligner_free(unc_dtw_aligner *a);
int unc_dtw_aligner_contig(const unc_dtw_aligner *a, const char *name, int32_t *rid, uint64_t *len);
int unc_dtw_aligner_set_budget(unc_dtw_aligner *a, uint64_t bytes);
/* unc_dtw_aligner_set_band: 0 (the default) aligns with the full matrix, as the reference does, and skips reads over 50 000
 * kept means; band >= 1 aligns with unc_dtw_batch_banded's sweep at that half-width (the recurrence of src/dtw.hpp:51-120
 * restricted to the band), where only the workspace budget limits a read's length: a query whose band alone exceeds it is
 * skipped with UNC_DTW_ALIGN_TOO_LARGE.  unc_dtw_align_last_times then counts in-band cells. */
int unc_dtw_aligner_set_band(unc_dtw_aligner *a, uint32_t band);
int unc_dtw_align_batch(unc_dtw_aligner *a, uint32_t n, const unc_read_desc *reads, const void *samples,
                        const unc_dtw_query *q, int keep_paths, unc_dtw_align_result *res);
int unc_dtw_align_path(const unc_dtw_aligner *a, uint32_t i, uint64_t *pairs, float *means, uint16_t *kmers);
int unc_dtw_align_last_times(const unc_dtw_aligner *a, float ms[8], uint64_t *launches, uint64_t *cells);

/* ---- iterative high-frequency k-mer masking of a reference (`mask-internal`) -----------------------------------
 *   unc_mask_internal   masking/mask_internal.sh <reference> <k> <iters> <out_prefix>: per iteration `jellyfish count`
 *                       (forward strand, no -C), the k-mer of the maximum count, masking/mask_kmers.py -k <kmer>
 * Each iteration counts the k-mers of the whole FASTA (bases case-insensitive; any other byte, a masked position or
 * a record boundary breaks a k-mer), takes the k-mer with the highest count -- ties go to the smallest 2-bit code
 * (A<C<G<T, the lexicographically smallest; jellyfish's choice is its hash order) -- and replaces every position of
 * every occurrence, overlapping ones included, by 'N'.  Iteration i's k-mer code (first base in the top bits) and
 * count go to kmer_codes[i] / counts[i]; when no k-mer is left the loop stops and *n_done < iters.  Only the final
 * FASTA is written to out_fasta: each header stripped, then the record's sequence on one line, '\n' line ends, every
 * byte not masked as in the input.  UNC_E_ARG (nothing written) for k outside 1..13, iters < 1, an empty file, a
 * first line not starting with '>' or a record without sequence; UNC_E_TOO_LARGE for 2^32 or more bases.
 * unc_mask_last_kernel_ms: CUDA-event time of the last call's device loop. */
int unc_mask_internal(const char *fasta_in, const char *out_fasta, uint32_t k, uint32_t iters, uint64_t *kmer_codes,
                      uint64_t *counts, uint32_t *n_done);
float unc_mask_last_kernel_ms(void);

/* ---- external repeat masking of a target against a full reference (`mask-external`) ----------------------------
 *   unc_mask_external   masking/mask_external.sh <full_bowtie> <target_fa> <min_len> <min_copy> <threads> <out_prefix>:
 *                       every full-length window of min_len bases of every target record (`bedtools makewindows -s 1`),
 *                       its exact hits on both strands of the full reference (`bowtie -fa -v 0`), the union of the
 *                       windows with more than min_copy hits masked (`bedtools merge` + `maskfasta`)
 * Both FASTA files are read as unc_mask_internal reads them.  A window's count is occ(w) + occ(revcomp(w)) over the
 * forward text of every full-reference record: bases are case-insensitive, any other byte and a record boundary break
 * an occurrence, a palindrome counts 2 per locus, counts saturate at UINT32_MAX.  A window with a non-ACGT byte has
 * count 0.  out_fasta: each stripped header, then the sequence on one line with the masked positions as 'N' and every
 * other byte as in the input.  out_bed: `name\tstart\tend` per maximal run of masked positions (0-based, half-open,
 * name = the header's first word), in record order.  window_counts (optional, one per target position in the order of
 * the records, one more between records): the count of the window starting there, 0 where none starts.  The full
 * reference is streamed through the device in pieces of piece_bases window starts (0 = 64 Mi), so device memory is
 * the target's table plus two pieces.  UNC_E_ARG (nothing written) for min_len outside 2..64, min_copy < 1, a missing
 * output directory, or either FASTA empty, not starting with '>' or with a record without sequence; UNC_E_TOO_LARGE
 * for 2^32 or more bases in either file.
 * unc_mask_external_last_kernel_ms: CUDA-event time of the last call's kernels.  unc_mask_external_last_times:
 * ms[0..3] = build, count (summed over the pieces), mark, and the count phase from the end of the build to the end of
 * the last count kernel (the part of it not spent in count kernels is copying and staging that was not hidden);
 * *h2d_bytes = the bytes copied to the device. */
int unc_mask_external(const char *full_fasta, const char *target_fasta, uint32_t min_len, uint32_t min_copy,
                      const char *out_fasta, const char *out_bed, uint64_t piece_bases, uint32_t *window_counts,
                      uint64_t *n_selected, uint64_t *n_masked_bp);
float unc_mask_external_last_kernel_ms(void);
void unc_mask_external_last_times(float ms[4], uint64_t *h2d_bytes);

/* ---- per-event view of the signal front end (`events`) -------------------------------------------------------
 *   unc_events_create     EventDetector(Params) + EventProfiler() + PoreModel loaded from a table: no FM index is needed
 *                         src/event_detector.cpp:17-38, src/event_profiler.cpp:3-9, src/pore_model.hpp:48-103
 *   unc_events_run        for every read, over its whole signal (no max_events cap):
 *                         EventDetector::get_events with create_event   src/event_detector.cpp:83-127,296-319
 *                         (mean, stdv, start, length of each event passing min_mean / max_mean, :104-108)
 *                         Normalizer::set_signal + at over the event means towards the model's mean and stdv, the
 *                         offline normaliser of Mapper::map_read        src/normalizer.cpp:31-44,114-118, src/mapper.cpp:193
 *                         EventProfiler::add_event / anno_event / get_full_mask   src/event_profiler.hpp:71-151
 *                         (the DEBUG_EVENTS columns win_mean, win_stdv, win_mask of src/mapper.cpp:894-905,968-989)
 *   unc_events_fetch      the events of the last run, reads in order
 *   unc_events_annotate   the normaliser and EventProfiler::get_full_mask over event means the caller supplies
 *   unc_match_probs_batch PoreModel::match_prob for many means at once  src/pore_model.hpp:163-165
 * Reads are described as for unc_map_batch (f32 pA, or i16 DAC calibrated on the device, one dtype per call).  win_mean
 * and win_stdv of an event are those of the add_event call after which it is next_evt_ (what anno_event() returns for
 * it); the last events of a read never get there and have NaN in both, and the tail loop of get_full_mask's mask.  The
 * scale and shift are the ones Normalizer::at computes (double division rounded to float), as the mapper applies them;
 * a read without events has scale = shift = 0.  Window lengths 3 / 6 and the profiler's 25-event window are fixed in
 * the device code (UNC_E_ARG otherwise).  Device memory: 32 bytes per sample of the largest run, plus the samples. */
typedef struct {
    uint32_t window_length1, window_length2;    /* 3, 6: fixed */
    float threshold1, threshold2, peak_height;  /* 1.4, 9.0, 0.2 */
    float min_mean, max_mean;                   /* 0, 400 */
    uint32_t win_len;                           /* EventProfiler::Params: 25, fixed */
    float win_stdv_min;                         /* 5 */
} unc_event_params;

typedef struct {          /* one event: Event (src/event_detector.hpp:19-24) and its annotations */
    uint32_t start;
    float length;         /* Event::length is an integer number of samples; exact in a float below 2^24 */
    float mean, stdv;
    float norm_mean;      /* scale * mean + shift */
    float win_mean, win_stdv;
    uint32_t win_mask;    /* 1: kept (get_full_mask true), 0: masked as a stall */
} unc_event_full;

typedef struct {
    uint32_t n_events;    /* events that passed the min_mean / max_mean filter */
    float mean_event_len; /* EventDetector::mean_event_len over every event, filtered or not (NaN without any) */
    float norm_scale, norm_shift;
} unc_event_read;

typedef struct unc_events unc_events;
int unc_event_params_default(unc_event_params *p);
/* model_table_path: 1024 x {mean, stdv} f32, template order (uncalled_b200/data/r94_5mer_template.f32 is the built-in
 * r9.4 model).  The device is the one selected by unc_init.  UNC_E_NO_DEVICE without a CUDA device. */
int unc_events_create(const char *model_table_path, const unc_event_params *prm, unc_events **out);
void unc_events_free(unc_events *h);
/* Synchronous.  samples_on_device: `samples` is a device pointer on the handle's device.  out[i]: read i's counts and
 * normaliser; the events stay on the device until unc_events_fetch or the next run. */
int unc_events_run(unc_events *h, const unc_read_desc *reads, uint32_t n_reads, const void *samples, int samples_on_device,
                   unc_event_read *out);
/* out: room for the sum of the last run's n_events; read i's events follow read i-1's. */
int unc_events_fetch(unc_events *h, unc_event_full *out);
/* The caller's event means: read i is means[off[i] .. off[i+1]).  Writes norm_mean, win_mean, win_stdv, win_mask of
 * each mean at the mean's own index (entries off[0] .. off[n_reads] of each array; any may be NULL) and scale / shift
 * per read (n_reads entries; may be NULL). */
int unc_events_annotate(unc_events *h, uint32_t n_reads, const uint64_t *off, const float *means, float *norm_mean,
                        float *win_mean, float *win_stdv, uint32_t *win_mask, float *scale, float *shift);
/* out[i * 1024 + k] = Mapper::model.match_prob(means[i], k): the model as the mapper holds it (pmodel_r94_complement,
 * src/mapper.cpp:57, built from the table as unc_index_load builds it), bit for bit what unc_match_probs returns for k. */
int unc_match_probs_batch(unc_events *h, const float *means, uint64_t n, float *out);
/* CUDA-event times of the last run in ms: H2D, detection, normaliser + profiler, D2H of the per-read results. */
int unc_events_last_times(const unc_events *h, float ms[4]);

/* ---- resource accounting (tests) -----------------------------------------------------------------------------
 * What the library holds at this moment: bytes of device memory, bytes of pinned host memory, and CUDA streams plus
 * events.  An object's free call, or the end of a call that holds nothing past its return, gives back what it took.
 * The DTW workspace stays held between unc_dtw_batch / unc_dtw_align_batch calls until unc_dtw_release. */
int unc_debug_held(uint64_t *device_bytes, uint64_t *pinned_bytes, uint32_t *handles);

/* ---- fast5 input (host; no libhdf5 needed) -------------------------------------------------------------
 *   unc_fast5_open      Fast5Reader::open_next: format detection and the list of reads
 *                                                      src/fast5_reader.cpp:134-177
 *   unc_fast5_info      ReadBuffer(hdf5_tools::File&, raw_path, ch_path): attributes as the reference parses
 *                       them (text -> atoi / atof)      src/read_buffer.cpp:198-225,
 *                                                      submods/fast5/include/fast5/hdf5_tools.hpp:1013-1141
 *   unc_fast5_load      the same constructor's `file.read(raw_path + "/Signal", int_data)` + truncation to
 *                       max_chunks * chunk_len samples  src/read_buffer.cpp:227-236
 *                       for a range of reads, decoded by several host threads into one staging buffer
 * The signal stays int16: unc_map_batch calibrates it on the device (unc_read_desc dtype 1) exactly as
 * src/read_buffer.cpp:239-242 does (u16 reinterpretation included). */
typedef struct {
    const char *read_id;        /* attribute read_id; valid until the next info/load call or close */
    int32_t number;             /* atoi(read_number) */
    int32_t start_sample;       /* atoi(start_time): 32 bit, like the reference */
    int32_t channel;            /* atoi(channel_number) -- what Paf prints as ch:i: */
    float cal_digitisation, cal_range, cal_offset;
    uint64_t n_samples;         /* after truncation, for unc_fast5_load */
    uint64_t sample_offset;     /* unc_fast5_load: where this read's samples start in dst */
} unc_fast5_read;

typedef struct unc_fast5 unc_fast5;
int unc_fast5_open(const char *path, unc_fast5 **out);
int unc_fast5_count(const unc_fast5 *f, uint32_t *n_reads, int *single_read_format);
int unc_fast5_info(unc_fast5 *f, uint32_t i, unc_fast5_read *info);
/* max_samples_per_read 0 = whole signals; threads 0 = all hardware threads.  UNC_E_TOO_LARGE when the signals
 * need more than `capacity` samples. */
int unc_fast5_load(unc_fast5 *f, uint32_t first, uint32_t n, uint64_t max_samples_per_read, int16_t *dst,
                   uint64_t capacity, unc_fast5_read *info, int threads);
void unc_fast5_close(unc_fast5 *f);
const char *unc_fast5_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
