// pyuncalled.cpp -- the `_uncalled` Python extension module over libunc_b200.so.
//
// The reference's Python package loads its C++ core as `_uncalled` (reference uncalled/__init__.py:1,
// src/pybinder.cpp:14-91).  This module carries the same names for the map / index / realtime paths -- Conf,
// Paf, MapPool, RealtimePool, Chunk, BwaIndex.create, self_align -- with the mapping done by the CUDA kernels
// behind include/unc_b200.h, so that the reference's own `scripts/uncalled index|map` and `uncalled/args.py`
// run unmodified with this module (and the reference's pure-Python `uncalled/` directory) on PYTHONPATH.
// Nothing here maps on the CPU: without a CUDA device MapPool(conf) raises.
//
// Build (uncalled_b200/_native.py build_pymodule): g++ -shared -fPIC $(python -m pybind11 --includes)
//        pyuncalled.cpp -L.. -lunc_b200 -Wl,-rpath,'$ORIGIN'
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <tuple>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <deque>
#include <fstream>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/unc_b200.h"

namespace py = pybind11;
typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

static void check(int rc, const char *what) {
    if (rc != UNC_OK && rc != UNC_E_OVERFLOW) throw std::runtime_error(std::string(what) + ": " + unc_last_error());
}

// ------------------------------------------------------------------ Conf (reference src/conf.hpp:57-340)
struct Conf {
    u16 threads = 1;
    std::string bwa_prefix, idx_preset = "default", model_path, dbg_prefix;
    u32 max_events = 30000, seed_len = 22, max_paths = 10000;            // src/mapper.cpp:29-52
    float chunk_time = 1.0f, sample_rate = 4000.0f, bp_per_sec = 450.0f;  // src/read_buffer.cpp:26-32
    u16 num_channels = 512;
    u32 max_chunks = 1000000;
    std::string fast5_list, read_list;                                    // src/fast5_reader.cpp:26-31
    u32 max_reads = 0, max_buffer = 100;
    std::string host = "127.0.0.1";                                       // src/realtime_pool.cpp:28-36
    u16 port = 8000;
    float duration = 72.0f;
    u32 max_active_reads = 512;
    int active_chs = 0, realtime_mode = 0;
    u32 min_active_reads = 0;
    std::string ctl_seqsum, unc_seqsum, unc_paf;
    float sim_speed = 1.0f, scan_time = 10.0f, scan_intv_time = 5400.0f, ej_time = 0.1f;
    u32 min_ch_reads = 10;
    // this module's own switches
    int device = 0;
    u32 batch_reads = 4096;
    int exact_ties = 0, ordered = 0;
    Conf() {}
    explicit Conf(const std::string &toml) {
        (void) toml;
        throw std::runtime_error("Conf(toml_file): TOML configuration files are not read by this module; set the attributes");
    }
    u32 chunk_len() const { return (u32) (u16) (chunk_time * sample_rate); }   // ReadBuffer::Params::chunk_len (u16), read_buffer.hpp:135-137
};

// ------------------------------------------------------------------ Paf (reference src/read_buffer.hpp:40-128, read_buffer.cpp:34-155)
struct Paf {
    enum Tag { MAP_TIME, WAIT_TIME, QUEUE_TIME, RECEIVE_TIME, CHANNEL, EJECT, READ_START, IN_SCAN, TOP_RATIO, MEAN_RATIO,
               ENDED, KEEP, DELAY, SEED_CLUSTER, CONFIDENT_EVENT };
    std::string rd_name, rf_name;
    bool mapped = false, ended = false, fwd = false;
    u64 rd_st = 0, rd_en = 0, rd_len = 0, rf_st = 0, rf_en = 0, rf_len = 0;
    u16 matches = 0;
    std::vector<std::pair<int, int>> int_tags;
    std::vector<std::pair<int, float>> float_tags;
    std::vector<std::pair<int, std::string>> str_tags;
    Paf() {}
    Paf(const std::string &name, u16 channel, u64 start_sample) : rd_name(name) {
        set_int(CHANNEL, channel);
        set_int(READ_START, (int) start_sample);
    }
    bool is_mapped() const { return mapped; }
    bool is_ended() const { return ended; }
    void set_ended() { ended = true; }
    void set_read_len(u64 n) { rd_len = n; }
    void set_mapped(u64 rd_st_, u64 rd_en_, const std::string &rf, u64 rf_st_, u64 rf_en_, u64 rf_len_, bool fwd_, u16 m) {
        mapped = true; rd_st = rd_st_; rd_en = rd_en_; rf_name = rf; rf_st = rf_st_; rf_en = rf_en_; rf_len = rf_len_; fwd = fwd_; matches = m;
    }
    void set_int(int t, int v) { int_tags.emplace_back(t, v); }
    void set_float(int t, float v) { float_tags.emplace_back(t, v); }
    void set_str(int t, const std::string &v) { str_tags.emplace_back(t, v); }
    std::string line() const {
        static const char *TAGS[] = {"mt", "wt", "qt", "rt", "ch", "ej", "st", "mx", "tr", "mr", "en", "kp", "dl", "sc", "ce"};
        std::string s = rd_name + "\t" + std::to_string(rd_len) + "\t";
        if (mapped) {
            s += std::to_string(rd_st) + "\t" + std::to_string(rd_en) + "\t" + (fwd ? "+" : "-") + "\t" + rf_name + "\t" +
                 std::to_string(rf_len) + "\t" + std::to_string(rf_st) + "\t" + std::to_string(rf_en) + "\t" +
                 std::to_string((unsigned) matches) + "\t" + std::to_string(rf_en - rf_st + 1) + "\t255";
        } else {
            s += "*\t*\t*\t*\t*\t*\t*\t*\t*\t255";
        }
        char buf[64];
        for (auto &t : int_tags) { snprintf(buf, sizeof(buf), "\t%s:i:%d", TAGS[t.first], t.second); s += buf; }
        for (auto &t : float_tags) { snprintf(buf, sizeof(buf), "\t%s:f:%.6f", TAGS[t.first], (double) t.second); s += buf; }
        for (auto &t : str_tags) s += std::string("\t") + TAGS[t.first] + ":Z:" + t.second;
        return s;
    }
    void print_paf() const { py::print(line()); }
};

static Paf paf_from_rec(const unc_index *idx, const unc_paf_rec &r, const std::string &id, u16 channel, u64 start) {
    Paf p(id, channel, start);                         // Mapper::set_ref_loc / set_failed (src/mapper.cpp:365-372,708-728)
    p.set_read_len(r.rd_len);
    if (r.mapped) {
        const char *name = "";
        uint64_t len = 0;
        if (r.rid >= 0) unc_index_seq(idx, r.rid, &name, &len);
        p.set_mapped(r.rd_st, r.rd_en, name, r.rf_st, r.rf_en, r.rf_len, r.fwd != 0, (u16) r.matches);
    }
    return p;
}

// shared: device + index + parameters from a Conf
struct Engine {
    unc_index *idx = nullptr;
    unc_params prm;
    explicit Engine(const Conf &c) {
        if (c.bwa_prefix.empty()) throw std::runtime_error("Conf.bwa_prefix is not set");
        check(unc_init(c.device), "unc_init");
        std::string table = c.model_path.empty() ? default_model_table() : c.model_path;
        check(unc_index_load(c.bwa_prefix.c_str(), c.idx_preset.c_str(), table.c_str(), &idx), "unc_index_load");
        unc_params_default(&prm);
        prm.max_events = c.max_events; prm.max_paths = c.max_paths; prm.seed_len = c.seed_len;
        prm.bp_per_sec = c.bp_per_sec; prm.sample_rate = c.sample_rate;
    }
    ~Engine() { if (idx) unc_index_free(idx); }
    static std::string default_model_table() {
        py::object here = py::module_::import("os").attr("path").attr("dirname")(py::module_::import("_uncalled").attr("__file__"));
        return py::str(here).cast<std::string>() + "/data/r94_5mer_template.f32";
    }
};

// ------------------------------------------------------------------ MapPool (reference src/map_pool.hpp:33-53, map_pool.cpp:28-158)
class MapPool {
    Conf conf_;
    Engine eng_;
    unc_pool *pool_ = nullptr;
    u32 cap_reads_ = 0;
    u64 cap_samples_ = 0;
    std::deque<std::string> files_;
    unc_fast5 *open_ = nullptr;
    u32 next_ = 0, open_n_ = 0;
    std::set<std::string> filter_;
    bool use_filter_ = false, stopped_ = false;
    u32 n_added_ = 0;
    uint32_t carry_[32];

    u64 max_len() const { return (u64) conf_.max_chunks * conf_.chunk_len(); }   // src/read_buffer.cpp:229-234
    bool input_left() {
        if (conf_.max_reads && n_added_ >= conf_.max_reads) {                      // Fast5Reader::all_buffered
            if (open_) { unc_fast5_close(open_); open_ = nullptr; }
            files_.clear();
        }
        return open_ != nullptr || !files_.empty();
    }

  public:
    explicit MapPool(Conf &conf) : conf_(conf), eng_(conf) {
        memset(carry_, 0, sizeof(carry_));
        if (!conf.fast5_list.empty()) {                                          // Fast5Reader::load_fast5_list, src/fast5_reader.cpp:77-92
            std::ifstream in(conf.fast5_list);
            for (std::string l; std::getline(in, l);) if (!l.empty()) files_.push_back(l);
        }
        if (!conf.read_list.empty()) {
            use_filter_ = true;
            std::ifstream in(conf.read_list);
            for (std::string l; std::getline(in, l);) if (!l.empty()) filter_.insert(l);
        }
    }
    ~MapPool() { stop(); }
    void add_fast5(const std::string &name) { files_.push_back(name); }         // Fast5Reader::add_fast5
    bool running() { return !stopped_ && input_left(); }
    void stop() {
        stopped_ = true;
        if (open_) { unc_fast5_close(open_); open_ = nullptr; }
        if (pool_) { unc_pool_free(pool_); pool_ = nullptr; }
    }

    // One batch: decode up to conf.batch_reads reads (int16 DAC values, calibrated on the device), map them on the
    // GPU, hand back their Paf records (the reference returns whatever its threads finished, src/map_pool.cpp:45-69).
    std::vector<Paf> update() {
        std::vector<Paf> out;
        if (stopped_) return out;
        std::vector<unc_fast5_read> infos;
        std::vector<std::string> ids;                 // unc_fast5_read::read_id is only valid until the next fast5 call
        std::vector<int16_t> samples;
        const u64 cap = max_len();
        while (infos.size() < conf_.batch_reads && input_left()) {
            if (!open_) {
                const std::string path = files_.front();
                files_.pop_front();
                if (unc_fast5_open(path.c_str(), &open_) != 0) { open_ = nullptr; throw std::runtime_error(std::string("fast5: ") + unc_fast5_last_error()); }
                int single = 0;
                unc_fast5_count(open_, &open_n_, &single);
                next_ = 0;
            }
            u32 want = conf_.batch_reads - (u32) infos.size(), n = std::min(want, open_n_ - next_);
            if (conf_.max_reads) n = std::min(n, conf_.max_reads - n_added_ + 0u);
            // pick the reads that pass the read-list filter (their ids come with unc_fast5_info)
            std::vector<u32> take;
            for (u32 i = 0; i < n; i++) {
                unc_fast5_read inf;
                if (unc_fast5_info(open_, next_ + i, &inf) != 0) throw std::runtime_error(std::string("fast5: ") + unc_fast5_last_error());
                if (use_filter_ && !filter_.count(inf.read_id ? inf.read_id : "")) continue;
                take.push_back(next_ + i);
            }
            for (u32 k = 0; k < take.size();) {                                  // load runs of consecutive reads in one call
                u32 e = k + 1;
                while (e < take.size() && take[e] == take[e - 1] + 1) e++;
                const u32 cnt = e - k;
                std::vector<unc_fast5_read> inf(cnt);
                u64 total = 0;
                for (u32 i = 0; i < cnt; i++) {
                    unc_fast5_info(open_, take[k + i], &inf[i]);
                    total += cap ? std::min<u64>(inf[i].n_samples, cap) : inf[i].n_samples;
                }
                const size_t base = samples.size();
                samples.resize(base + total + 1);
                if (unc_fast5_load(open_, take[k], cnt, cap, samples.data() + base, total, inf.data(), conf_.threads) != 0)
                    throw std::runtime_error(std::string("fast5: ") + unc_fast5_last_error());
                samples.resize(base + total);
                for (u32 i = 0; i < cnt; i++) { inf[i].sample_offset += base; ids.push_back(inf[i].read_id ? inf[i].read_id : ""); infos.push_back(inf[i]); }
                n_added_ += cnt;
                k = e;
            }
            next_ += n;
            if (next_ >= open_n_ || n == 0) { unc_fast5_close(open_); open_ = nullptr; }
        }
        if (infos.empty()) return out;
        const u32 n = (u32) infos.size();
        if (!pool_ || n > cap_reads_ || samples.size() > cap_samples_) {
            if (pool_) unc_pool_free(pool_);
            cap_reads_ = std::max<u32>(n, std::max<u32>(cap_reads_, 64));
            cap_samples_ = std::max<u64>(samples.size(), std::max<u64>(cap_samples_, 1u << 20));
            check(unc_pool_create(eng_.idx, &eng_.prm, cap_reads_, cap_samples_, &pool_), "unc_pool_create");
            if (conf_.exact_ties) check(unc_pool_set_tie_order(pool_, 1), "unc_pool_set_tie_order");
        }
        std::vector<unc_read_desc> d(n);
        for (u32 i = 0; i < n; i++) {
            d[i].offset = infos[i].sample_offset; d[i].n_samples = (u32) infos[i].n_samples; d[i].dtype = UNC_DTYPE_I16;
            d[i].cal_range = infos[i].cal_range; d[i].cal_offset = infos[i].cal_offset; d[i].cal_digit = infos[i].cal_digitisation;
        }
        std::vector<unc_paf_rec> rec(n);
        const auto t0 = std::chrono::steady_clock::now();
        {
            py::gil_scoped_release nogil;
            int rc = conf_.ordered ? unc_map_batch_ordered(pool_, d.data(), n, samples.data(), 0, carry_, rec.data(), nullptr, nullptr)
                                   : unc_map_batch(pool_, d.data(), n, samples.data(), rec.data());
            if (rc != UNC_OK && rc != UNC_E_OVERFLOW) { py::gil_scoped_acquire gil; throw std::runtime_error(unc_last_error()); }
        }
        const float ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count() / n;
        for (u32 i = 0; i < n; i++) {
            if (rec[i].status != 0)
                fprintf(stderr, "Warning: read %s overflowed its device workspace; reported unmapped\n", ids[i].c_str());
            Paf p = paf_from_rec(eng_.idx, rec[i], ids[i], (u16) infos[i].channel, (u64) (u32) infos[i].start_sample);
            p.set_float(Paf::MAP_TIME, ms);
            out.push_back(p);
        }
        return out;
    }
};

// ------------------------------------------------------------------ Chunk (reference src/chunk.hpp:33-81)
struct Chunk {
    std::string id;
    u16 channel = 1;
    u32 number = 0;
    u64 start = 0;
    std::vector<float> raw;
    Chunk() {}
    Chunk(const std::string &id_, u16 ch, u32 num, u64 st, const std::vector<float> &raw_, u32 raw_st, u32 raw_len)
        : id(id_), channel(ch), number(num), start(st) {
        if (raw_st > raw_.size()) raw_st = (u32) raw_.size();
        if ((u64) raw_st + raw_len > raw_.size()) raw_len = (u32) raw_.size() - raw_st;   // Chunk::Chunk clips (src/chunk.cpp:74-83)
        raw.assign(raw_.begin() + raw_st, raw_.begin() + raw_st + raw_len);
    }
    // the MinKNOW form (scripts/uncalled:270-275): raw bytes of `dtype` ("float32" | "int16" -- pA values either way)
    Chunk(const std::string &id_, u16 ch, u32 num, u64 st, const std::string &dtype, const std::string &bytes)
        : id(id_), channel(ch), number(num), start(st) {
        if (dtype == "float32") { raw.resize(bytes.size() / 4); memcpy(raw.data(), bytes.data(), raw.size() * 4); }
        else if (dtype == "int16") { raw.resize(bytes.size() / 2); const int16_t *p = (const int16_t *) bytes.data(); for (size_t i = 0; i < raw.size(); i++) raw[i] = (float) p[i]; }
        else throw std::runtime_error("Chunk: unsupported raw dtype " + dtype);
    }
    size_t size() const { return raw.size(); }
    bool empty() const { return raw.empty(); }
};

// ------------------------------------------------------------------ RealtimePool (reference src/realtime_pool.hpp:33-91, realtime_pool.cpp:38-261)
class RealtimePool {
    Conf conf_;
    Engine eng_;
    unc_stream *st_ = nullptr;
    struct Chan { bool active = false, has_chunk = false, new_read = false; u32 number = 0; Chunk chunk; std::string id; u64 start = 0; };
    std::vector<Chan> ch_;

  public:
    enum Mode { DEPLETE, ENRICH };
    enum ActiveChs { FULL, EVEN, ODD };
    explicit RealtimePool(Conf &conf) : conf_(conf), eng_(conf), ch_(conf.num_channels) {
        check(unc_stream_create(eng_.idx, &eng_.prm, conf.num_channels, std::max<u32>(conf.chunk_len(), 1), conf.max_chunks, &st_), "unc_stream_create");
        if (conf.exact_ties) check(unc_stream_set_tie_order(st_, 1), "unc_stream_set_tie_order");
    }
    ~RealtimePool() { stop_all(); }
    // RealtimePool::add_chunk + try_add_chunk (src/realtime_pool.cpp:74-139): one buffered chunk per channel; a chunk of a
    // new read replaces what the channel was doing
    bool add_chunk(Chunk &c) {
        if (c.channel < 1 || c.channel > ch_.size()) return false;
        Chan &h = ch_[c.channel - 1];
        if (h.active && h.number == c.number && h.has_chunk) return false;        // the previous chunk is not mapped yet
        h.new_read = !h.active || h.number != c.number;
        h.active = true; h.number = c.number; h.id = c.id; h.start = h.new_read ? c.start : h.start;
        h.chunk = c; h.has_chunk = true;
        c.raw.clear();
        return true;
    }
    bool try_add_chunk(Chunk &c) { return add_chunk(c); }
    // RealtimePool::update (src/realtime_pool.cpp:141-261): map the buffered chunk of every channel in ONE device step
    std::vector<std::tuple<u16, u32, Paf>> update() {
        std::vector<std::tuple<u16, u32, Paf>> ret;
        std::vector<unc_chunk_desc> d;
        std::vector<float> samples;
        std::vector<u32> who;
        for (u32 c = 0; c < ch_.size(); c++) {
            Chan &h = ch_[c];
            if (!h.active || !h.has_chunk) continue;
            unc_chunk_desc x;
            memset(&x, 0, sizeof(x));
            x.channel = c; x.new_read = h.new_read ? 1 : 0; x.offset = samples.size(); x.n_samples = (u32) h.chunk.raw.size();
            x.dtype = UNC_DTYPE_F32; x.cal_range = 1.f; x.cal_offset = 0.f; x.cal_digit = 1.f;
            samples.insert(samples.end(), h.chunk.raw.begin(), h.chunk.raw.end());
            d.push_back(x); who.push_back(c);
            h.has_chunk = false; h.new_read = false;
        }
        if (d.empty()) return ret;
        if (samples.empty()) samples.push_back(0.f);
        std::vector<unc_stream_result> r(d.size());
        {
            py::gil_scoped_release nogil;
            int rc = unc_stream_step(st_, d.data(), (u32) d.size(), samples.data(), r.data());
            if (rc != UNC_OK && rc != UNC_E_OVERFLOW) { py::gil_scoped_acquire gil; throw std::runtime_error(unc_last_error()); }
        }
        for (size_t i = 0; i < d.size(); i++) {
            if (r[i].state == UNC_STREAM_MAPPING) continue;                         // SUCCESS or FAILURE: the read is finished
            Chan &h = ch_[who[i]];
            Paf p = paf_from_rec(eng_.idx, r[i].rec, h.id, (u16) (who[i] + 1), h.start);
            if (r[i].ended) p.set_ended();
            ret.emplace_back((u16) (who[i] + 1), h.number, p);
            h.active = false;
        }
        return ret;
    }
    bool all_finished() const { for (auto &h : ch_) if (h.active) return false; return true; }
    void stop_all() { if (st_) { unc_stream_free(st_); st_ = nullptr; } }
};

// ------------------------------------------------------------------ index side
// Range (reference src/range.hpp:34-68, src/range.cpp)
struct Range {
    u64 start_ = 1, end_ = 0;
    Range() = default;
    Range(u64 s, u64 e) : start_(s), end_(e) {}
    bool is_valid() const { return start_ <= end_; }
    u64 length() const { return end_ - start_ + 1; }
    bool intersects(const Range &q) const {
        return is_valid() && q.is_valid() && !(start_ > q.end_ || end_ < q.start_) && !(q.start_ > end_ || q.end_ < start_);
    }
    Range intersect(const Range &r) const { return intersects(r) ? Range(std::max(start_, r.start_), std::min(end_, r.end_)) : Range(); }
    Range merge(const Range &r) const { return intersects(r) ? Range(std::min(start_, r.start_), std::max(end_, r.end_)) : Range(); }
    float get_recp_overlap(const Range &r) const {
        return intersects(r) ? float(intersect(r).length()) / float(merge(r).length()) : 0.f;
    }
    Range split_range(const Range &r) {
        Range left;
        if (start_ < r.start_) { left = *this; left.end_ = r.start_ - 1; }
        if (start_ <= r.end_) {
            if (end_ > r.end_) start_ = r.end_ + 1;
            else { start_ = 1; end_ = 0; }
        }
        return left;
    }
    bool same_range(const Range &q) const { return start_ == q.start_ && end_ == q.end_; }
    bool operator<(const Range &q) const { return start_ < q.start_ || (start_ == q.start_ && end_ < q.end_); }
    bool operator==(const Range &q) const { return same_range(q); }
};

// k-mer helpers of src/bp.hpp for k = 5
static const u8 KLEN = 5;
static u16 kmer_count() { return 1024; }
static u16 str_to_kmer(const std::string &kmer, u64 offset) {
    auto b = [](char c) -> u16 {
        switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2;
                     case 'T': case 't': return 3; default: return 4; }
    };
    if (offset + KLEN > kmer.size()) throw std::out_of_range("k-mer string too short");
    u16 index = b(kmer[offset]);
    for (u8 i = 1; i < KLEN; i++) index = (u16) ((index << 2) | b(kmer[offset + i]));
    return index;
}
static u16 kmer_comp(u16 kmer) { return kmer ^ 0x3FF; }
static u16 kmer_revcomp(u16 kmer) {          // complement, then reverse the order of the 2-bit bases
    u16 x = (kmer ^ 0x3FF) & 0x3FF, r = 0;
    for (u8 i = 0; i < KLEN; i++) { r = (u16) ((r << 2) | (x & 3)); x >>= 2; }
    return r;
}
static u8 kmer_head(u16 kmer) { return (u8) ((kmer >> (2 * KLEN - 2)) & 3); }
static u16 kmer_neighbor(u16 kmer, u8 i) { return (u16) (((kmer << 2) & 0x3FF) | i); }
static u8 kmer_base(u16 kmer, u8 i) {
    if (i >= KLEN) throw std::out_of_range("base index outside the k-mer");
    return (u8) ((kmer >> (2 * (KLEN - i - 1))) & 3);
}
static std::string kmer_to_str(u16 kmer) {
    std::string s(KLEN, 'N');
    for (u8 i = 0; i < KLEN; i++) s[i] = "ACGT"[kmer_base(kmer, i)];
    return s;
}

// BwaIndex<5> (reference src/bwa_index.hpp:88-377) over unc_bwa_*: FM-index queries on the GPU, the rest on the host
struct BwaIndex {
    unc_bwa *h_ = nullptr;
    std::vector<Range> kr_;
    BwaIndex() = default;
    BwaIndex(const std::string &prefix, bool pacseq) {
        if (!prefix.empty()) load_index(prefix);
        if (pacseq) load_pacseq();
    }
    ~BwaIndex() { destroy(); }
    BwaIndex(const BwaIndex &) = delete;
    BwaIndex &operator=(const BwaIndex &) = delete;

    static void create(const std::string &fasta, const std::string &prefix) {        // BwaIndex::create, src/bwa_index.hpp:92-101
        // the device builder where a CUDA device is visible; both write the same files
        if (unc_device_count() > 0) check(unc_index_build_device(fasta.c_str(), prefix.c_str()), "unc_index_build_device");
        else check(unc_index_build(fasta.c_str(), prefix.c_str()), "unc_index_build");
    }
    void load_index(const std::string &prefix) {
        destroy();
        check(unc_bwa_open(prefix.c_str(), 0, 0, &h_), "unc_bwa_open");
    }
    bool is_loaded() const { return h_ != nullptr; }
    unc_bwa *hd() const {
        if (!h_) throw std::runtime_error("no index loaded");
        return h_;
    }
    void load_pacseq() { check(unc_bwa_load_pac(hd()), "unc_bwa_load_pac"); }
    bool pacseq_loaded() const {
        int32_t pl = 0;
        if (h_) check(unc_bwa_info(h_, nullptr, nullptr, nullptr, &pl, nullptr), "unc_bwa_info");
        return pl != 0;
    }
    void destroy() {
        if (h_) unc_bwa_free(h_);
        h_ = nullptr;
        kr_.clear();
    }
    Range get_neighbor(Range r, u8 base) const {
        u64 s, e;
        check(unc_bwa_neighbor(hd(), 1, &r.start_, &r.end_, &base, &s, &e), "unc_bwa_neighbor");
        return Range(s, e);
    }
    const std::vector<Range> &kmer_ranges() {
        if (kr_.empty()) {
            std::vector<u64> st(1024), en(1024);
            check(unc_bwa_kmer_ranges(hd(), st.data(), en.data()), "unc_bwa_kmer_ranges");
            for (int k = 0; k < 1024; k++) kr_.emplace_back(st[k], en[k]);
        }
        return kr_;
    }
    Range get_kmer_range(u16 kmer) { return kmer_ranges().at(kmer); }
    u64 get_kmer_count(u16 kmer) { return get_kmer_range(kmer).length(); }
    u64 L2(int b) const {
        u64 l2[5];
        check(unc_bwa_info(hd(), nullptr, nullptr, nullptr, nullptr, l2), "unc_bwa_info");
        return l2[b];
    }
    Range get_base_range(u8 base) const {
        if (base > 3) throw std::out_of_range("base above 3");
        return Range(L2(base), L2(base + 1));
    }
    u64 sa(u64 i) const {
        u64 v;
        check(unc_bwa_sa(hd(), 1, &i, &v), "unc_bwa_sa");
        return v;
    }
    u64 size() const {
        u64 n;
        check(unc_bwa_info(hd(), &n, nullptr, nullptr, nullptr, nullptr), "unc_bwa_info");
        return n;
    }
    void seq(int rid, const char **name, u64 *off, u64 *len) const { check(unc_bwa_seq(hd(), rid, name, off, len), "unc_bwa_seq"); }
    int get_rid(u64 sa_loc) const { return unc_bwa_pos2rid(hd(), sa_loc); }
    std::pair<int, u32> get_ref_coord(u64 sa_loc) const {
        const int rid = get_rid(sa_loc);
        u64 off;
        seq(rid, nullptr, &off, nullptr);
        return {rid, (u32) (sa_loc - off)};
    }
    std::string get_ref_name(int rid) const { const char *nm; seq(rid, &nm, nullptr, nullptr); return nm; }
    u64 get_ref_len(int rid) const { u64 len; seq(rid, nullptr, nullptr, &len); return len; }
    u64 get_sa_loc(const std::string &name, u64 coord) const {
        const u64 p = coord_to_pacseq(name, coord);
        return p == (u64) INT_MAX && !has_seq(name) ? 0 : p;
    }
    bool has_seq(const std::string &name) const {
        int32_t n = 0;
        check(unc_bwa_info(hd(), nullptr, nullptr, &n, nullptr, nullptr), "unc_bwa_info");
        for (int i = 0; i < n; i++) if (get_ref_name(i) == name) return true;
        return false;
    }
    // translate_loc(sa_loc, &ref_name, &ref_loc) returns through its arguments in C++: here (ref_len, ref_name, ref_loc)
    std::tuple<u64, std::string, u64> translate_loc(u64 sa_loc) const {
        const int rid = get_rid(sa_loc);
        if (rid < 0) return std::make_tuple((u64) 0, std::string(), (u64) 0);
        const char *nm;
        u64 off, len;
        seq(rid, &nm, &off, &len);
        return std::make_tuple(len, std::string(nm), sa_loc - off);
    }
    std::vector<std::pair<std::string, u64>> get_seqs() const {
        int32_t n = 0;
        check(unc_bwa_info(hd(), nullptr, nullptr, &n, nullptr, nullptr), "unc_bwa_info");
        std::vector<std::pair<std::string, u64>> ret;
        for (int i = 0; i < n; i++) ret.emplace_back(get_ref_name(i), get_ref_len(i));
        return ret;
    }
    u64 coord_to_pacseq(const std::string &name, u64 coord) const {
        u64 p;
        check(unc_bwa_coord_to_pacseq(hd(), name.c_str(), coord, &p), "unc_bwa_coord_to_pacseq");
        return p;
    }
    u8 get_base(u64 i) const {
        u8 b;
        check(unc_bwa_get_base(hd(), i, &b), "unc_bwa_get_base");
        return b;
    }
    std::vector<u16> get_kmers(u64 st, u64 en) {
        std::vector<u16> ret(en > st + 4 ? en - st - 4 : 0);
        check(unc_bwa_get_kmers(hd(), st, en, ret.data()), "unc_bwa_get_kmers");
        return ret;
    }
    std::vector<u16> get_kmers_named(std::string nm, u64 st, u64 en) { return get_kmers(coord_to_pacseq(nm, st), coord_to_pacseq(nm, en)); }
    std::pair<std::vector<u64>, std::vector<u64>> range_to_fms(std::string ref_name, u64 start, u64 end) {
        const u64 n = end > start ? end - start : 0;
        std::vector<u64> first(n ? n : 1), second(n ? n : 1);
        check(unc_bwa_range_to_fms(hd(), ref_name.c_str(), start, end, first.data(), second.data()), "unc_bwa_range_to_fms");
        first.resize(n); second.resize(n);
        return {first, second};
    }
};
static std::vector<std::vector<u64>> self_align(const std::string &prefix, u32 sample_dist) {   // src/self_align_ref.cpp:34-91
    uint64_t n = 0, *off = nullptr, *val = nullptr;
    check(unc_self_align(prefix.c_str(), sample_dist, &n, &off, &val), "unc_self_align");
    std::vector<std::vector<u64>> ret(n);
    for (uint64_t i = 0; i < n; i++) ret[i].assign(val + off[i], val + off[i + 1]);
    unc_free(off); unc_free(val);
    return ret;
}
// ------------------------------------------------------------------ DTW (reference src/dtw.hpp:9-28,188-232, src/pybinder.cpp:75-91)
struct DTWParams { int32_t subseq; float dw, hw, vw; };          // = unc_dtw_params; subseq: DTWSubSeq NONE 0, ROW 1, COL 2
static const DTWParams DTW_EVENT_GLOB = {0, 2, 1, 100}, DTW_EVENT_QSUB = {2, 2, 1, 100}, DTW_EVENT_RSUB = {1, 2, 1, 100},
                       DTW_RAW_GLOB = {0, 10, 1, 1000};
template <int COST>
class DTWr94 {
    std::vector<std::pair<u64, u64>> path_;
    float score_ = 0;
  public:
    DTWr94(const std::vector<float> &means, const std::vector<uint16_t> &kmers, const DTWParams &p) {
        std::string table = Engine::default_model_table();
        std::vector<float> model(2048);
        FILE *fp = fopen(table.c_str(), "rb");
        if (!fp || fread(model.data(), 4, 2048, fp) != 2048) { if (fp) fclose(fp); throw std::runtime_error("cannot read " + table); }
        fclose(fp);
        const uint64_t moff[2] = {0, means.size()}, koff[2] = {0, kmers.size()}, poff[2] = {0, means.size() + kmers.size()};
        std::vector<uint64_t> path(2 * poff[1] + 2);
        uint64_t n = 0;
        unc_dtw_params prm = {p.subseq, p.dw, p.hw, p.vw};
        check(unc_dtw_batch(model.data(), COST, &prm, 1, means.data(), moff, kmers.data(), koff, path.data(), poff, &n, &score_), "unc_dtw_batch");
        path_.resize(n);
        for (uint64_t i = 0; i < n; i++) path_[i] = {path[2 * i], path[2 * i + 1]};
    }
    std::vector<std::pair<u64, u64>> get_path() { return path_; }
    float score() { return score_; }
    float mean_score() { return score_ / path_.size(); }
};

struct ClientSim {
    explicit ClientSim(Conf &) { throw std::runtime_error("ClientSim (`uncalled sim`) is outside the scope of this module"); }
};

// ------------------------------------------------------------------ signal front end (reference src/pybinder.cpp:44-56)
// Event, EventDetector, EventProfiler and PoreModel with the reference's names, computed by the `events` kernels
// (unc_events_*).  Only whole-signal / whole-read methods are offered: the per-sample and streaming ones (add_sample,
// add_event, Normalizer push / pop) would cost one GPU launch per sample or event and are deliberately left out.
struct Event { float mean = 0, stdv = 0; u32 start = 0, length = 0; };   // src/event_detector.hpp:19-24

static unc_events *events_create(const unc_event_params &p) {
    unc_events *h = nullptr;
    check(unc_events_create(Engine::default_model_table().c_str(), &p, &h), "unc_events_create");
    return h;
}

// EventDetector (src/event_detector.cpp:17-153): get_events / get_means over a whole signal, mean_event_len of the last
class EventDetector {
    unc_event_params prm_;
    unc_events *h_ = nullptr;
    float mel_ = NAN;
    std::vector<unc_event_full> run(const std::vector<float> &raw) {
        if (!h_) h_ = events_create(prm_);
        unc_read_desc d = {0, (u32) raw.size(), UNC_DTYPE_F32, 1.0f, 0.0f, 1.0f};
        unc_event_read r;
        std::vector<float> buf(raw.empty() ? 1 : raw.size());
        std::copy(raw.begin(), raw.end(), buf.begin());
        check(unc_events_run(h_, &d, 1, buf.data(), 0, &r), "unc_events_run");
        std::vector<unc_event_full> ev(r.n_events);
        if (r.n_events) check(unc_events_fetch(h_, ev.data()), "unc_events_fetch");
        mel_ = r.mean_event_len;
        return ev;
    }
  public:
    EventDetector() { unc_event_params_default(&prm_); }
    explicit EventDetector(const unc_event_params &p) : prm_(p) {
        if (p.window_length1 != 3 || p.window_length2 != 6) throw std::invalid_argument("window lengths are fixed at 3 and 6");
    }
    ~EventDetector() { if (h_) unc_events_free(h_); }
    EventDetector(const EventDetector &) = delete;
    std::vector<Event> get_events(const std::vector<float> &raw) {
        std::vector<Event> out;
        for (const unc_event_full &e : run(raw)) out.push_back(Event{e.mean, e.stdv, e.start, (u32) e.length});
        return out;
    }
    std::vector<float> get_means(const std::vector<float> &raw) {
        std::vector<float> out;
        for (const unc_event_full &e : run(raw)) out.push_back(e.mean);
        return out;
    }
    float mean_event_len() const { return mel_; }
};

// EventProfiler (src/event_profiler.hpp:14-151, defaults src/event_profiler.cpp:3-9): get_full_mask over given events
class EventProfiler {
    unc_events *h_ = nullptr;
  public:
    EventProfiler() = default;
    ~EventProfiler() { if (h_) unc_events_free(h_); }
    EventProfiler(const EventProfiler &) = delete;
    std::vector<bool> get_full_mask(const std::vector<Event> &events) {
        if (!h_) { unc_event_params p; unc_event_params_default(&p); h_ = events_create(p); }
        std::vector<float> means(events.size() + 1);
        for (size_t i = 0; i < events.size(); i++) means[i] = events[i].mean;
        const uint64_t off[2] = {0, events.size()};
        std::vector<uint32_t> mask(events.size() + 1);
        check(unc_events_annotate(h_, 1, off, means.data(), nullptr, nullptr, nullptr, mask.data(), nullptr, nullptr),
              "unc_events_annotate");
        return std::vector<bool>(mask.begin(), mask.begin() + events.size());
    }
};

// PoreModel (src/pore_model.hpp:163-165): match_prob of the r9.4 model in template or complement k-mer order (the
// mapper holds the complement one, src/mapper.cpp:57)
class PoreModel {
    bool complement_;
    unc_events *h_ = nullptr;
  public:
    explicit PoreModel(bool complement) : complement_(complement) {}
    ~PoreModel() { if (h_) unc_events_free(h_); }
    PoreModel(const PoreModel &o) : complement_(o.complement_) {}
    py::array_t<float> match_probs(py::array_t<float, py::array::c_style | py::array::forcecast> means) {
        if (!h_) { unc_event_params p; unc_event_params_default(&p); h_ = events_create(p); }
        const uint64_t n = (uint64_t) means.size();
        py::array_t<float> dev({(py::ssize_t) n, (py::ssize_t) 1024});
        if (n) check(unc_match_probs_batch(h_, means.data(), n, dev.mutable_data()), "unc_match_probs_batch");
        if (complement_) return dev;
        // the device table is in complement order: template k-mer k sits at k ^ 0x3FF (src/bp.hpp:77-80)
        py::array_t<float> out({(py::ssize_t) n, (py::ssize_t) 1024});
        for (uint64_t i = 0; i < n; i++)
            for (u32 k = 0; k < 1024; k++) out.mutable_data()[i * 1024 + k] = dev.data()[i * 1024 + (k ^ 0x3FFu)];
        return out;
    }
    float match_prob(float samp, u16 kmer) {
        if (kmer >= 1024) throw std::invalid_argument("k-mer out of range");
        py::array_t<float> m(1);
        m.mutable_data()[0] = samp;
        return match_probs(m).data()[kmer];
    }
};

static u32 fixed_window(u32 v, u32 want) {
    if (v != want) throw std::invalid_argument("the event window lengths are fixed at 3 and 6 on the device");
    return v;
}

#define PRP(N, DOC) conf.def_readwrite(#N, &Conf::N, DOC)

PYBIND11_MODULE(_uncalled, m) {
    m.doc() = "UNCALLED's C++ core (`_uncalled`) with the map path on the GPU (libunc_b200.so)";

    py::class_<Conf> conf(m, "Conf");
    conf.def(py::init<>()).def(py::init<const std::string &>());
    PRP(threads, "Number of threads (fast5 decoding threads here; the GPU mapper has no CPU mapping threads)");
    PRP(bwa_prefix, "BWA prefix to map to");
    PRP(idx_preset, "Mapping mode preset line of the .uncl file");
    PRP(model_path, "k-mer model file (empty: built-in r9.4 5-mer template model)");
    PRP(dbg_prefix, "unused");
    PRP(max_events, "Will give up on a read after this many events have been processed");
    PRP(seed_len, "Seed length in events");
    PRP(max_paths, "Maximum number of paths to consider per event");
    PRP(chunk_time, "Length of chunks in seconds");
    PRP(sample_rate, "Raw samples per second");
    PRP(bp_per_sec, "Expected bases sequenced per second");
    PRP(num_channels, "Number of channels used in sequencing");
    PRP(max_chunks, "Will give up on a read after this many chunks have been processed");
    PRP(fast5_list, "File containing a list of paths to fast5 files, one per line");
    PRP(read_list, "Only map reads listed in this file");
    PRP(max_reads, "Maximum number of reads to map");
    PRP(max_buffer, "Maximum number of reads to store in memory");
    PRP(host, "MinKNOW host address");
    PRP(port, "MinKNOW port");
    PRP(duration, "Duration to map real-time run in hours");
    PRP(max_active_reads, "Maximum number of reads being mapped at once");
    PRP(active_chs, "RealtimePool.FULL, EVEN or ODD");
    PRP(realtime_mode, "RealtimePool.DEPLETE or RealtimePool.ENRICH");
    PRP(min_active_reads, "unused");
    PRP(ctl_seqsum, "simulator input"); PRP(unc_seqsum, "simulator input"); PRP(unc_paf, "simulator input");
    PRP(sim_speed, "simulator speed"); PRP(scan_time, "simulator"); PRP(scan_intv_time, "simulator"); PRP(ej_time, "simulator");
    PRP(min_ch_reads, "simulator");
    PRP(device, "CUDA device of this process (one process per GPU)");
    PRP(batch_reads, "Reads per GPU batch");
    PRP(exact_ties, "1: the reference's unstable child sort reproduced (exact-ties kernel, slower)");
    PRP(ordered, "1: reads mapped in input order by ONE long-lived Mapper, i.e. `-t 1` exactly");

    py::class_<Paf> paf(m, "Paf");
    paf.def(py::init<>())
        .def(py::init<const std::string &, u16, u64>())
        .def("print_paf", &Paf::print_paf)
        .def("line", &Paf::line)
        .def("is_mapped", &Paf::is_mapped)
        .def("is_ended", &Paf::is_ended)
        .def("set_int", &Paf::set_int)
        .def("set_float", &Paf::set_float)
        .def("set_str", &Paf::set_str)
        .def_readonly("rd_name", &Paf::rd_name).def_readonly("rf_name", &Paf::rf_name)
        .def_readonly("rd_st", &Paf::rd_st).def_readonly("rd_en", &Paf::rd_en).def_readonly("rd_len", &Paf::rd_len)
        .def_readonly("rf_st", &Paf::rf_st).def_readonly("rf_en", &Paf::rf_en).def_readonly("rf_len", &Paf::rf_len)
        .def_readonly("fwd", &Paf::fwd).def_readonly("matches", &Paf::matches);
    py::enum_<Paf::Tag>(paf, "Tag")
        .value("MAP_TIME", Paf::MAP_TIME).value("WAIT_TIME", Paf::WAIT_TIME).value("QUEUE_TIME", Paf::QUEUE_TIME)
        .value("RECEIVE_TIME", Paf::RECEIVE_TIME).value("CHANNEL", Paf::CHANNEL).value("EJECT", Paf::EJECT)
        .value("READ_START", Paf::READ_START).value("IN_SCAN", Paf::IN_SCAN).value("TOP_RATIO", Paf::TOP_RATIO)
        .value("MEAN_RATIO", Paf::MEAN_RATIO).value("ENDED", Paf::ENDED).value("KEEP", Paf::KEEP).value("DELAY", Paf::DELAY)
        .value("SEED_CLUSTER", Paf::SEED_CLUSTER).value("CONFIDENT_EVENT", Paf::CONFIDENT_EVENT)
        .export_values();

    py::class_<MapPool>(m, "MapPool")
        .def(py::init<Conf &>())
        .def("add_fast5", &MapPool::add_fast5)
        .def("update", &MapPool::update)
        .def("running", &MapPool::running)
        .def("stop", &MapPool::stop);

    py::class_<Chunk>(m, "Chunk")
        .def(py::init<>())
        .def(py::init<const std::string &, u16, u32, u64, const std::vector<float> &, u32, u32>())
        .def(py::init([](const std::string &id, u16 ch, u32 num, u64 st, const std::string &dtype, py::bytes raw) {
            return Chunk(id, ch, num, st, dtype, (std::string) raw);
        }))
        .def("size", &Chunk::size)
        .def("empty", &Chunk::empty);

    py::class_<RealtimePool> rp(m, "RealtimePool");
    rp.def(py::init<Conf &>())
        .def("add_chunk", &RealtimePool::add_chunk)
        .def("try_add_chunk", &RealtimePool::try_add_chunk)
        .def("update", &RealtimePool::update)
        .def("all_finished", &RealtimePool::all_finished)
        .def("stop_all", &RealtimePool::stop_all);
    py::enum_<RealtimePool::Mode>(rp, "Mode").value("DEPLETE", RealtimePool::DEPLETE).value("ENRICH", RealtimePool::ENRICH).export_values();
    py::enum_<RealtimePool::ActiveChs>(rp, "ActiveChs").value("FULL", RealtimePool::FULL).value("EVEN", RealtimePool::EVEN).value("ODD", RealtimePool::ODD).export_values();

    py::class_<ClientSim>(m, "ClientSim").def(py::init<Conf &>());
    py::class_<Range>(m, "Range")
        .def(py::init<>()).def(py::init<u64, u64>()).def(py::init<const Range &>())
        .def_readwrite("start", &Range::start_).def_readwrite("end", &Range::end_)
        .def("length", &Range::length).def("is_valid", &Range::is_valid).def("intersect", &Range::intersect)
        .def("merge", &Range::merge).def("split_range", &Range::split_range).def("same_range", &Range::same_range)
        .def("intersects", &Range::intersects).def("get_recp_overlap", &Range::get_recp_overlap)
        .def("__lt__", &Range::operator<).def("__eq__", &Range::operator==)
        .def("__repr__", [](const Range &r) { return "Range(" + std::to_string(r.start_) + ", " + std::to_string(r.end_) + ")"; });
    // the method list of BwaIndex<KLEN>::pybind_defs (reference src/bwa_index.hpp:339-365)
    py::class_<BwaIndex>(m, "BwaIndex")
        .def(py::init<>())
        .def(py::init<const std::string &, bool>())
        .def_static("create", &BwaIndex::create)
        .def("load_index", &BwaIndex::load_index)
        .def("is_loaded", &BwaIndex::is_loaded)
        .def("load_pacseq", &BwaIndex::load_pacseq)
        .def("destroy", &BwaIndex::destroy)
        .def("get_neighbor", &BwaIndex::get_neighbor)
        .def("get_kmer_range", &BwaIndex::get_kmer_range)
        .def("get_kmer_count", &BwaIndex::get_kmer_count)
        .def("get_base_range", &BwaIndex::get_base_range)
        .def("sa", &BwaIndex::sa)
        .def("size", &BwaIndex::size)
        .def("translate_loc", &BwaIndex::translate_loc)
        .def("get_seqs", &BwaIndex::get_seqs)
        .def("coord_to_pacseq", &BwaIndex::coord_to_pacseq)
        .def("pacseq_loaded", &BwaIndex::pacseq_loaded)
        .def("get_base", &BwaIndex::get_base)
        .def("get_rid", &BwaIndex::get_rid)
        .def("get_sa_loc", &BwaIndex::get_sa_loc)
        .def("get_ref_coord", &BwaIndex::get_ref_coord)
        .def("get_ref_name", &BwaIndex::get_ref_name)
        .def("get_ref_len", &BwaIndex::get_ref_len)
        .def("range_to_fms", &BwaIndex::range_to_fms)
        .def("get_kmers", &BwaIndex::get_kmers)
        .def("get_kmers", &BwaIndex::get_kmers_named);
    m.def("kmer_count", &kmer_count);
    m.def("str_to_kmer", &str_to_kmer, py::arg("kmer"), py::arg("offset") = 0);
    m.def("kmer_comp", &kmer_comp);
    m.def("kmer_revcomp", &kmer_revcomp);
    m.def("kmer_head", &kmer_head);
    m.def("kmer_base", &kmer_base);
    m.def("kmer_to_str", &kmer_to_str);
    m.def("kmer_neighbor", &kmer_neighbor);
    m.def("self_align", &self_align);

    py::class_<DTWr94<0>>(m, "DTWr94p").def(py::init<const std::vector<float> &, const std::vector<uint16_t> &, const DTWParams &>())
        .def("get_path", &DTWr94<0>::get_path).def("score", &DTWr94<0>::score).def("mean_score", &DTWr94<0>::mean_score);
    py::class_<DTWr94<1>>(m, "DTWr94d").def(py::init<const std::vector<float> &, const std::vector<uint16_t> &, const DTWParams &>())
        .def("get_path", &DTWr94<1>::get_path).def("score", &DTWr94<1>::score).def("mean_score", &DTWr94<1>::mean_score);
    py::class_<DTWParams>(m, "DTWParams").def_readwrite("dw", &DTWParams::dw).def_readwrite("hw", &DTWParams::hw).def_readwrite("vw", &DTWParams::vw);
    m.attr("DTW_EVENT_GLOB") = py::cast(DTW_EVENT_GLOB);
    m.attr("DTW_RAW_GLOB") = py::cast(DTW_RAW_GLOB);
    m.attr("DTW_EVENT_QSUB") = py::cast(DTW_EVENT_QSUB);
    m.attr("DTW_EVENT_RSUB") = py::cast(DTW_EVENT_RSUB);
    m.attr("DTW_RAW_QSUB") = py::cast(DTW_EVENT_QSUB);        // as bound by the reference (src/pybinder.cpp:90-91): the EVENT presets
    m.attr("DTW_RAW_RSUB") = py::cast(DTW_EVENT_RSUB);
    py::class_<Event>(m, "Event")
        .def(py::init<>())
        .def_readwrite("mean", &Event::mean).def_readwrite("stdv", &Event::stdv)
        .def_readwrite("start", &Event::start).def_readwrite("length", &Event::length);
    py::class_<EventDetector> evd(m, "EventDetector", "EventDetector on the GPU: get_events / get_means over whole signals. "
                                  "add_sample is not offered (one GPU launch per sample).");
    py::class_<unc_event_params>(evd, "Params")
        .def(py::init([]() { unc_event_params p; unc_event_params_default(&p); return p; }))
        .def_property("window_length1", [](const unc_event_params &p) { return p.window_length1; },
                      [](unc_event_params &p, u32 v) { p.window_length1 = fixed_window(v, 3); })
        .def_property("window_length2", [](const unc_event_params &p) { return p.window_length2; },
                      [](unc_event_params &p, u32 v) { p.window_length2 = fixed_window(v, 6); })
        .def_readwrite("threshold1", &unc_event_params::threshold1).def_readwrite("threshold2", &unc_event_params::threshold2)
        .def_readwrite("peak_height", &unc_event_params::peak_height).def_readwrite("min_mean", &unc_event_params::min_mean)
        .def_readwrite("max_mean", &unc_event_params::max_mean);
    evd.def(py::init<>()).def(py::init<const unc_event_params &>())
        .def("get_events", &EventDetector::get_events)
        .def("get_means", &EventDetector::get_means)
        .def("mean_event_len", &EventDetector::mean_event_len);
    py::class_<EventProfiler>(m, "EventProfiler", "EventProfiler on the GPU: get_full_mask over a read's events. "
                              "add_event / anno_event are not offered (one GPU launch per event).")
        .def(py::init<>())
        .def("get_full_mask", &EventProfiler::get_full_mask);
    py::class_<PoreModel>(m, "PoreModel", "The r9.4 pore model on the GPU: match_prob of one mean, or of an array of "
                          "means against all 1024 k-mers")
        .def(py::init<bool>(), py::arg("complement") = true)
        .def("match_prob", &PoreModel::match_prob)
        .def("match_prob", &PoreModel::match_probs);
    m.attr("pmodel_r94_template") = py::cast(PoreModel(false));
    m.attr("pmodel_r94_complement") = py::cast(PoreModel(true));
}
