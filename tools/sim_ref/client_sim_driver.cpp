// Runs a scripted scenario through the reference's own ClientSim (src/client_sim.cpp, compiled where it lies) with its
// clock under the script's control, and prints every get_read_chunks result and unblock_read return value.
// tools/make_sim_golden.py builds it and stores the output as tests/golden/sim/client_golden.json, which the
// restatement in uncalled_b200/sim.py must reproduce.  Test tooling only.
//
// Script lines (stdin):
//   conf <num_channels> <sample_rate> <chunk_time> <max_chunks> <scan_time> <ej_time>   (first line)
//   intv <ch> <i> <st> <en> | gap <ch> <i> <len> | delay <ch> <i> <len> | read <ch> <id> <offs>
//   load <id> <number> <n_samples>   a read whose calibrated samples are 0, 1, ..., n-1
//   run
//   tick <ms>                        set the clock, then get_read_chunks
//   stop <ch> <number> | unblock <ch> <number>
// Output lines:
//   chunk <ms> <ch> <number> <id> <start> <len> <first sample>
//   running <ms> <0|1>
//   unblock <ch> <number> <delay>
#include <cmath>
#include <cstdint>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#define private public
#include "client_sim.hpp"
#undef private

int64_t g_fake_now_ns = 0;

int main() {
    std::string line, op;
    Conf conf;
    ClientSim *client = nullptr;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        if (!(in >> op)) continue;
        if (op == "conf") {
            u32 n_channels, max_chunks;
            float sample_rate, chunk_time, scan_time, ej_time;
            in >> n_channels >> sample_rate >> chunk_time >> max_chunks >> scan_time >> ej_time;
            conf.set_num_channels(n_channels);
            conf.set_sample_rate(sample_rate);
            conf.set_chunk_time(chunk_time);
            conf.set_max_chunks(max_chunks);
            conf.sim_prms.scan_time = scan_time;
            conf.sim_prms.ej_time = ej_time;
            client = new ClientSim(conf);
        } else if (op == "intv") {
            u32 ch, i, st, en;
            in >> ch >> i >> st >> en;
            client->add_intv(ch, i, st, en);
        } else if (op == "gap" || op == "delay") {
            u32 ch, i, len;
            in >> ch >> i >> len;
            if (op == "gap") client->add_gap(ch, i, len);
            else client->add_delay(ch, i, len);
        } else if (op == "read") {
            u32 ch, offs;
            std::string id;
            in >> ch >> id >> offs;
            client->add_read(ch, id, offs);
        } else if (op == "load") {
            // what ClientSim::load_fast5s does with one ReadBuffer, the signal truncated to max_chunks chunks as the
            // fast5 constructor of ReadBuffer truncates it
            std::string id;
            u32 number, n;
            in >> id >> number >> n;
            const u32 L = ReadBuffer::PRMS.chunk_len();
            if ((n + L - 1) / L > ReadBuffer::PRMS.max_chunks) n = ReadBuffer::PRMS.max_chunks * L;
            std::vector<float> sig(n);
            for (u32 k = 0; k < n; k++) sig[k] = (float) k;
            ClientSim::ReadLoc r = client->read_locs[id];
            Chunk c(id, r.ch, number, 0, sig, 0, n);
            ReadBuffer read(c);
            read.full_signal_.swap(read.chunk_);
            read.set_channel(r.ch);
            client->channels_[r.ch - 1].load_read(r.i, r.offs, read);
        } else if (op == "run") {
            g_fake_now_ns = 0;
            client->run();
        } else if (op == "tick") {
            int64_t ms;
            in >> ms;
            g_fake_now_ns = ms * 1000000;
            for (auto &p : client->get_read_chunks()) {
                Chunk &c = p.second;
                std::cout << "chunk " << ms << " " << p.first << " " << c.get_number() << " " << c.get_id() << " "
                          << c.get_start() << " " << c.size() << " " << (c.size() ? (int64_t) c[0] : -1) << "\n";
            }
            std::cout << "running " << ms << " " << (client->is_running() ? 1 : 0) << "\n";
        } else if (op == "stop") {
            u32 ch, number;
            in >> ch >> number;
            client->stop_receiving_read(ch, number);
        } else if (op == "unblock") {
            u32 ch, number;
            in >> ch >> number;
            std::cout << "unblock " << ch << " " << number << " " << client->unblock_read(ch, number) << "\n";
        }
    }
    return 0;
}
