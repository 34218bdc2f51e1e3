// Force-included (g++ -include) ahead of the reference's ClientSim sources: after <chrono> is in, every later use of
// std::chrono::high_resolution_clock names this clock, whose time the scenario driver sets.  So the reference's Timer,
// and with it ClientSim::get_time, reads the driver's clock.  Test tooling only.
#pragma once
#include <chrono>
#include <cstdint>

extern int64_t g_fake_now_ns;

namespace std {
namespace chrono {
struct sim_fake_clock {
    typedef nanoseconds duration;
    typedef duration::rep rep;
    typedef duration::period period;
    typedef time_point<sim_fake_clock> time_point;
    static constexpr bool is_steady = true;
    static time_point now() { return time_point(duration(g_fake_now_ns)); }
};
}
}

#define high_resolution_clock sim_fake_clock
