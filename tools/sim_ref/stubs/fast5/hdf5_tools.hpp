// Stand-in for the hdf5_tools::File interface that the reference's Fast5Reader and ReadBuffer compile against, so that
// its ClientSim can be built without HDF5.  The scenario driver never opens a file: reads are handed to the client as
// ReadBuffer(Chunk&) objects.  Test tooling only.
#pragma once
// (the standard headers below are the ones the reference's sources get through the real hdf5_tools.hpp)
#include <algorithm>
#include <array>
#include <cassert>
#include <climits>
#include <cstring>
#include <deque>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

namespace hdf5_tools {
class File {
  public:
    void open(const std::string &) {}
    void close() {}
    bool is_open() const { return false; }
    std::vector<std::string> list_group(const std::string &) const { return {}; }
    std::map<std::string, std::string> get_attr_map(const std::string &) const { return {}; }
    template <class T> void read(const std::string &, std::vector<T> &) const {}
};
}
