// Owners of the libcfrb200 objects (include/cfrb200.h) the `rela` module creates.  Each one is released by its owner on every way
// out of the scope that holds it, a throwing constructor included.  Where one object refers to another (a match or an agent reads
// its handles when it is destroyed), the referring owner is declared after the one it refers to, so that it is released first.
#pragma once
#include <memory>
#include <stdexcept>
#include <string>

#include "../../../include/cfrb200.h"

namespace rela {

// rc when the call succeeded (rc >= 0), else an exception with the library's message.
inline int check(int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + cfrb_last_error());
  return rc;
}

template <auto Destroy>
struct Destroyer {
  template <class T>
  void operator()(T* p) const { Destroy(p); }
};
using HandlePtr = std::unique_ptr<cfrb_handle, Destroyer<cfrb_destroy>>;
using MatchPtr = std::unique_ptr<cfrb_match, Destroyer<cfrb_match_destroy>>;
using AgentPtr = std::unique_ptr<cfrb_agent, Destroyer<cfrb_agent_destroy>>;
using RowsPtr = std::unique_ptr<cfrb_rows, Destroyer<cfrb_rows_destroy>>;
using CommPtr = std::unique_ptr<cfrb_comm, Destroyer<cfrb_comm_destroy>>;
using FullGamePtr = std::unique_ptr<cfrb_full_game, Destroyer<cfrb_full_game_destroy>>;
using BlueprintPtr = std::unique_ptr<cfrb_blueprint, Destroyer<cfrb_blueprint_destroy>>;

// fp32 device memory of cfrb_dev_alloc, which cfrb_dev_free releases on the device it came from.
struct DevFree {
  int device = 0;
  void operator()(float* p) const { cfrb_dev_free(device, p); }
};
using DevFloats = std::unique_ptr<float, DevFree>;

inline DevFloats dev_alloc(int device, size_t count) {
  void* p = nullptr;
  check(cfrb_dev_alloc(device, count * sizeof(float), &p), "cfrb_dev_alloc");
  return DevFloats(static_cast<float*>(p), DevFree{device});
}

inline HandlePtr open_handle(const cfrb_config& c) {
  cfrb_handle* h = nullptr;
  check(cfrb_create(&c, &h), "cfrb_create");
  return HandlePtr(h);
}

}  // namespace rela
