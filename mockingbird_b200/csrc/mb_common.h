// Shared host-side helpers for libmockingbird_b200 (error reporting, launch counting, the weight table, workspaces).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/mockingbird_b200.h"

namespace mb {

// thread-local error string behind mb_last_error()
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);
// every kernel launch of the library goes through this counter (mb_launch_count())
void count_launch(int n = 1);

#define MB_CUDA_CHECK(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return ::mb::fail(MB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                        __FILE__, __LINE__);                                                 \
  } while (0)

#define MB_LAUNCH_CHECK(what)                                                              \
  do {                                                                                     \
    cudaError_t _e = cudaGetLastError();                                                   \
    if (_e != cudaSuccess)                                                                 \
      return ::mb::fail(MB_ERR_CUDA, "launch of %s failed: %s (%s:%d)", what,              \
                        cudaGetErrorString(_e), __FILE__, __LINE__);                       \
    ::mb::count_launch();                                                                  \
  } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// The weight-upload protocol of every model handle (set_arena, set_weight per tensor, finalize): null, size and
// alignment check of an arena.  `fn` names the entry point in the error message.
int check_arena(const char* fn, const void* h, const void* arena, size_t bytes, size_t need, size_t align);

// The regions of a compute call's workspace, handed out in declaration order, each rounded up to `align` bytes.  total()
// adds `align` bytes of slack so that any workspace pointer can be aligned up in place.  A `*_workspace_bytes` query and
// its compute call build the same layout.
struct WsLayout {
  size_t align = 256, bytes = 0;
  // n elements of T; the offset comes back in elements of T
  template <class T = char>
  size_t take(size_t n) {
    const size_t at = bytes;
    bytes += align_up(n * sizeof(T), align);
    return at / sizeof(T);
  }
  size_t total() const { return bytes + align; }
};

// `ws` aligned up to `align` bytes
template <class T = char>
T* aligned(void* ws, size_t align = 256) {
  return (T*)(((uintptr_t)ws + align - 1) & ~(uintptr_t)(align - 1));
}

// The workspace of compute entry point `fn`: MB_ERR_INVALID if it is null, MB_ERR_WORKSPACE if it has fewer than `need`
// bytes, otherwise *base (if given) is the workspace aligned up to `align` bytes.  Call it before any CUDA call of the entry
// point.
template <class T = char>
int bind(const char* fn, void* ws, size_t bytes, size_t need, T** base = nullptr, size_t align = 256) {
  if (!ws) return fail(MB_ERR_INVALID, "%s: null workspace", fn);
  if (bytes < need) return fail(MB_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", fn, bytes, need);
  if (base) *base = aligned<T>(ws, align);
  return MB_OK;
}

// The tensors at the start of a model's arena, laid out in declaration order at align_up(n, 64) floats each.  A
// checkpoint tensor has an exact shape, is settable and is required by finalize; a derived region of n floats is
// written by the model itself and is neither settable nor required.
class WeightTable {
 public:
  void add(const std::string& name, std::vector<int64_t> dims);
  void add_derived(const std::string& name, size_t n);
  // names set() accepts and drops: in the checkpoint, never read by inference
  std::function<bool(const std::string&)> ignored = [](const std::string&) { return false; };

  size_t floats() const { return total_; }
  bool has(const std::string& name) const { return index_.count(name) != 0; }
  size_t size(const std::string& name) const;  // floats of `name`, 0 if undeclared
  float* ptr(const std::string& name) const;   // nullptr if undeclared

  // Arguments, name and exact shape first (MB_ERR_INVALID), then an attached arena (MB_ERR_STATE), then the copy.
  int set(const char* fn, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream);
  // a new arena holds none of the tensors set before
  void attach(float* arena);
  // MB_ERR_STATE naming the first checkpoint tensor that was never set
  int check_all_set(const char* fn) const;

 private:
  struct Entry {
    std::string name;
    std::vector<int64_t> dims;  // empty for a derived region
    size_t off, n;
    bool derived, set;
  };
  void append(const std::string& name, std::vector<int64_t> dims, size_t n, bool derived);
  std::vector<Entry> entries_;
  std::map<std::string, size_t> index_;
  size_t total_ = 0;
  float* arena_ = nullptr;
};

}  // namespace mb
