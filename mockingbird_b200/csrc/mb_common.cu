#include "mb_common.h"

#include <atomic>
#include <cstring>

namespace mb {

static thread_local char g_err[1024] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int check_arena(const char* fn, const void* h, const void* arena, size_t bytes, size_t need, size_t align) {
  if (!h || !arena) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  if (bytes < need) return fail(MB_ERR_WORKSPACE, "%s: need %zu bytes, got %zu", fn, need, bytes);
  if ((uintptr_t)arena % align) return fail(MB_ERR_INVALID, "%s: arena must be %zu-byte aligned", fn, align);
  return MB_OK;
}

void WeightTable::append(const std::string& name, std::vector<int64_t> dims, size_t n, bool derived) {
  index_[name] = entries_.size();
  entries_.push_back({name, std::move(dims), total_, n, derived, false});
  total_ += align_up(n, 64);
}

void WeightTable::add(const std::string& name, std::vector<int64_t> dims) {
  size_t n = 1;
  for (int64_t d : dims) n *= (size_t)d;
  append(name, std::move(dims), n, false);
}

void WeightTable::add_derived(const std::string& name, size_t n) { append(name, {}, n, true); }

size_t WeightTable::size(const std::string& name) const {
  auto it = index_.find(name);
  return it == index_.end() ? 0 : entries_[it->second].n;
}

float* WeightTable::ptr(const std::string& name) const {
  auto it = index_.find(name);
  return it == index_.end() ? nullptr : arena_ + entries_[it->second].off;
}

static std::string shape_str(const int64_t* dims, int32_t ndim) {
  std::string s = "[";
  for (int i = 0; i < ndim; ++i) s += (i ? "," : "") + std::to_string(dims[i]);
  return s + "]";
}

int WeightTable::set(const char* fn, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream) {
  if (!name || !w || ndim < 0 || (!dims && ndim > 0)) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  const bool drop = ignored(name);
  auto it = index_.find(name);
  if (!drop && (it == index_.end() || entries_[it->second].derived))
    return fail(MB_ERR_INVALID, "%s: unknown tensor '%s'", fn, name);
  if (!drop) {
    const Entry& e = entries_[it->second];
    bool ok = (int)e.dims.size() == ndim;
    for (int i = 0; ok && i < ndim; ++i) ok = e.dims[i] == dims[i];
    if (!ok)
      return fail(MB_ERR_INVALID, "%s: %s has shape %s, expected %s", fn, name, shape_str(dims, ndim).c_str(),
                  shape_str(e.dims.data(), (int32_t)e.dims.size()).c_str());
  }
  if (!arena_) return fail(MB_ERR_STATE, "%s: set the arena first", fn);
  if (drop) return MB_OK;
  Entry& e = entries_[it->second];
  MB_CUDA_CHECK(cudaMemcpyAsync(arena_ + e.off, w, e.n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  e.set = true;
  return MB_OK;
}

void WeightTable::attach(float* arena) {
  arena_ = arena;
  for (Entry& e : entries_) e.set = false;
}

int WeightTable::check_all_set(const char* fn) const {
  for (const Entry& e : entries_)
    if (!e.derived && !e.set) return fail(MB_ERR_STATE, "%s: tensor %s was never set", fn, e.name.c_str());
  return MB_OK;
}

}  // namespace mb

extern "C" {

const char* mb_last_error(void) { return mb::g_err; }

const char* mb_version(void) { return "mockingbird_b200 0.1 sm_90a"; }

uint64_t mb_launch_count(void) { return mb::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
