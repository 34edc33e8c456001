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

}  // namespace mb

extern "C" {

const char* mb_last_error(void) { return mb::g_err; }

const char* mb_version(void) { return "mockingbird_b200 0.1 sm_90a"; }

uint64_t mb_launch_count(void) { return mb::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
