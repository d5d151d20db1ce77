// Library-level entry points of the C ABI: version, thread-local error text, launch counter.
#include <stdarg.h>

#include <map>
#include <mutex>

#include "../../include/pfd_b200.h"
#include "common.h"

namespace pfd {
thread_local std::string g_last_error;
std::atomic<int64_t> g_launches{0};

int set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return 1;
}
}  // namespace pfd

namespace pfd {
static std::mutex g_opt_mu;
static std::map<std::string, int>& opt_table() {
  static std::map<std::string, int> t;
  return t;
}
int option(const char* name, int dflt) {
  std::lock_guard<std::mutex> lk(g_opt_mu);
  auto it = opt_table().find(name);
  return it == opt_table().end() ? dflt : it->second;
}

// PFD_DETERMINISTIC=1 in the environment when the library is loaded makes deterministic mode the default, so that
// unmodified programs can run in either mode; pfd_set_option("deterministic", v) overrides it, a reset restores it.
static const int g_det_default = [] {
  const char* e = getenv("PFD_DETERMINISTIC");
  return (e && e[0] == '1') ? 1 : 0;
}();
bool deterministic() { return option("deterministic", g_det_default) != 0; }
}  // namespace pfd

extern "C" PFD_API int pfd_set_option(const char* name, int32_t value) {
  std::lock_guard<std::mutex> lk(pfd::g_opt_mu);
  if (!name) {
    pfd::opt_table().clear();          // NULL: back to the built-in defaults
    return 0;
  }
  pfd::opt_table()[name] = value;
  return 0;
}

extern "C" PFD_API int pfd_version(void) { return PFD_ABI_VERSION; }
extern "C" PFD_API const char* pfd_last_error(void) { return pfd::g_last_error.c_str(); }
extern "C" PFD_API int64_t pfd_launch_count(void) { return pfd::g_launches.load(); }
