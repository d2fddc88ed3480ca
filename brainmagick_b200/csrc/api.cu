// Library state of libbm_b200.so: the last error, the launch counter and the debug switches (include/bm_b200.h).
#include "api.cuh"

namespace bm {
thread_local char g_last_error[512] = "";
unsigned long long g_launches = 0;
int g_debug_flags = 0;
long long* g_debug_buf = nullptr;
}

extern "C" const char* bm_last_error(void) { return bm::g_last_error; }
extern "C" int bm_abi_version(void) { return 1; }
extern "C" unsigned long long bm_launch_count(void) { return bm::g_launches; }
extern "C" int bm_set_debug_buffer(long long* buf) { bm::g_debug_buf = buf; return 0; }
extern "C" int bm_set_debug_flags(int flags) { int old = bm::g_debug_flags; bm::g_debug_flags = flags; return old; }
