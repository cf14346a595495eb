// Library-wide bookkeeping: number of kernel launches issued through the C ABI (bench.py's `gpu_launches`).
#include <atomic>

std::atomic<long long> g_hb_launches{0};

extern "C" {
long long hb_launch_count(void) { return g_hb_launches.load(); }
void hb_launch_count_reset(void) { g_hb_launches.store(0); }
const char* hb_version(void) { return "holocron_b200 0.1.0 (sm_90a)"; }
}
