// runtime.cu -- error string, launch counter, device queries for libpointrcnn_b200.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"

namespace prb {
static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

int num_sms() {
    static std::atomic<int> cache[64];   // per device ordinal; 0 = not queried yet
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;  // H100 SXM
    int sms = cache[dev].load(std::memory_order_relaxed);
    if (sms == 0) {
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 148;
        cache[dev].store(sms, std::memory_order_relaxed);
    }
    return sms;
}

static int env_int(const char *name, int dflt) {
    const char *v = getenv(name);
    return v ? atoi(v) : dflt;
}
// process defaults: built-in values, overridden ONCE (first use) by PRB_* environment variables for experiment scripts
static prb_options make_defaults() {
    prb_options o;
    o.mlp_occ = env_int("PRB_MLP_OCC", 0);
    o.mlp_sms = env_int("PRB_MLP_SMS", 0);
    o.mlp_resident = env_int("PRB_MLP_RESIDENT", 1);
    o.nn_sort_queries = env_int("PRB_NN_SORT_QUERIES", 0);
    return o;
}
static const prb_options &defaults() {
    static const prb_options d = make_defaults();
    return d;
}
static thread_local prb_options t_opts;
static thread_local bool t_opts_set = false;
const prb_options &opts() { return t_opts_set ? t_opts : defaults(); }
}  // namespace prb

extern "C" void prb_options_init(prb_options *o) { if (o) *o = prb::defaults(); }
extern "C" int prb_set_thread_options(const prb_options *o) {
    if (o) { prb::t_opts = *o; prb::t_opts_set = true; } else prb::t_opts_set = false;
    return 0;
}
extern "C" void prb_get_thread_options(prb_options *o) { if (o) *o = prb::opts(); }

extern "C" int prb_abi_version(void) { return PRB_ABI_VERSION; }
extern "C" const char *prb_last_error(void) { return prb::g_err; }
extern "C" unsigned long long prb_launch_count(void) { return prb::g_launches.load(); }
