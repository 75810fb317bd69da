// api.cu -- error reporting, device cache and parameter-layout queries of libgcbf_b200.so.
#include <atomic>
#include <mutex>
#include <stdarg.h>

#include "common.cuh"

namespace gcbf {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};
static std::once_flag g_dev_once;
static int g_sm_count = 132;   // H100 SXM; replaced by the device query on first use

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int32_t check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return (int32_t)e;
}

void count_launch(int64_t n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
    std::call_once(g_dev_once, [] {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            g_sm_count = n;
    });
    return g_sm_count;
}

}  // namespace gcbf

extern "C" __attribute__((visibility("default"))) const char* gcbf_last_error_string(void) { return gcbf::g_err; }
extern "C" __attribute__((visibility("default"))) int32_t gcbf_version(void) { return 101; }
extern "C" __attribute__((visibility("default"))) int64_t gcbf_launch_count(void) { return gcbf::g_launches.load(); }

extern "C" __attribute__((visibility("default"))) int32_t gcbf_param_count_l(int32_t edge_dim, int32_t out_dim,
                                                                             int32_t n_layers) {
    if (edge_dim < 1 || edge_dim > 6 || out_dim < 1 || out_dim > 4 || n_layers < 1 || n_layers > gcbf::GCBF_MAX_LAYERS)
        return -1;
    return gcbf::make_deep_layout(edge_dim, out_dim, n_layers).total;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_param_offsets_l(int32_t edge_dim, int32_t out_dim,
                                                                               int32_t n_layers, int32_t* off) {
    if (edge_dim < 1 || edge_dim > 6 || out_dim < 1 || out_dim > 4 || n_layers < 1 ||
        n_layers > gcbf::GCBF_MAX_LAYERS || !off) {
        gcbf::set_error("gcbf_param_offsets_l: bad argument");
        return -1;
    }
    const gcbf::DeepLayout D = gcbf::make_deep_layout(edge_dim, out_dim, n_layers);
    int k = 0;
    for (int l = 0; l < n_layers; ++l)
        for (int i = 0; i < gcbf::L_HEAD0; ++i) {
            off[k++] = D.layer[l].w[i];
            off[k++] = D.layer[l].b[i];
        }
    for (int i = gcbf::L_HEAD0; i <= gcbf::L_OUT; ++i) {
        off[k++] = D.layer[0].w[i];
        off[k++] = D.layer[0].b[i];
    }
    return 0;
}
