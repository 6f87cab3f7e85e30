#include "common.cuh"
#include <mutex>
namespace ms {
static std::mutex g_mu;
static std::string g_err;
void set_error(const std::string& s) { std::lock_guard<std::mutex> l(g_mu); g_err = s; }
const char* last_error_cstr() { std::lock_guard<std::mutex> l(g_mu); return g_err.c_str(); }
static bool g_pdl_suppressed = false;
void pdl_set_suppressed(bool s) { g_pdl_suppressed = s; }
bool pdl_enabled() { return !g_pdl_suppressed; }
static long long g_launches = 0;
long long launch_count() { return g_launches; }
void add_launches(long long n) { g_launches += n; }
int check_launch(const char* what, int n_kernels) {
    g_launches += n_kernels;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error(std::string(what) + ": " + cudaGetErrorString(e)); return -1; }
    return 0;
}
}  // namespace ms
