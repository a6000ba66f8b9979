// Library-wide bits: status strings, last-error slot, device query.
#include <map>
#include <mutex>
#include <utility>

#include "b200yolo.h"
#include "common.cuh"

// ---- accumulators of the order-independent reductions (common.cuh: stream_acc) -----------------------------------
namespace {
struct StreamAcc {
    double* ptr = nullptr;
    long long n = 0;
};
std::mutex g_acc_mutex;
std::map<std::pair<int, cudaStream_t>, StreamAcc> g_acc;

__global__ void zero_doubles_kernel(double* p, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        p[i] = 0.0;
}
}  // namespace

double* stream_acc(cudaStream_t st, long long n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || n <= 0) return nullptr;
    std::lock_guard<std::mutex> lock(g_acc_mutex);
    StreamAcc& a = g_acc[std::make_pair(dev, st)];
    if (a.n >= n) return a.ptr;
    // a larger buffer replaces the old one, which stays allocated: CUDA graphs captured earlier may still use it.  The
    // allocation is not a stream operation, so it is allowed while the stream is being captured (relaxed mode); the
    // zero fill runs on the stream itself, ahead of the first use.
    const long long want = n < 16384 ? 16384 : n;
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, (size_t)want * sizeof(double));
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (e != cudaSuccess) {
        b2y_set_last_cuda_error((int)e);
        return nullptr;
    }
    long long grid = (want + 255) / 256;
    if (grid > 4096) grid = 4096;
    zero_doubles_kernel<<<(int)grid, 256, 0, st>>>(static_cast<double*>(p), want);
    if (cudaGetLastError() != cudaSuccess) return nullptr;
    a.ptr = static_cast<double*>(p);
    a.n = want;
    return a.ptr;
}

// ---- split-K partial tiles of the weight gradient (common.cuh: stream_ws) -------------------------------------------
namespace {
struct StreamWs {
    float* ptr = nullptr;
    long long n = 0;
};
std::mutex g_ws_mutex;
std::map<std::pair<int, cudaStream_t>, StreamWs> g_ws;
}  // namespace

float* stream_ws(cudaStream_t st, long long n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || n <= 0) return nullptr;
    std::lock_guard<std::mutex> lock(g_ws_mutex);
    StreamWs& w = g_ws[std::make_pair(dev, st)];
    if (w.n >= n) return w.ptr;
    // as in stream_acc: the replaced buffer stays allocated for graphs captured earlier, and the allocation is allowed
    // during a (relaxed) capture.  No fill: every slice is written in full before it is read.
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, (size_t)n * sizeof(float));
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (e != cudaSuccess) {
        b2y_set_last_cuda_error((int)e);
        return nullptr;
    }
    w.ptr = static_cast<float*>(p);
    w.n = n;
    return w.ptr;
}

static thread_local int g_last_cuda_error = 0;

extern "C" void b2y_set_last_cuda_error(int e) { g_last_cuda_error = e; }
extern "C" int b2y_last_cuda_error(void) { return g_last_cuda_error; }
extern "C" int b2y_abi_version(void) { return B2Y_ABI_VERSION; }

extern "C" const char* b2y_strerror(int status) {
    switch (status) {
        case B2Y_OK: return "ok";
        case B2Y_ERR_INVALID: return "invalid argument (shape/alignment/null pointer)";
        case B2Y_ERR_CUDA: return "CUDA runtime error (see b2y_last_cuda_error)";
        case B2Y_ERR_UNSUPPORTED: return "unsupported configuration for the sm_90a kernels";
        case B2Y_ERR_DRIVER: return "CUDA driver entry point unavailable or tensor-map encode failed";
        default: return "unknown status";
    }
}

extern "C" int b2y_device_sm_count(void) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
    return n;
}
