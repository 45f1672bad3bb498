// serde.cuh -- the chunked host <-> device pipeline shared by the params-file codec (serde.cu) and the proving-key file codec
// (pk_serde.cu).
#pragma once
#include "common.cuh"

namespace zkb {

constexpr uint32_t SERDE_THREADS = 256;

inline bool is_device_ptr(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// The chunked pipeline of a host-side buffer: two slots, each with its own stream, pinned staging and device staging.
struct SerdePipe {
    zkb_ctx *ctx;
    DevPool pool;
    cudaStream_t s[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    uint8_t *h_in[2] = {nullptr, nullptr}, *h_out[2] = {nullptr, nullptr};
    uint8_t *d_in[2] = {nullptr, nullptr}, *d_out[2] = {nullptr, nullptr};
    explicit SerdePipe(zkb_ctx *c) : ctx(c) { pool.ctx = c; }
    ~SerdePipe() {
        for (int j = 0; j < 2; ++j) {
            if (s[j]) { cudaStreamSynchronize(s[j]); cudaStreamDestroy(s[j]); }
            if (done[j]) cudaEventDestroy(done[j]);
            if (h_in[j]) cudaFreeHost(h_in[j]);
            if (h_out[j]) cudaFreeHost(h_out[j]);
        }
    }
};

}  // namespace zkb
