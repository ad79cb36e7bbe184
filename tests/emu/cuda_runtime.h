/*
 * cuda_runtime.h -- TEST INFRASTRUCTURE: the handful of CUDA runtime entry
 * points hyperscan_b200/csrc/device/*.cu use, restated over host memory with
 * synchronous semantics, so that the library compiles as plain C++ for the SIMT
 * emulator (tests/emu/simt_emu.h).  "Device" pointers are host pointers; streams
 * and events are tokens; there is one "device" with HSB_EMU_SMS (default 2) SMs.
 */
#ifndef HSB_EMU_CUDA_RUNTIME_H
#define HSB_EMU_CUDA_RUNTIME_H

#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "simt_emu.h"

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
typedef struct hsb_emu_stream *cudaStream_t;
typedef struct hsb_emu_event *cudaEvent_t;
struct cudaIpcMemHandle_t { char reserved[64]; };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEventBlockingSync = 1,
       cudaIpcMemLazyEnablePeerAccess = 1 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount, cudaDevAttrMaxSharedMemoryPerBlockOptin,
                      cudaDevAttrComputeCapabilityMajor, cudaDevAttrComputeCapabilityMinor };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize };

static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int d) { return d == 0 ? cudaSuccess : cudaErrorInvalidValue; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr a, int) {
    switch (a) {
    case cudaDevAttrMultiProcessorCount: {
        const char *s = getenv("HSB_EMU_SMS");
        *v = s && atoi(s) > 0 ? atoi(s) : 2;
        break;
    }
    case cudaDevAttrMaxSharedMemoryPerBlockOptin: *v = 232448; break;
    case cudaDevAttrComputeCapabilityMajor: *v = 9; break;
    case cudaDevAttrComputeCapabilityMinor: *v = 0; break;
    }
    return cudaSuccess;
}
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

static inline cudaError_t cudaMalloc(void **p, size_t n) {
    return posix_memalign(p, 256, n ? n : 1) ? cudaErrorMemoryAllocation : cudaSuccess;
}
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc((void **)p, n); }
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void **p, size_t n) { return cudaMalloc(p, n); }
template <class T> static inline cudaError_t cudaMallocHost(T **p, size_t n) { return cudaMalloc((void **)p, n); }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) {
    memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = 0) {
    memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dpitch, const void *s, size_t spitch, size_t width,
                                            size_t height, cudaMemcpyKind, cudaStream_t = 0) {
    for (size_t r = 0; r < height; r++) {
        memmove((char *)d + r * dpitch, (const char *)s + r * spitch, width);
    }
    return cudaSuccess;
}
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = 0) {
    memset(d, v, n);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) {
    *s = (cudaStream_t)malloc(1);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = (cudaEvent_t)malloc(1); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
/* "peer" buffers live in this process: the handle carries the pointer */
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) {
    memset(h, 0, sizeof(*h));
    memcpy(h->reserved, &p, sizeof(p));
    return cudaSuccess;
}
static inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) {
    memcpy(p, h.reserved, sizeof(*p));
    return cudaSuccess;
}
static inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }

#endif
