// wf_host.cu — the parts of the shared host layer (wf_host.hpp) that cannot live in the header: fill_kernel, and the
// functions around CUDA calls that all three engines make the same way.
#include "wf_host.hpp"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <map>

namespace wf {

static __global__ void fill_kernel(float *p, long long n, float v)
{
    for(long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        p[i] = v;
}

HostCore::~HostCore()
{
    if(ev0)
        cudaEventDestroy(ev0);
    if(ev1)
        cudaEventDestroy(ev1);
    for(void *p : kept)
        cudaFree(p);
    for(void *p : kept_host)
        cudaFreeHost(p);
    if(stream)
        cudaStreamDestroy(stream);
}

int fail(HostCore *c, int code, const char *fmt, ...)
{
    if(c)
    {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof(buf), fmt, ap);
        va_end(ap);
        c->last_error = buf;
    }
    return code;
}

int open_device(HostCore *c, int requested)
{
    int ndev = 0;
    if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    {
        cudaGetLastError();
        return fail(c, WF_ERR_NO_DEVICE, "no CUDA device (this engine has no CPU fallback)");
    }
    int dev = requested;
    if(dev < 0 && cudaGetDevice(&dev) != cudaSuccess)
        return fail(c, WF_ERR_CUDA, "cudaGetDevice failed");
    if(dev >= ndev)
        return fail(c, WF_ERR_INVALID_ARG, "device %d out of range (%d devices)", dev, ndev);
    c->device = dev;
    WF_CHECK(c, cudaSetDevice(dev));
    cudaDeviceProp prop{};
    WF_CHECK(c, cudaGetDeviceProperties(&prop, dev));
    if(prop.major != 9 || prop.minor != 0) // sm_90a code runs on compute capability 9.0 only
        return fail(c, WF_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major,
                    prop.minor);
    c->sm_count = prop.multiProcessorCount;
    WF_CHECK(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    WF_CHECK(c, cudaEventCreate(&c->ev0));
    WF_CHECK(c, cudaEventCreate(&c->ev1));
    return WF_OK;
}

int ptr_kind(const void *p)
{
    cudaPointerAttributes a{};
    if(cudaPointerGetAttributes(&a, p) != cudaSuccess)
    {
        cudaGetLastError();
        return 0;
    }
    if(a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)
        return 1;
    if(a.type == cudaMemoryTypeHost && a.devicePointer == p) // unified addressing: the same pointer is valid on the device
        return 2;
    return 0;
}

int fill_device(HostCore *c, float *p, long long n, float v, cudaStream_t st)
{
    if(n <= 0)
        return WF_OK;
    const int blocks = (int)std::min<long long>((n + 255) / 256, 1184);
    WF_CHECK(c, launch_kernel(fill_kernel, c->device, blocks, 256, 0, st, {}, p, n, v));
    c->launches++;
    return WF_OK;
}

cudaError_t opt_in_smem(const void *kernel, int device, size_t bytes)
{
    if(bytes <= 48 * 1024)
        return cudaSuccess;
    thread_local std::map<std::pair<const void *, int>, size_t> granted; // (kernel, device) -> bytes
    size_t &have = granted[{kernel, device}];
    if(bytes <= have)
        return cudaSuccess;
    const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if(err == cudaSuccess)
        have = bytes;
    return err;
}

cudaError_t launch_kernel(const void *kernel, int device, dim3 grid, unsigned block, size_t smem, cudaStream_t st,
                          LaunchMode mode, void **args)
{
    if(!kernel)
        return cudaErrorInvalidDeviceFunction;
    if(cudaError_t err = opt_in_smem(kernel, device, smem))
        return err;
    cudaLaunchAttribute attr[2] = {};
    unsigned n = 0;
    if(mode.pdl)
    {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n++].val.programmaticStreamSerializationAllowed = 1;
    }
    if(mode.cluster > 1)
    {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n++].val.clusterDim = {mode.cluster, 1, 1};
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelExC(&cfg, kernel, args);
}

int pcm_sample_bytes(HostCore *c, int32_t format, const void *pcm, size_t *bytes)
{
    if(format != WF_PCM_F32 && format != WF_PCM_S16)
        return fail(c, WF_ERR_INVALID_ARG, "pcm_format %d is not a wf_pcm_format", format);
    const bool s16 = format == WF_PCM_S16;
    if(s16 && ((uintptr_t)pcm & 1u) != 0)
        return fail(c, WF_ERR_INVALID_ARG, "int16 pcm must be 2-byte aligned");
    *bytes = s16 ? sizeof(int16_t) : sizeof(float);
    return WF_OK;
}

float last_kernel_ms(HostCore *c)
{
    if(!c || !c->ev_valid || cudaEventSynchronize(c->ev1) != cudaSuccess)
        return -1.0f;
    float ms = -1.0f;
    if(cudaEventElapsedTime(&ms, c->ev0, c->ev1) != cudaSuccess)
        return -1.0f;
    return ms;
}

cudaError_t begin_call(HostCore *c, cudaStream_t st)
{
    cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
    const cudaError_t err = cudaStreamIsCapturing(st, &status);
    c->capturing = err == cudaSuccess && status == cudaStreamCaptureStatusActive;
    c->captured = c->captured || c->capturing;
    return err;
}

cudaError_t time_begin(HostCore *c, cudaStream_t st)
{
    c->ev_valid = false;
    return c->capturing ? cudaSuccess : cudaEventRecord(c->ev0, st);
}

cudaError_t time_end(HostCore *c, cudaStream_t st)
{
    if(c->capturing)
        return cudaSuccess;
    const cudaError_t err = cudaEventRecord(c->ev1, st);
    c->ev_valid = err == cudaSuccess;
    return err;
}

cudaError_t device_alloc(HostCore *c, void **p, size_t bytes)
{
    return outside_capture(c, [&] { return cudaMalloc(p, bytes); });
}

int keep_upload(HostCore *c, const void *src, size_t bytes, cudaStream_t st, void **dev)
{
    void *h = nullptr, *d = nullptr;
    WF_CHECK(c, outside_capture(c, [&] { return cudaHostAlloc(&h, bytes, cudaHostAllocDefault); }));
    c->kept_host.push_back(h);
    WF_CHECK(c, device_alloc(c, &d, bytes));
    c->kept.push_back(d);
    memcpy(h, src, bytes);
    WF_CHECK(c, cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st));
    *dev = d;
    return WF_OK;
}

int refuse_pageable(HostCore *c, std::initializer_list<const void *> ptrs)
{
    if(!c->capturing)
        return WF_OK;
    for(const void *p : ptrs)
        if(p && ptr_kind(p) == 0)
            return fail(c, WF_ERR_INVALID_ARG, "a call captured into a CUDA graph needs device or page-locked host buffers "
                                               "(wf_host_alloc); a pageable host buffer cannot be replayed");
    return WF_OK;
}

} // namespace wf
