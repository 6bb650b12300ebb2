// wf_host.hpp — the host layer the three C-ABI engines share: spectrum (wf_engine.cu), level meter / RMS feed
// (wf_meter.cu) and waveform (wf_wave.cu).  Device, stream, timing events and error reporting (HostCore), grow-only device
// buffers, pointer classification, struct-size compatibility, environment knobs and the staging of host buffers.  What
// cannot live in a header (fill_kernel and the functions around CUDA calls) is in wf_host.cu.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "wfstft.h"

namespace wf {

// What every engine owns besides its tables and kernels; the engine structs derive from it.  The destructor releases the
// stream, the events and the buffers kept for captured graphs: the engines' *_destroy synchronise the stream before the
// handle goes, so nothing is freed while a kernel may still use it.
struct HostCore {
    int device = 0, sm_count = 0;
    cudaStream_t stream = nullptr;            // the engine's own stream (calls without a caller stream)
    cudaEvent_t ev0 = nullptr, ev1 = nullptr; // around the kernels of the last call (wf_*last_kernel_ms)
    bool ev_valid = false;
    int64_t launches = 0;
    std::string last_error;
    // CUDA graphs: `capturing` while a call is enqueued on a stream that is being captured (begin_call); `captured` once any
    // call was.  From then on no device buffer is freed before the engine goes, since a graph may still point at it: a
    // growing DevBuf leaves its old allocation in `kept`, and a captured call's own inputs (keep_upload) stay there too.
    bool capturing = false, captured = false;
    std::vector<void *> kept, kept_host;

    HostCore() = default;
    HostCore(const HostCore &) = delete;
    HostCore &operator=(const HostCore &) = delete;
    ~HostCore();
};

// Keeps the message for wf_*last_error (when there is an engine) and returns `code`.
int fail(HostCore *c, int code, const char *fmt, ...) __attribute__((format(printf, 3, 4)));

// WF_ERR_CAPACITY, with a message naming the range, unless slots [first, first + count) of `max_streams` exist (count >= 0).
// `what` names the call's kind of range ("stream", "state", "reset", "ring").
inline int check_slot_range(HostCore *c, int32_t first, int32_t count, int max_streams, const char *what)
{
    if(first < 0 || count < 0 || (int64_t)first + count > max_streams)
        return fail(c, WF_ERR_CAPACITY, "%s range [%d, %lld) exceeds max_streams %d", what, first, (long long)first + count,
                    max_streams);
    return WF_OK;
}

// Returns WF_ERR_OOM / WF_ERR_CUDA from the calling function, with the failing call and CUDA's reason as the message,
// unless `call` succeeds.
#define WF_CHECK(core, call)                                                                                       \
    do                                                                                                             \
    {                                                                                                              \
        const cudaError_t _err = (call);                                                                           \
        if(_err != cudaSuccess)                                                                                    \
            return ::wf::fail((core), (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s failed: %s", \
                              #call, cudaGetErrorString(_err));                                                    \
    } while(0)

// Allocates an engine, runs its create steps and hands it out.  When a step fails, the engine's message stays readable
// through the engine kind's wf_*last_error(NULL) (`create_error`) and `destroy` releases what was set up.
template<class E, class Init>
int create_engine(E **out, std::string &create_error, void (*destroy)(E *), Init &&init)
{
    E *e = new(std::nothrow) E();
    if(!e)
        return WF_ERR_OOM;
    const int rc = init(e);
    if(rc != WF_OK)
    {
        create_error = e->last_error;
        destroy(e);
        return rc;
    }
    *out = e;
    return WF_OK;
}

// Device `requested` (< 0: the current one) for a new engine: it must exist and be sm_90.  Makes it current, stores its SM
// count and creates the engine's stream and timing events.  WF_ERR_NO_DEVICE without a CUDA device or on another
// architecture, WF_ERR_INVALID_ARG for a device number out of range, WF_ERR_CUDA / WF_ERR_OOM when a CUDA call fails.
int open_device(HostCore *c, int requested);

// 0 = pageable host memory (or unknown), 1 = device / managed memory, 2 = page-locked host memory the device can address
// directly under the same pointer
int ptr_kind(const void *p);
inline bool is_device_ptr(const void *p) { return p && ptr_kind(p) == 1; }

// p[0, n) := v on `st` (fill_kernel); counts as one launch of the engine.
int fill_device(HostCore *c, float *p, long long n, float v, cudaStream_t st);

// Milliseconds between the events around the last call's kernels, -1 before the first call, after a captured call or when
// the events fail.
float last_kernel_ms(HostCore *c);

// Starts a call on `st`: sets c->capturing from cudaStreamIsCapturing (and c->captured with it).
cudaError_t begin_call(HostCore *c, cudaStream_t st);

// The timing events around a call's kernels (ev0 before, ev1 after).  A captured call records none: its replays are not
// timed, and last_kernel_ms stays < 0 until an eager call.
cudaError_t time_begin(HostCore *c, cudaStream_t st);
cudaError_t time_end(HostCore *c, cudaStream_t st);

// cudaMalloc, also while c's call is being captured: cudaMalloc is not stream-ordered, so it runs under the thread's
// relaxed capture mode and the capture (global mode included) stays valid.
cudaError_t device_alloc(HostCore *c, void **p, size_t bytes);

// Runs `f` (CUDA calls outside the captured work: allocation, a one-time initialisation on the engine's own stream) under
// the relaxed capture mode while c's call is being captured, else as it is.
template<class F>
cudaError_t outside_capture(HostCore *c, F &&f)
{
    if(!c->capturing)
        return f();
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    if(cudaError_t err = cudaThreadExchangeStreamCaptureMode(&mode))
        return err;
    const cudaError_t err = f();
    cudaThreadExchangeStreamCaptureMode(&mode);
    return err;
}

// `bytes` of `src` (host) into fresh device memory on `st`, through fresh page-locked host memory; *dev := the copy.  Both
// stay until the engine goes, so that a captured call's replays read the values it was captured with whatever later calls do.
int keep_upload(HostCore *c, const void *src, size_t bytes, cudaStream_t st, void **dev);

// WF_ERR_INVALID_ARG while c's call is being captured and one of `ptrs` (nulls aside) is pageable host memory, which a graph
// cannot copy: the call then enqueues nothing and the capture stays valid.
int refuse_pageable(HostCore *c, std::initializer_list<const void *> ptrs);

// A device buffer that only grows: reserve(n) keeps the allocation when it holds n elements already, else frees it and
// allocates exactly n (the contents are not kept).  Freed with its owner.  Once the owner has had a call captured, the old
// allocation goes to HostCore::kept instead of being freed (a graph may still use it).
template<class T>
struct DevBuf {
    T *p = nullptr;
    size_t cap = 0;

    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DevBuf &operator=(DevBuf &&o) noexcept
    {
        std::swap(p, o.p);
        std::swap(cap, o.cap);
        return *this;
    }
    ~DevBuf()
    {
        if(p)
            cudaFree(p);
    }
    operator T *() const { return p; }

    int reserve(HostCore *c, size_t n)
    {
        if(n <= cap)
            return WF_OK;
        if(p && c->captured)
            c->kept.push_back(p);
        else if(p)
            cudaFree(p);
        p = nullptr;
        cap = 0;
        WF_CHECK(c, device_alloc(c, (void **)&p, n * sizeof(T)));
        cap = n;
        return WF_OK;
    }
    // a table uploaded once at create time; an empty table leaves the buffer null
    int upload(HostCore *c, const std::vector<T> &v)
    {
        if(v.empty())
            return WF_OK;
        if(int rc = reserve(c, v.size()))
            return rc;
        WF_CHECK(c, cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
        return WF_OK;
    }
};

// A caller's struct of the current size, or of one of the earlier ABI sizes in `prev_sizes` (each ends before the fields
// added since, which then read as zero).  False for any other struct_size.  `out` carries the current struct_size either way;
// `is_current` tells whether the caller passed the current size.
template<class T>
bool accept_struct(const T *in, std::initializer_list<size_t> prev_sizes, T &out, bool *is_current = nullptr)
{
    const bool cur = in->struct_size == sizeof(T);
    size_t n = cur ? sizeof(T) : 0;
    for(const size_t prev : prev_sizes)
        if(!cur && in->struct_size == prev)
            n = prev;
    if(n == 0)
        return false;
    out = T{};
    memcpy(&out, in, n);
    out.struct_size = (uint32_t)sizeof(T);
    if(is_current)
        *is_current = cur;
    return true;
}

// The sample format of a call's PCM (wf_pcm_format; wf_batch, wf_meter_batch and wf_wave_batch carry the same field):
// `bytes` := bytes per sample.  WF_ERR_INVALID_ARG for a value that is not a wf_pcm_format, or for int16 PCM at an odd
// address.
int pcm_sample_bytes(HostCore *c, int32_t format, const void *pcm, size_t *bytes);

// A call's PCM as the kernels read it: `pcm` in the call's sample type (behind a `const float *`), strides in samples.
struct PcmView {
    const float *pcm;
    long long stream_stride, channel_stride;
};

// What check_pcm_batch finds of a level-meter or waveform batch's PCM.
struct PcmBatch {
    size_t sample_bytes = 0;
    bool s16 = false;
    size_t span = 0; // samples from pcm to the end of the last row: (S-1)*stream_stride + (cc-1)*channel_stride + T*hop
};

// The checks of a wf_meter_batch or wf_wave_batch `b` (at least one stream, `cc` capture channels) that both engines make
// alike, in this order: no negative stride, the sample format (pcm_sample_bytes), and n_ticks * hop within int range with
// `reserve` samples ahead of the call's own in every row the kernels index (the meter's window, the waveform's holdback).
template<class B>
int check_pcm_batch(HostCore *c, const B &b, int cc, int reserve, PcmBatch *out)
{
    if(b.stream_stride < 0 || b.channel_stride < 0)
        return fail(c, WF_ERR_INVALID_ARG, "negative strides are not supported");
    if(int rc = pcm_sample_bytes(c, b.pcm_format, b.pcm, &out->sample_bytes))
        return rc;
    out->s16 = b.pcm_format == WF_PCM_S16;
    if((long long)b.n_ticks * b.hop > 0x7fffffffLL - reserve)
        return fail(c, WF_ERR_INVALID_ARG, "n_ticks * hop too large for one call");
    out->span = (size_t)(b.n_streams - 1) * (size_t)b.stream_stride + (size_t)(cc - 1) * (size_t)b.channel_stride +
                (size_t)b.n_ticks * (size_t)b.hop;
    return WF_OK;
}

// Lets `kernel` use `bytes` of dynamic shared memory on `device` (the opt-in above the default 48 KB).  Asks CUDA once per
// kernel, device and size: a size at or below one already granted returns at once.
cudaError_t opt_in_smem(const void *kernel, int device, size_t bytes);

// How cudaLaunchKernelEx launches: with programmatic dependent launch (the kernel's prologue overlaps the tail of the
// previous launch on the stream) and / or as clusters of `cluster` consecutive CTAs.
struct LaunchMode {
    bool pdl = false;
    unsigned cluster = 1;
};

// Launches kernel(*args[0], *args[1], ...) as `grid` CTAs of `block` threads with `smem` bytes of dynamic shared memory on
// stream `st` of `device` (the current one), opted in to `smem` first.  A null kernel (no instantiation for the asked
// template arguments) is cudaErrorInvalidDeviceFunction.
cudaError_t launch_kernel(const void *kernel, int device, dim3 grid, unsigned block, size_t smem, cudaStream_t st,
                          LaunchMode mode, void **args);

// The same for a typed kernel and its arguments.
template<class... P, class... A>
cudaError_t launch_kernel(void (*kernel)(P...), int device, dim3 grid, unsigned block, size_t smem, cudaStream_t st,
                          LaunchMode mode, A &&...args)
{
    return [&](P... a) {
        void *argv[] = {&a...};
        return launch_kernel((const void *)kernel, device, grid, block, smem, st, mode, argv);
    }(std::forward<A>(args)...);
}

// One compiled instantiation of a spectrum kernel family, as the unit that compiles it hands it out: the kernel and the
// sizes of its launch shape that follow from its template arguments.  kernel == nullptr: none is compiled for them.
struct KernelRef {
    const void *kernel = nullptr;
    unsigned block = 0; // threads per CTA
    size_t smem = 0;    // dynamic shared memory per CTA
};

// Environment knobs (A/B switches for tests and tools).  A flag that is on by default is switched off by a value starting
// with '0'; one that is off by default is switched on by a value starting with '1'.
inline bool env_flag(const char *name, bool dflt)
{
    const char *v = getenv(name);
    return v ? (dflt ? v[0] != '0' : v[0] == '1') : dflt;
}
inline int env_int(const char *name, int dflt)
{
    const char *v = getenv(name);
    return v ? atoi(v) : dflt;
}

// Host buffers of one meter / waveform call, staged through the engine's grow-only device buffers on stream `st`.  With
// `host` false (the call passed device pointers) every buffer passes through as it is.  in() uploads an input at once and
// returns its device copy; out() returns device space for an output, and finish() copies the outputs back, after the
// launch, in the order they were declared.  Null buffers pass through.  After a failure later declarations do nothing and
// `rc` holds the status, which the caller checks before it launches.
class Staging {
  public:
    Staging(HostCore *c, cudaStream_t st, bool host) : core(c), st(st), host(host) {}
    int rc = WF_OK;

    template<class T>
    const T *in(DevBuf<T> &buf, const T *src, size_t n)
    {
        return in_bytes(buf, src, n * sizeof(T));
    }
    // an input of `bytes` bytes held in a buffer of T (int16 PCM behind a `const float *`): exactly those bytes are copied
    template<class T>
    const T *in_bytes(DevBuf<T> &buf, const T *src, size_t bytes)
    {
        if(!take(buf, src, (bytes + sizeof(T) - 1) / sizeof(T)))
            return src;
        rc = copy(buf.p, src, bytes, cudaMemcpyHostToDevice);
        return buf.p;
    }
    template<class T>
    T *out(DevBuf<T> &buf, T *dst, size_t n)
    {
        if(!take(buf, dst, n))
            return dst;
        back[n_back++] = {dst, buf.p, n * sizeof(T)};
        return buf.p;
    }
    int finish()
    {
        for(int i = 0; i < n_back; ++i)
            if(int r = copy(back[i].host, back[i].dev, back[i].bytes, cudaMemcpyDeviceToHost))
                return r;
        return WF_OK;
    }

  private:
    struct Back {
        void *host;
        const void *dev;
        size_t bytes;
    };
    HostCore *core;
    cudaStream_t st;
    bool host;
    Back back[8];
    int n_back = 0;

    template<class T>
    bool take(DevBuf<T> &buf, const void *p, size_t n)
    {
        if(rc || !host || !p)
            return false;
        rc = buf.reserve(core, n);
        return rc == WF_OK;
    }
    int copy(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind)
    {
        WF_CHECK(core, cudaMemcpyAsync(dst, src, bytes, kind, st));
        return WF_OK;
    }
};

// The host buffers of a state call (wf_meter_get_state, wf_wave_set_state, ...) as the sections of one staging buffer, so
// that the call makes one copy and one launch.  add() places a section 16-byte aligned (null or empty: skipped); after
// reserve(), dev() gives a section's device pointer (null when skipped).  run() does the call on `st`: a set call packs
// the sections, copies them to the device and launches; a get call launches, copies them back and unpacks them.  The
// stream is synchronised before it returns.  Whether the launch counts as one of the engine's is the caller's choice.
class StateSections {
  public:
    int add(const void *host, size_t bytes)
    {
        if(!host || !bytes)
            return -1;
        sec[n] = {const_cast<void *>(host), total, bytes};
        total = (total + bytes + 15) & ~(size_t)15;
        return n++;
    }
    int reserve(HostCore *c, DevBuf<unsigned char> &d, std::vector<unsigned char> &h)
    {
        if(int rc = d.reserve(c, total))
            return rc;
        if(h.size() < total)
            h.resize(total);
        dbase = d.p;
        hbase = h.data();
        return WF_OK;
    }
    template<class T>
    T *dev(int i) const
    {
        return (i < 0) ? nullptr : reinterpret_cast<T *>(dbase + sec[i].off);
    }
    bool empty() const { return n == 0; }
    // `launch` enqueues the kernel on `st` and returns the launch's error
    template<class Launch>
    int run(HostCore *c, cudaStream_t st, bool set, Launch &&launch)
    {
        if(set)
        {
            for(int i = 0; i < n; ++i)
                memcpy(hbase + sec[i].off, sec[i].host, sec[i].bytes);
            WF_CHECK(c, cudaMemcpyAsync(dbase, hbase, total, cudaMemcpyHostToDevice, st));
        }
        WF_CHECK(c, launch());
        if(!set)
            WF_CHECK(c, cudaMemcpyAsync(hbase, dbase, total, cudaMemcpyDeviceToHost, st));
        WF_CHECK(c, cudaStreamSynchronize(st));
        if(!set)
            for(int i = 0; i < n; ++i)
                memcpy(sec[i].host, hbase + sec[i].off, sec[i].bytes);
        return WF_OK;
    }

  private:
    struct Sec {
        void *host;
        size_t off, bytes;
    };
    Sec sec[4]{};
    int n = 0;
    size_t total = 0;
    unsigned char *dbase = nullptr, *hbase = nullptr;
};

} // namespace wf
