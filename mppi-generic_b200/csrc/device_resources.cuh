/*
 * device_resources.cuh — owners of the CUDA resources an engine holds (engine_internal.cuh: mppib_engine). Each one releases
 * what it holds in its destructor, so a resource is one member declaration and no failure path can leak it or free it twice.
 * They live in place inside the engine and are neither copied nor moved; each reads as the raw handle it owns (empty: null).
 * They return their library's status, so CUDA_TRY(buf.reserve(n, stream)) reads like any other runtime call.
 */
#pragma once
#include <cuda_runtime.h>
#include <cufft.h>
#include <curand.h>

#include <cstddef>
#include <utility>

namespace mppib
{
struct NoCopy
{
  NoCopy() = default;
  NoCopy(const NoCopy&) = delete;
  NoCopy& operator=(const NoCopy&) = delete;
};

// Device memory: pointer + capacity in elements.
template <class T>
class DeviceBuffer : NoCopy
{
public:
  ~DeviceBuffer()
  {
    reset();
  }
  T* get() const
  {
    return p_;
  }
  operator T*() const
  {
    return p_;
  }
  size_t capacity() const
  {
    return n_;
  }
  void reset()
  {
    cudaFree(p_);
    p_ = nullptr;
    n_ = 0;
  }
  // exactly n elements, whatever it held; empty on failure
  cudaError_t alloc(size_t n)
  {
    reset();
    const cudaError_t rc = cudaMalloc(&p_, n * sizeof(T));
    if (rc == cudaSuccess)
      n_ = n;
    else
      p_ = nullptr;
    return rc;
  }
  // Room for n elements; the contents are not kept. Grows only after `s` has drained, because a kernel enqueued on it may
  // still be reading the old allocation. A call that does not grow touches nothing.
  cudaError_t reserve(size_t n, cudaStream_t s)
  {
    if (n <= n_)
      return cudaSuccess;
    const cudaError_t rc = cudaStreamSynchronize(s);
    return rc != cudaSuccess ? rc : alloc(n);
  }

private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

// Pinned host memory (cudaHostAlloc): pointer + capacity in elements.
template <class T>
class PinnedBuffer : NoCopy
{
public:
  ~PinnedBuffer()
  {
    if (p_)
      cudaFreeHost((void*)p_);
  }
  operator T*() const
  {
    return p_;
  }
  // n elements with the cudaHostAlloc* flags given, allocated once; for cudaHostAllocMapped memory, *device_alias = the
  // address kernels use
  cudaError_t alloc(size_t n, unsigned flags, T** device_alias = nullptr)
  {
    cudaError_t rc = cudaHostAlloc((void**)&p_, n * sizeof(T), flags);
    if (rc == cudaSuccess)
      n_ = n;
    if (rc == cudaSuccess && device_alias)
      rc = cudaHostGetDevicePointer((void**)device_alias, (void*)p_, 0);
    return rc;
  }
  // Room for n elements; the contents are not kept. No copy may still be in flight to or from it. Empty on failure.
  cudaError_t reserve(size_t n, unsigned flags)
  {
    if (n <= n_)
      return cudaSuccess;
    if (p_)
      cudaFreeHost((void*)p_);
    p_ = nullptr;
    n_ = 0;
    const cudaError_t rc = alloc(n, flags);
    if (rc != cudaSuccess)
      p_ = nullptr;
    return rc;
  }

private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

class Event : NoCopy
{
public:
  ~Event()
  {
    if (ev_)
      cudaEventDestroy(ev_);
  }
  operator cudaEvent_t() const
  {
    return ev_;
  }
  cudaError_t create(unsigned flags = cudaEventDefault)
  {
    return cudaEventCreateWithFlags(&ev_, flags);
  }

private:
  cudaEvent_t ev_ = nullptr;
};

// A stream the engine created, or one the caller supplied (mppib_desc.stream), which is used and never destroyed.
class Stream : NoCopy
{
public:
  ~Stream()
  {
    if (owned_)
      cudaStreamDestroy(s_);
  }
  operator cudaStream_t() const
  {
    return s_;
  }
  cudaError_t create(unsigned flags, int priority)
  {
    const cudaError_t rc = cudaStreamCreateWithPriority(&s_, flags, priority);
    owned_ = rc == cudaSuccess;
    return rc;
  }
  void borrow(cudaStream_t s)
  {
    s_ = s;
  }

private:
  cudaStream_t s_ = nullptr;
  bool owned_ = false;
};

// A 2-D CUDA array and the texture object that reads it. Reads as the cudaTextureObject_t (0 until one is set).
class ArrayTexture : NoCopy
{
public:
  ~ArrayTexture()
  {
    if (tex_)
      cudaDestroyTextureObject(tex_);
    if (array_)
      cudaFreeArray(array_);
  }
  operator cudaTextureObject_t() const
  {
    return tex_;
  }
  // A width x height array of `ch` texels filled from the tightly packed rows at `host` (copied on `s`, which is drained),
  // read as `tex` describes. The pair it held is released only once the new one exists; on failure it is kept.
  cudaError_t replace(const cudaChannelFormatDesc& ch, size_t width, size_t height, const void* host, size_t row_bytes,
                      const cudaTextureDesc& tex, cudaStream_t s)
  {
    ArrayTexture fresh;
    cudaError_t rc = cudaMallocArray(&fresh.array_, &ch, width, height);
    if (rc == cudaSuccess)
      rc = cudaMemcpy2DToArrayAsync(fresh.array_, 0, 0, host, row_bytes, row_bytes, height, cudaMemcpyHostToDevice, s);
    if (rc == cudaSuccess)
      rc = cudaStreamSynchronize(s);
    cudaResourceDesc res{};
    res.resType = cudaResourceTypeArray;
    res.res.array.array = fresh.array_;
    if (rc == cudaSuccess)
      rc = cudaCreateTextureObject(&fresh.tex_, &res, &tex, nullptr);
    if (rc != cudaSuccess)
      return rc;
    std::swap(array_, fresh.array_);  // `fresh` leaves with the old pair and releases it
    std::swap(tex_, fresh.tex_);
    return cudaSuccess;
  }

private:
  cudaArray_t array_ = nullptr;
  cudaTextureObject_t tex_ = 0;
};

// A cuRAND generator or cuFFT plan, made by a call such as cufftPlan1d(&h, ...) and destroyed only if that call
// succeeded (a cufftHandle has no null value)
template <class H, class R, R (*Destroy)(H), R kOk>
class LibraryHandle : NoCopy
{
public:
  ~LibraryHandle()
  {
    if (made_)
      Destroy(h_);
  }
  operator H() const { return h_; }
  template <class... P, class... A>
  R make(R (*create)(H*, P...), A... a)
  {
    const R r = create(&h_, a...);
    made_ = r == kOk;
    return r;
  }

private:
  H h_{};
  bool made_ = false;
};
using CurandGenerator = LibraryHandle<curandGenerator_t, curandStatus_t, curandDestroyGenerator, CURAND_STATUS_SUCCESS>;
using CufftPlan = LibraryHandle<cufftHandle, cufftResult, cufftDestroy, CUFFT_SUCCESS>;
}  // namespace mppib
