// Device memory of one engine (AR engine, codec decoder, codec stream, codec encoder, speaker encoder): its named
// tensors and its scratch.  Every block is allocated through the store and freed when the store is destroyed.
// Host-only.
#pragma once
#include "common.cuh"

#include <map>
#include <string>
#include <vector>

enum DevDtype { DT_BF16 = 2, DT_F32 = 4 };  // value = element size

class DevStore {
 public:
  explicit DevStore(const char* engine) : engine_(engine) {}
  ~DevStore() {
    for (void* p : blocks_) cudaFree(p);
  }
  DevStore(const DevStore&) = delete;
  DevStore& operator=(const DevStore&) = delete;

  // a new block of `bytes`, zero-filled if `zero`.  cudaMemset returns before the block is zero and is not ordered
  // against non-blocking streams, so the device is drained before the block is handed out.
  int alloc(void** p, size_t bytes, bool zero = false) {
    cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();  // the failure stays ours: a later error check (ours or the framework's) must not report it
      return q3_set_err("%s: cudaMalloc(%zu B) failed: %s", engine_, bytes, cudaGetErrorString(e));
    }
    blocks_.push_back(*p);
    if (zero && ((e = cudaMemset(*p, 0, bytes)) != cudaSuccess || (e = cudaDeviceSynchronize()) != cudaSuccess))
      return q3_set_err("%s: cudaMemset(%zu B) failed: %s", engine_, bytes, cudaGetErrorString(e));
    return 0;
  }
  // a new block of `count` elements of T
  template <class T>
  int alloc(T** p, size_t count, bool zero) {
    void* q = nullptr;
    if (alloc(&q, count * sizeof(T), zero)) return 1;
    *p = static_cast<T*>(q);
    return 0;
  }

  // replace the block *p (null, or a block of this store) by a new one of `bytes`, zero-filled if `zero`.  Work queued
  // on `stream` may still read the old block, so the stream is drained before it is freed.
  template <class T>
  int grow(T** p, size_t bytes, cudaStream_t stream, bool zero = false) {
    if (*p) {
      Q3_CUDA(cudaStreamSynchronize(stream));
      if (release(*p)) return 1;
      *p = nullptr;
    }
    void* q = nullptr;
    if (alloc(&q, bytes, zero)) return 1;
    *p = static_cast<T*>(q);
    return 0;
  }

  // free the block p of this store before the store ends.  The caller has drained every stream that may still use it.
  int release(void* p) {
    for (size_t i = 0; i < blocks_.size(); ++i)
      if (blocks_[i] == p) {
        blocks_.erase(blocks_.begin() + i);
        Q3_CUDA(cudaFree(p));
        return 0;
      }
    return q3_set_err("%s: block %p is not one of this store's", engine_, p);
  }

  // copy the device tensor `dev` (shape[ndim], elements of `dtype`) in as `name`.  `dev` may still be being produced on
  // the caller's stream (no stream crosses the load ABIs), so the device is drained before the copy; the copy is
  // complete when load returns, so the caller may free `dev` then.
  int load(const std::string& name, const void* dev, const int64_t* shape, int ndim, DevDtype dtype) {
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) n *= shape[i];
    const size_t bytes = (size_t)n * dtype;
    void* p = nullptr;
    if (alloc(&p, (bytes + 255) & ~(size_t)255)) return 1;
    Q3_CUDA(cudaDeviceSynchronize());
    Q3_CUDA(cudaMemcpy(p, dev, bytes, cudaMemcpyDeviceToDevice));
    Q3_CUDA(cudaDeviceSynchronize());
    tensors_[name] = Tensor{p, n, dtype};
    return 0;
  }

  // free the tensor `name` (load) before the store ends, so the name may be loaded again.  The caller has drained every
  // stream that may still read it.
  int drop(const std::string& name) {
    const auto it = tensors_.find(name);
    if (it == tensors_.end()) return q3_set_err("%s: tensor %s is missing", engine_, name.c_str());
    void* p = it->second.p;
    tensors_.erase(it);
    return release(p);
  }

  // the tensor `name` of `numel` elements of T (float or bf16); null, with the error recorded, when it is missing or
  // has another element count or type
  template <class T>
  const T* need(const std::string& name, int64_t numel) const {
    static_assert(sizeof(T) == DT_BF16 || sizeof(T) == DT_F32, "tensors are bf16 or fp32");
    const auto it = tensors_.find(name);
    if (it != tensors_.end() && it->second.numel == numel && it->second.dtype == (int)sizeof(T))
      return static_cast<const T*>(it->second.p);
    const std::string have = it == tensors_.end() ? std::string("is missing")
                                                  : "has " + std::to_string(it->second.numel) + " " + dtype_name(it->second.dtype) + " elements";
    q3_set_err("%s: tensor %s %s, expected %lld %s elements", engine_, name.c_str(), have.c_str(), (long long)numel,
               dtype_name((int)sizeof(T)));
    return nullptr;
  }

 private:
  struct Tensor {
    void* p;
    int64_t numel;
    int dtype;
  };
  static const char* dtype_name(int dtype) { return dtype == DT_BF16 ? "bf16" : "fp32"; }

  const char* engine_;
  std::map<std::string, Tensor> tensors_;
  std::vector<void*> blocks_;
};
