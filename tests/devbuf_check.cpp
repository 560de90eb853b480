// Checks of mm_devbuf (mashmap_b200/csrc/mm_devbuf.h), driven by test_devbuf.py.
//   devbuf_check nodevice   a failed reserve returns the runtime's error and leaves the array empty (exit 77: a device
//                           is present, so nothing fails)
//   devbuf_check gpu        the same for a request no device can satisfy, plus: the pending error is cleared, the array
//                           is usable again, and reserve_keep keeps its prefix
#include <cstdio>
#include <cstring>
#include <utility>
#include <vector>

#include "mm_devbuf.h"

#define CHECK(x)                                                                 \
  do {                                                                           \
    if (!(x)) {                                                                  \
      std::fprintf(stderr, "%s:%d: check failed: %s\n", __FILE__, __LINE__, #x); \
      return 1;                                                                  \
    }                                                                            \
  } while (0)

template <typename T>
static bool empty(const mm_devbuf<T> &b)
{
  return !b && b.get() == nullptr && b.capacity() == 0;
}

static int no_device()
{
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) == cudaSuccess && n_dev > 0) return 77;
  void *p = nullptr;
  const cudaError_t direct = cudaMalloc(&p, 8);
  std::printf("cudaMalloc without a device: %s\n", cudaGetErrorName(direct));
  CHECK(direct != cudaSuccess);
  mm_devbuf<uint64_t> b;
  CHECK(b.reserve(1000) == direct);
  CHECK(empty(b));
  CHECK(b.reserve_keep(1000, 0, nullptr) == direct);
  CHECK(empty(b));
  return 0;
}

static int gpu()
{
  const uint64_t huge = 1ULL << 60; /* bytes */
  mm_devbuf<unsigned char> big;
  CHECK(big.reserve(huge) == cudaErrorMemoryAllocation);
  CHECK(empty(big));
  CHECK(cudaGetLastError() == cudaSuccess);

  /* an array that held memory is empty after a failed reserve, and usable again */
  mm_devbuf<uint32_t> b;
  CHECK(b.reserve(256) == cudaSuccess && b && b.capacity() == 256);
  CHECK(b.reserve(huge / 4) == cudaErrorMemoryAllocation);
  CHECK(empty(b));
  CHECK(cudaGetLastError() == cudaSuccess);
  CHECK(b.reserve(1000) == cudaSuccess && b && b.capacity() == 1000);
  uint32_t *const p = b.get();
  CHECK(b.reserve(10) == cudaSuccess && b.get() == p && b.capacity() == 1000);

  /* reserve_keep grows and keeps [0, used) */
  cudaStream_t st = nullptr;
  CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess);
  std::vector<uint32_t> h(1000), back(1000, 0);
  for (uint32_t i = 0; i < 1000; i++) h[i] = i * 2654435761u;
  CHECK(cudaMemcpy(b.get(), h.data(), 1000 * 4, cudaMemcpyHostToDevice) == cudaSuccess);
  CHECK(b.reserve_keep(1 << 20, 1000, st) == cudaSuccess && b.capacity() == (1u << 20));
  CHECK(cudaMemcpy(back.data(), b.get(), 1000 * 4, cudaMemcpyDeviceToHost) == cudaSuccess);
  CHECK(back == h);
  CHECK(b.reserve_keep(huge / 4, 1000, st) == cudaErrorMemoryAllocation);
  CHECK(empty(b));
  CHECK(cudaGetLastError() == cudaSuccess);
  CHECK(cudaStreamDestroy(st) == cudaSuccess);

  /* moves hand the array over */
  mm_devbuf<uint32_t> m;
  CHECK(m.reserve(10) == cudaSuccess);
  mm_devbuf<uint32_t> n(std::move(m));
  CHECK(empty(m) && n.capacity() == 10);
  m = std::move(n);
  CHECK(empty(n) && m.capacity() == 10);
  return 0;
}

int main(int argc, char **argv)
{
  if (argc == 2 && !std::strcmp(argv[1], "nodevice")) return no_device();
  if (argc == 2 && !std::strcmp(argv[1], "gpu")) {
    const int rc = gpu();
    if (rc == 0) std::printf("ok\n");
    return rc;
  }
  std::fprintf(stderr, "usage: %s nodevice|gpu\n", argv[0]);
  return 2;
}
