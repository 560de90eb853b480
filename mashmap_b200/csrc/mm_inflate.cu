/*
 * mm_inflate.cu -- BGZF block inflation on the device: the kernel around mm_inflate.h and the mm_inflater handle of
 * include/mashmap_b200.h.
 *
 * One warp inflates one block (DESIGN §8): the decoder's tables sit in the warp's slice of shared memory, every lane
 * runs the Huffman decode on the same bits (uniform control flow, broadcast loads), lane 0 writes literals, and the
 * lanes split the match copies, the table fills and the CRC-32. Warps take blocks in a grid-stride loop, so thousands
 * of blocks are in flight at once. The host walks the caller's arrays in slices that fit the handle's device buffers.
 */
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "../../include/mashmap_b200.h"
#include "mm_devbuf.h"
#include "mm_inflate.h"

namespace {

constexpr int kWarps = 8; /* warps per CTA: 8 decoders' tables = 26 KB of shared memory; 4 CTAs per SM fit 56 registers */
constexpr uint64_t kSliceBytes = 256ULL << 20;    /* inflated bytes per slice (a larger single block gets its own) */

thread_local std::string g_create_error;

__global__ void __launch_bounds__(kWarps * 32, 4) k_inflate(const uint8_t *__restrict__ comp, const uint64_t *__restrict__ coff,
                                                        const uint64_t *__restrict__ ooff, const uint32_t *__restrict__ crc,
                                                        uint64_t n, uint8_t *out, int32_t *__restrict__ status)
{
  __shared__ mmi_tables tb[kWarps];
  __shared__ uint32_t crc_tab[256];
  mmi_crc_table(crc_tab, (int)threadIdx.x, (int)blockDim.x);
  __syncthreads();
  const int lane = (int)(threadIdx.x & 31), w = (int)(threadIdx.x >> 5);
  for (uint64_t i = (uint64_t)blockIdx.x * kWarps + (uint64_t)w; i < n; i += (uint64_t)gridDim.x * kWarps) {
    const uint64_t ob = ooff[i], on = ooff[i + 1] - ob;
    int rc = mmi_inflate(comp + coff[i], coff[i + 1] - coff[i], out + ob, on, tb[w], lane, 32);
    if (rc == MMI_OK) {
      uint32_t s = mmi_crc_share(crc_tab, out + ob, on, lane, 32);
      for (int d = 16; d; d >>= 1) s ^= __shfl_xor_sync(0xFFFFFFFFu, s, d);
      if (mmi_crc_finish(s, on) != crc[i]) rc = MMI_E_CRC;
    }
    if (lane == 0) status[i] = rc;
    __syncwarp();
  }
}

const char *status_text(int rc)
{
  switch (rc) {
    case MMI_E_INPUT: return "the stream runs past its compressed bytes";
    case MMI_E_OUTPUT: return "the stream inflates to more bytes than its output range (ISIZE)";
    case MMI_E_SHORT: return "the stream inflates to fewer bytes than its output range (ISIZE)";
    case MMI_E_BTYPE: return "invalid block type";
    case MMI_E_STORED: return "stored block length does not match its complement";
    case MMI_E_CODES: return "invalid code lengths";
    case MMI_E_SYMBOL: return "invalid code or symbol";
    case MMI_E_DIST: return "distance too far back";
    case MMI_E_TRAILING: return "the stream ends before its compressed bytes do";
    case MMI_E_CRC: return "CRC-32 mismatch";
    default: return "unknown error";
  }
}

}  // namespace

const char *mmi_status_text(int rc) { return status_text(rc); }

cudaError_t mmi_launch_inflate(const uint8_t *comp, const uint64_t *coff, const uint64_t *ooff, const uint32_t *crc, uint64_t n,
                               uint8_t *out, int32_t *status, cudaStream_t st)
{
  if (n == 0) return cudaSuccess;
  int dev = 0, per_sm = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_inflate, kWarps * 32, 0);
  if (e != cudaSuccess) return e;
  const unsigned grid = (unsigned)std::min<uint64_t>((uint64_t)std::max(per_sm, 1) * (uint64_t)sms, (n + kWarps - 1) / kWarps);
  k_inflate<<<grid, kWarps * 32, 0, st>>>(comp, coff, ooff, crc, n, out, status);
  return cudaGetLastError();
}

struct mm_inflater {
  int device = -1;
  int grid = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[3] = {nullptr, nullptr, nullptr}; /* call start, kernels start, kernels end (of the last slice) */
  float ms[2] = {0, 0};                           /* mm_inflater_last_ms */
  std::string error;
  mm_devbuf<uint8_t> d_comp, d_out;
  mm_devbuf<uint64_t> d_coff, d_ooff;
  mm_devbuf<uint32_t> d_crc;
  mm_devbuf<int32_t> d_status;
  std::vector<uint64_t> h_coff, h_ooff;
  std::vector<int32_t> h_status;
  ~mm_inflater()
  {
    if (device >= 0) cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

static int inf_fail(mm_inflater *inf, int rc, const char *fmt, ...)
{
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  (inf ? inf->error : g_create_error) = buf;
  return rc;
}

extern "C" {

int mm_inflater_create(int device, mm_inflater **out)
{
  if (!out) return inf_fail(nullptr, MM_EINVAL, "null argument");
  *out = nullptr;
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return inf_fail(nullptr, MM_ENODEVICE, "no CUDA device: %s (this library has no CPU path)", cudaGetErrorString(e));
  if (device < 0 || device >= n_dev) return inf_fail(nullptr, MM_ENODEVICE, "device %d out of range (%d devices)", device, n_dev);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return inf_fail(nullptr, MM_ENODEVICE, "cannot query device");
  if (prop.major != 9 || prop.minor != 0)
    return inf_fail(nullptr, MM_ENODEVICE, "device %d is sm_%d%d; this build is sm_90a only", device, prop.major, prop.minor);
  std::unique_ptr<mm_inflater> inf(new mm_inflater());
  inf->device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&inf->stream, cudaStreamNonBlocking) != cudaSuccess)
    return inf_fail(nullptr, MM_ECUDA, "cannot create stream");
  for (cudaEvent_t &ev : inf->ev)
    if (cudaEventCreate(&ev) != cudaSuccess) return inf_fail(nullptr, MM_ECUDA, "cannot create the timing events");
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_inflate, kWarps * 32, 0) != cudaSuccess || per_sm < 1)
    return inf_fail(nullptr, MM_ECUDA, "cannot size the inflate grid");
  inf->grid = per_sm * prop.multiProcessorCount;
  *out = inf.release();
  return MM_OK;
}

int mm_inflater_destroy(mm_inflater *inf)
{
  delete inf;
  return MM_OK;
}

const char *mm_inflater_error(const mm_inflater *inf) { return inf ? inf->error.c_str() : g_create_error.c_str(); }

int mm_inflater_last_ms(const mm_inflater *inf, float ms[2])
{
  if (!inf || !ms) return MM_EINVAL;
  ms[0] = inf->ms[0];
  ms[1] = inf->ms[1];
  return MM_OK;
}

int mm_inflate_blocks(mm_inflater *inf, const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off,
                      const uint32_t *crc, uint64_t n_blocks, uint8_t *out, int64_t *bad_block)
{
  if (!inf) return inf_fail(nullptr, MM_EINVAL, "null handle");
  if (bad_block) *bad_block = -1;
  inf->ms[0] = inf->ms[1] = 0;
  if (n_blocks == 0) return MM_OK;
  if (!comp_off || !out_off || !crc || (!comp && comp_off[n_blocks] > comp_off[0]) || (!out && out_off[n_blocks] > out_off[0]))
    return inf_fail(inf, MM_EINVAL, "null argument");
  for (uint64_t i = 0; i < n_blocks; i++)
    if (comp_off[i + 1] < comp_off[i] || out_off[i + 1] < out_off[i])
      return inf_fail(inf, MM_EINVAL, "block %llu: offsets decrease", (unsigned long long)i);
  if (cudaSetDevice(inf->device) != cudaSuccess) return inf_fail(inf, MM_ECUDA, "cannot select device %d", inf->device);
  cudaStream_t st = inf->stream;
  float kernel_ms = 0;
  cudaEventRecord(inf->ev[0], st);
  for (uint64_t b = 0; b < n_blocks;) {
    /* a slice: consecutive blocks up to kSliceBytes of output and of input, at least one block */
    uint64_t e = b + 1;
    while (e < n_blocks && out_off[e + 1] - out_off[b] <= kSliceBytes && comp_off[e + 1] - comp_off[b] <= kSliceBytes) e++;
    const uint64_t ns = e - b, cbytes = comp_off[e] - comp_off[b], obytes = out_off[e] - out_off[b];
    cudaError_t ce = inf->d_comp.reserve(std::max<uint64_t>(cbytes, 1));
    if (ce == cudaSuccess) ce = inf->d_out.reserve(std::max<uint64_t>(obytes, 1));
    if (ce == cudaSuccess) ce = inf->d_coff.reserve(ns + 1);
    if (ce == cudaSuccess) ce = inf->d_ooff.reserve(ns + 1);
    if (ce == cudaSuccess) ce = inf->d_crc.reserve(ns);
    if (ce == cudaSuccess) ce = inf->d_status.reserve(ns);
    if (ce != cudaSuccess) return inf_fail(inf, MM_ENOMEM, "device allocation for %llu blocks failed: %s", (unsigned long long)ns, cudaGetErrorString(ce));
    inf->h_coff.resize(ns + 1);
    inf->h_ooff.resize(ns + 1);
    for (uint64_t i = 0; i <= ns; i++) {
      inf->h_coff[i] = comp_off[b + i] - comp_off[b];
      inf->h_ooff[i] = out_off[b + i] - out_off[b];
    }
    ce = cudaMemcpyAsync(inf->d_comp.get(), comp + comp_off[b], cbytes, cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(inf->d_coff.get(), inf->h_coff.data(), (ns + 1) * 8, cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(inf->d_ooff.get(), inf->h_ooff.data(), (ns + 1) * 8, cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(inf->d_crc.get(), crc + b, ns * 4, cudaMemcpyHostToDevice, st);
    if (ce != cudaSuccess) return inf_fail(inf, MM_ECUDA, "upload: %s", cudaGetErrorString(ce));
    cudaEventRecord(inf->ev[1], st);
    const unsigned grid = (unsigned)std::min<uint64_t>((uint64_t)inf->grid, (ns + kWarps - 1) / kWarps);
    k_inflate<<<grid, kWarps * 32, 0, st>>>(inf->d_comp.get(), inf->d_coff.get(), inf->d_ooff.get(), inf->d_crc.get(), ns,
                                            inf->d_out.get(), inf->d_status.get());
    ce = cudaGetLastError();
    if (ce != cudaSuccess) return inf_fail(inf, MM_ECUDA, "k_inflate: %s", cudaGetErrorString(ce));
    cudaEventRecord(inf->ev[2], st);
    inf->h_status.resize(ns);
    ce = cudaMemcpyAsync(inf->h_status.data(), inf->d_status.get(), ns * 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(out + out_off[b], inf->d_out.get(), obytes, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) return inf_fail(inf, MM_ECUDA, "inflate: %s", cudaGetErrorString(ce));
    float ms = 0;
    cudaEventElapsedTime(&ms, inf->ev[1], inf->ev[2]);
    kernel_ms += ms;
    for (uint64_t i = 0; i < ns; i++)
      if (inf->h_status[i] != MMI_OK) {
        if (bad_block) *bad_block = (int64_t)(b + i);
        return inf_fail(inf, MM_EINVAL, "block %llu: %s", (unsigned long long)(b + i), status_text(inf->h_status[i]));
      }
    b = e;
  }
  cudaEventRecord(inf->ev[2], st);
  cudaEventSynchronize(inf->ev[2]);
  cudaEventElapsedTime(&inf->ms[1], inf->ev[0], inf->ev[2]);
  inf->ms[0] = kernel_ms;
  return MM_OK;
}

}  // extern "C"
