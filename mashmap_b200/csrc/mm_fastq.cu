/*
 * mm_fastq.cu -- FASTQ parsed on the device: the kernels around mm_fastq.h and the mm_fastq handle of
 * include/mashmap_b200.h.
 *
 * A cut of the window (DESIGN §8):
 *   1. k_fq_count: the newlines of each 16 KiB tile (one CTA; 16-byte loads, a word mask, popc, a block reduce);
 *   2. cub::DeviceScan over the tile counts: the index of each tile's first newline;
 *   3. k_fq_lines: each tile ranks its newlines and writes their positions; line L is a header iff L % 4 == 0, so the
 *      record table follows from these positions alone; an atomicMin finds the first empty header line;
 *   4. k_fq_extent (one thread): how many records the cut returns and what it consumes (mmf_extent);
 *   5. k_fq_records, one thread per record: name and sequence, then two scans give the name and nibble offsets;
 *   6. k_fq_pack and k_fq_names: the nibbles and the names, balanced over output bytes (each thread finds its record by
 *      binary search), so a few 1 Mbp reads beside many short ones spread over the whole grid.
 * Only the nibbles (~0.5 B per base), the names and the table go back over PCIe. The tail of the window (the start of
 * the next record) moves to the front of the other window buffer for the next append.
 */
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "../../include/mashmap_b200.h"
#include "mm_devbuf.h"
#include "mm_fastq.h"
#include "mm_inflate.h"

namespace {

constexpr int kThreads = 256;
constexpr int kBytesPerThread = 64;
constexpr uint64_t kTile = (uint64_t)kThreads * kBytesPerThread; /* 16 KiB of text per CTA */
constexpr int kOutPerThread = 8;                                  /* output bytes per thread of the pack and name kernels */

thread_local std::string g_create_error;

struct Extent {
  uint64_t n_records, consumed, first_empty;
  int ended;
};

__global__ void __launch_bounds__(kThreads) k_fq_count(const uint8_t *__restrict__ text, uint64_t n, uint64_t *__restrict__ counts)
{
  typedef cub::BlockReduce<uint32_t, kThreads> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  const uint64_t pos = (uint64_t)blockIdx.x * kTile + (uint64_t)threadIdx.x * kBytesPerThread;
  uint32_t c = 0;
  if (pos + kBytesPerThread <= n) {
    const uint4 *p = (const uint4 *)(text + pos);
#pragma unroll
    for (int i = 0; i < kBytesPerThread / 16; i++) {
      const uint4 v = p[i];
      c += __popc(mmf_newline_mask(v.x)) + __popc(mmf_newline_mask(v.y)) + __popc(mmf_newline_mask(v.z)) + __popc(mmf_newline_mask(v.w));
    }
  } else {
    c = mmf_count_newlines(text, n, pos, kBytesPerThread);
  }
  const uint32_t s = Reduce(tmp).Sum(c);
  if (threadIdx.x == 0) counts[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) k_fq_lines(const uint8_t *__restrict__ text, uint64_t n, const uint64_t *__restrict__ base,
                                                      uint64_t *__restrict__ nl, unsigned long long *__restrict__ first_empty)
{
  typedef cub::BlockScan<uint32_t, kThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const uint64_t pos = (uint64_t)blockIdx.x * kTile + (uint64_t)threadIdx.x * kBytesPerThread;
  uint32_t c = 0;
#pragma unroll
  for (int i = 0; i < kBytesPerThread / 4; i++) c += __popc(mmf_newline_mask(mmf_word(text, n, pos + 4 * i)));
  uint32_t rank;
  Scan(tmp).ExclusiveSum(c, rank);
  uint64_t j = base[blockIdx.x] + rank;
  uint64_t empty = MMF_NONE;
  for (int i = 0; i < kBytesPerThread / 4 && c; i++) { /* the words again (from L1): ranks in order */
    for (uint32_t w = mmf_newline_mask(mmf_word(text, n, pos + 4 * i)); w; w &= w - 1) {
      const uint64_t p = pos + 4 * i + (uint64_t)((__ffs(w) - 1) >> 3);
      nl[j] = p;
      empty = min(empty, mmf_empty_header_after(text, n, j, p));
      j++;
      c--;
    }
  }
  if (empty != MMF_NONE) atomicMin(first_empty, (unsigned long long)empty);
}

__global__ void k_fq_extent(const uint8_t *__restrict__ text, const uint64_t *__restrict__ nl, uint64_t N, uint64_t n, int last,
                            Extent *__restrict__ ext)
{
  uint64_t fe = ext->first_empty;
  fe = min(fe, mmf_empty_header_after(text, n, ~0ULL, ~0ULL)); /* the window's first line */
  ext->n_records = mmf_extent(nl, N, n, last, fe, &ext->consumed, &ext->ended);
}

/* records [0, rmax]: the fields of those the cut returns, zero lengths for the rest (so the scans' last entry is the total) */
__global__ void __launch_bounds__(kThreads) k_fq_records(const uint8_t *__restrict__ text, uint64_t n, const uint64_t *__restrict__ nl,
                                                        uint64_t N, const Extent *__restrict__ ext, uint64_t rmax,
                                                        uint64_t *__restrict__ name_at, uint64_t *__restrict__ name_len,
                                                        uint64_t *__restrict__ seq_at, uint64_t *__restrict__ seq_len,
                                                        uint64_t *__restrict__ nib_bytes)
{
  const uint64_t R = ext->n_records;
  for (uint64_t r = (uint64_t)blockIdx.x * kThreads + threadIdx.x; r <= rmax; r += (uint64_t)gridDim.x * kThreads) {
    if (r < R) {
      const mmf_record f = mmf_fields(text, n, nl, N, r);
      name_at[r] = f.name;
      name_len[r] = f.name_len;
      seq_at[r] = f.seq;
      seq_len[r] = f.seq_len;
      nib_bytes[r] = (f.seq_len + 1) / 2;
    } else {
      name_len[r] = 0;
      seq_len[r] = 0;
      nib_bytes[r] = 0;
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_fq_pack(const uint8_t *__restrict__ text, const uint64_t *__restrict__ seq_at,
                                                     const uint64_t *__restrict__ seq_len, const uint64_t *__restrict__ nib_off,
                                                     uint64_t R, uint64_t total, uint8_t *__restrict__ out)
{
  const uint64_t o0 = ((uint64_t)blockIdx.x * kThreads + threadIdx.x) * kOutPerThread;
  if (o0 >= total) return;
  uint64_t r = mmf_find(nib_off, R, o0);
  const uint64_t o1 = min(total, o0 + kOutPerThread);
  for (uint64_t o = o0; o < o1; o++) {
    while (o >= nib_off[r + 1]) r++;
    out[o] = mmf_nib_byte(text + seq_at[r], seq_len[r], o - nib_off[r]);
  }
}

__global__ void __launch_bounds__(kThreads) k_fq_names(const uint8_t *__restrict__ text, const uint64_t *__restrict__ name_at,
                                                      const uint64_t *__restrict__ name_off, uint64_t R, uint64_t total,
                                                      char *__restrict__ out)
{
  const uint64_t o0 = ((uint64_t)blockIdx.x * kThreads + threadIdx.x) * kOutPerThread;
  if (o0 >= total) return;
  uint64_t r = mmf_find(name_off, R, o0);
  const uint64_t o1 = min(total, o0 + kOutPerThread);
  for (uint64_t o = o0; o < o1; o++) {
    while (o >= name_off[r + 1]) r++;
    out[o] = (char)text[name_at[r] + (o - name_off[r])];
  }
}

unsigned grid_for(uint64_t items, uint64_t per_cta)
{
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((items + per_cta - 1) / per_cta, 1u << 30));
}

/* pinned host memory owned by the handle */
struct Pinned {
  void *p = nullptr;
  uint64_t cap = 0;
  ~Pinned() { if (p) cudaFreeHost(p); }
  bool reserve(uint64_t bytes)
  {
    if (bytes <= cap) return true;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    const uint64_t c = std::max<uint64_t>(bytes, 4096) + bytes / 4;
    if (cudaMallocHost(&p, c) != cudaSuccess) {
      p = nullptr;
      cudaGetLastError();
      return false;
    }
    cap = c;
    return true;
  }
};

struct OutSet {
  Pinned table, names, nibbles; /* table: name_off [R+1], nib_off [R+1], seq_len [R] */
};

}  // namespace

struct mm_fastq {
  int device = -1;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[7] = {}; /* call start; then (begin, end) of the three kernel stretches */
  float ms[2] = {0, 0};
  std::string error;
  mm_devbuf<uint8_t> text[2]; /* the window, and the buffer its tail moves to */
  int cur = 0;
  uint64_t used = 0;
  mm_devbuf<uint64_t> counts, tile_base, nl, name_at, name_len, name_off, seq_at, seq_len, nib_bytes, nib_off;
  mm_devbuf<uint8_t> cub_tmp, d_nibbles, d_comp;
  mm_devbuf<char> d_names;
  mm_devbuf<uint64_t> d_coff, d_ooff;
  mm_devbuf<uint32_t> d_crc;
  mm_devbuf<int32_t> d_status;
  mm_devbuf<Extent> d_ext;
  Pinned h_small; /* N, then the extent and the totals */
  OutSet out[2];
  int out_next = 0;
  std::vector<uint64_t> h_coff, h_ooff;
  std::vector<int32_t> h_status;
  ~mm_fastq()
  {
    if (device >= 0) cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

static int fq_fail(mm_fastq *fq, int rc, const char *fmt, ...)
{
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  (fq ? fq->error : g_create_error) = buf;
  return rc;
}

/* room for `extra` more bytes of text at the end of the window (both window buffers: the tail moves between them) */
static cudaError_t window_room(mm_fastq *fq, uint64_t extra)
{
  const uint64_t need = fq->used + extra + 16;
  if (need <= fq->text[fq->cur].capacity()) return cudaSuccess;
  const uint64_t cap = std::max<uint64_t>(need, fq->text[fq->cur].capacity() + fq->text[fq->cur].capacity() / 2);
  cudaError_t e = fq->text[fq->cur].reserve_keep(cap, fq->used, fq->stream);
  if (e == cudaSuccess) e = fq->text[fq->cur ^ 1].reserve(cap);
  return e;
}

template <typename F>
static cudaError_t cub_run(mm_devbuf<uint8_t> &tmp, F &&f)
{
  size_t bytes = 0;
  cudaError_t e = f((void *)nullptr, bytes);
  if (e == cudaSuccess) e = tmp.reserve(std::max<size_t>(bytes, 1));
  if (e == cudaSuccess) e = f((void *)tmp.get(), bytes);
  return e;
}

extern "C" {

int mm_fastq_create(int device, mm_fastq **out)
{
  if (!out) return fq_fail(nullptr, MM_EINVAL, "null argument");
  *out = nullptr;
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return fq_fail(nullptr, MM_ENODEVICE, "no CUDA device: %s (this library has no CPU path)", cudaGetErrorString(e));
  if (device < 0 || device >= n_dev) return fq_fail(nullptr, MM_ENODEVICE, "device %d out of range (%d devices)", device, n_dev);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fq_fail(nullptr, MM_ENODEVICE, "cannot query device");
  if (prop.major != 9 || prop.minor != 0)
    return fq_fail(nullptr, MM_ENODEVICE, "device %d is sm_%d%d; this build is sm_90a only", device, prop.major, prop.minor);
  std::unique_ptr<mm_fastq> fq(new mm_fastq());
  fq->device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&fq->stream, cudaStreamNonBlocking) != cudaSuccess)
    return fq_fail(nullptr, MM_ECUDA, "cannot create stream");
  for (cudaEvent_t &ev : fq->ev)
    if (cudaEventCreate(&ev) != cudaSuccess) return fq_fail(nullptr, MM_ECUDA, "cannot create the timing events");
  if (fq->d_ext.reserve(1) != cudaSuccess || !fq->h_small.reserve(64)) return fq_fail(nullptr, MM_ENOMEM, "cannot allocate");
  *out = fq.release();
  return MM_OK;
}

int mm_fastq_destroy(mm_fastq *fq)
{
  delete fq;
  return MM_OK;
}

const char *mm_fastq_error(const mm_fastq *fq) { return fq ? fq->error.c_str() : g_create_error.c_str(); }

int mm_fastq_last_ms(const mm_fastq *fq, float ms[2])
{
  if (!fq || !ms) return MM_EINVAL;
  ms[0] = fq->ms[0];
  ms[1] = fq->ms[1];
  return MM_OK;
}

int mm_fastq_append_text(mm_fastq *fq, const uint8_t *text, uint64_t n)
{
  if (!fq) return fq_fail(nullptr, MM_EINVAL, "null handle");
  if (n == 0) return MM_OK;
  if (!text) return fq_fail(fq, MM_EINVAL, "null argument");
  if (cudaSetDevice(fq->device) != cudaSuccess) return fq_fail(fq, MM_ECUDA, "cannot select device %d", fq->device);
  cudaError_t e = window_room(fq, n);
  if (e != cudaSuccess) return fq_fail(fq, MM_ENOMEM, "window of %llu bytes: %s", (unsigned long long)(fq->used + n), cudaGetErrorString(e));
  e = cudaMemcpyAsync(fq->text[fq->cur].get() + fq->used, text, n, cudaMemcpyHostToDevice, fq->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(fq->stream);
  if (e != cudaSuccess) return fq_fail(fq, MM_ECUDA, "upload: %s", cudaGetErrorString(e));
  fq->used += n;
  return MM_OK;
}

int mm_fastq_append_blocks(mm_fastq *fq, const uint8_t *comp, const uint64_t *comp_off, const uint64_t *out_off,
                           const uint32_t *crc, uint64_t n_blocks, int64_t *bad_block)
{
  if (!fq) return fq_fail(nullptr, MM_EINVAL, "null handle");
  if (bad_block) *bad_block = -1;
  if (n_blocks == 0) return MM_OK;
  if (!comp_off || !out_off || !crc || (!comp && comp_off[n_blocks] > comp_off[0])) return fq_fail(fq, MM_EINVAL, "null argument");
  for (uint64_t i = 0; i < n_blocks; i++)
    if (comp_off[i + 1] < comp_off[i] || out_off[i + 1] < out_off[i])
      return fq_fail(fq, MM_EINVAL, "block %llu: offsets decrease", (unsigned long long)i);
  if (cudaSetDevice(fq->device) != cudaSuccess) return fq_fail(fq, MM_ECUDA, "cannot select device %d", fq->device);
  const uint64_t cbytes = comp_off[n_blocks] - comp_off[0], obytes = out_off[n_blocks] - out_off[0];
  cudaError_t e = window_room(fq, obytes);
  if (e == cudaSuccess) e = fq->d_comp.reserve(std::max<uint64_t>(cbytes, 1));
  if (e == cudaSuccess) e = fq->d_coff.reserve(n_blocks + 1);
  if (e == cudaSuccess) e = fq->d_ooff.reserve(n_blocks + 1);
  if (e == cudaSuccess) e = fq->d_crc.reserve(n_blocks);
  if (e == cudaSuccess) e = fq->d_status.reserve(n_blocks);
  if (e != cudaSuccess) return fq_fail(fq, MM_ENOMEM, "device allocation for %llu blocks failed: %s", (unsigned long long)n_blocks, cudaGetErrorString(e));
  fq->h_coff.resize(n_blocks + 1);
  fq->h_ooff.resize(n_blocks + 1);
  for (uint64_t i = 0; i <= n_blocks; i++) {
    fq->h_coff[i] = comp_off[i] - comp_off[0];
    fq->h_ooff[i] = out_off[i] - out_off[0];
  }
  cudaStream_t st = fq->stream;
  e = cudaMemcpyAsync(fq->d_comp.get(), comp + comp_off[0], cbytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(fq->d_coff.get(), fq->h_coff.data(), (n_blocks + 1) * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(fq->d_ooff.get(), fq->h_ooff.data(), (n_blocks + 1) * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(fq->d_crc.get(), crc, n_blocks * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    e = mmi_launch_inflate(fq->d_comp.get(), fq->d_coff.get(), fq->d_ooff.get(), fq->d_crc.get(), n_blocks,
                           fq->text[fq->cur].get() + fq->used, fq->d_status.get(), st);
  fq->h_status.resize(n_blocks);
  if (e == cudaSuccess) e = cudaMemcpyAsync(fq->h_status.data(), fq->d_status.get(), n_blocks * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fq_fail(fq, MM_ECUDA, "inflate: %s", cudaGetErrorString(e));
  for (uint64_t i = 0; i < n_blocks; i++)
    if (fq->h_status[i] != MMI_OK) {
      if (bad_block) *bad_block = (int64_t)i;
      return fq_fail(fq, MM_EINVAL, "block %llu: %s", (unsigned long long)i, mmi_status_text(fq->h_status[i]));
    }
  fq->used += obytes;
  return MM_OK;
}

int mm_fastq_cut(mm_fastq *fq, int last, mm_fastq_records *res)
{
  if (!fq) return fq_fail(nullptr, MM_EINVAL, "null handle");
  if (!res) return fq_fail(fq, MM_EINVAL, "null argument");
  memset(res, 0, sizeof *res);
  fq->ms[0] = fq->ms[1] = 0;
  if (cudaSetDevice(fq->device) != cudaSuccess) return fq_fail(fq, MM_ECUDA, "cannot select device %d", fq->device);
  cudaStream_t st = fq->stream;
  const uint64_t n = fq->used;
  const uint8_t *text = fq->text[fq->cur].get();
  OutSet &os = fq->out[fq->out_next];
  uint64_t *small = (uint64_t *)fq->h_small.p;
  cudaError_t e = cudaSuccess;
#define FQ_CHECK(what)                                                                                            \
  do {                                                                                                            \
    if (e != cudaSuccess) return fq_fail(fq, e == cudaErrorMemoryAllocation ? MM_ENOMEM : MM_ECUDA, "%s: %s", what, \
                                         cudaGetErrorString(e));                                                  \
  } while (0)
  cudaEventRecord(fq->ev[0], st);

  /* 1-2: newlines per tile, their scan, and the total N */
  const uint64_t tiles = std::max<uint64_t>(1, (n + kTile - 1) / kTile);
  e = fq->counts.reserve(tiles);
  if (e == cudaSuccess) e = fq->tile_base.reserve(tiles);
  FQ_CHECK("tile arrays");
  cudaEventRecord(fq->ev[1], st);
  k_fq_count<<<(unsigned)tiles, kThreads, 0, st>>>(text, n, fq->counts.get());
  e = cudaGetLastError();
  FQ_CHECK("k_fq_count");
  uint64_t *cnt = fq->counts.get(), *tb = fq->tile_base.get();
  e = cub_run(fq->cub_tmp, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, cnt, tb, (int64_t)tiles, st);
  });
  FQ_CHECK("tile scan");
  cudaEventRecord(fq->ev[2], st);
  e = cudaMemcpyAsync(small, tb + tiles - 1, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(small + 1, cnt + tiles - 1, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  FQ_CHECK("newline count");
  const uint64_t N = small[0] + small[1];

  /* 3-5: newline positions, the extent, the records and their offsets */
  const uint64_t rmax = N / 4 + 1; /* records [0, rmax) at most; entry rmax stays zero */
  e = fq->nl.reserve(std::max<uint64_t>(N, 1));
  for (mm_devbuf<uint64_t> *b : {&fq->name_at, &fq->name_len, &fq->name_off, &fq->seq_at, &fq->seq_len, &fq->nib_bytes, &fq->nib_off})
    if (e == cudaSuccess) e = b->reserve(rmax + 1);
  FQ_CHECK("record arrays");
  Extent ext0{0, 0, MMF_NONE, 0};
  e = cudaMemcpyAsync(fq->d_ext.get(), &ext0, sizeof ext0, cudaMemcpyHostToDevice, st);
  FQ_CHECK("extent upload");
  cudaEventRecord(fq->ev[3], st);
  if (n) {
    k_fq_lines<<<(unsigned)tiles, kThreads, 0, st>>>(text, n, tb, fq->nl.get(), (unsigned long long *)&fq->d_ext.get()->first_empty);
    e = cudaGetLastError();
    FQ_CHECK("k_fq_lines");
  }
  k_fq_extent<<<1, 1, 0, st>>>(text, fq->nl.get(), N, n, last, fq->d_ext.get());
  k_fq_records<<<grid_for(rmax + 1, kThreads), kThreads, 0, st>>>(text, n, fq->nl.get(), N, fq->d_ext.get(), rmax, fq->name_at.get(),
                                                                   fq->name_len.get(), fq->seq_at.get(), fq->seq_len.get(),
                                                                   fq->nib_bytes.get());
  e = cudaGetLastError();
  FQ_CHECK("k_fq_records");
  uint64_t *nlen = fq->name_len.get(), *noff = fq->name_off.get(), *nb = fq->nib_bytes.get(), *nboff = fq->nib_off.get();
  e = cub_run(fq->cub_tmp, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, nlen, noff, (int64_t)(rmax + 1), st);
  });
  if (e == cudaSuccess)
    e = cub_run(fq->cub_tmp, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(tmp, bytes, nb, nboff, (int64_t)(rmax + 1), st);
    });
  FQ_CHECK("record scans");
  cudaEventRecord(fq->ev[4], st);
  Extent *hext = (Extent *)(small + 2);
  e = cudaMemcpyAsync(hext, fq->d_ext.get(), sizeof(Extent), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(small, noff + rmax, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(small + 1, nboff + rmax, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  FQ_CHECK("record totals");
  const Extent ext = *hext;
  const uint64_t R = ext.n_records, name_total = small[0], nib_total = small[1];

  /* 6: nibbles and names, then everything back to pinned memory */
  e = fq->d_nibbles.reserve(std::max<uint64_t>(nib_total, 1));
  if (e == cudaSuccess) e = fq->d_names.reserve(std::max<uint64_t>(name_total, 1));
  FQ_CHECK("output arrays");
  if (!os.table.reserve((3 * R + 2) * 8) || !os.names.reserve(name_total + 1) || !os.nibbles.reserve(nib_total + 1))
    return fq_fail(fq, MM_ENOMEM, "cannot allocate pinned memory for %llu records", (unsigned long long)R);
  cudaEventRecord(fq->ev[5], st);
  if (nib_total)
    k_fq_pack<<<grid_for(nib_total, (uint64_t)kThreads * kOutPerThread), kThreads, 0, st>>>(text, fq->seq_at.get(), fq->seq_len.get(),
                                                                                            nboff, R, nib_total, fq->d_nibbles.get());
  if (name_total)
    k_fq_names<<<grid_for(name_total, (uint64_t)kThreads * kOutPerThread), kThreads, 0, st>>>(text, fq->name_at.get(), noff, R,
                                                                                              name_total, fq->d_names.get());
  e = cudaGetLastError();
  FQ_CHECK("k_fq_pack / k_fq_names");
  cudaEventRecord(fq->ev[6], st);
  uint64_t *tab = (uint64_t *)os.table.p;
  e = cudaMemcpyAsync(tab, noff, (R + 1) * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(tab + R + 1, nboff, (R + 1) * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && R) e = cudaMemcpyAsync(tab + 2 * R + 2, fq->seq_len.get(), R * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && name_total) e = cudaMemcpyAsync(os.names.p, fq->d_names.get(), name_total, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && nib_total) e = cudaMemcpyAsync(os.nibbles.p, fq->d_nibbles.get(), nib_total, cudaMemcpyDeviceToHost, st);
  FQ_CHECK("download");

  /* the tail (the start of the next record) to the front of the other buffer */
  const uint64_t keep = n - ext.consumed;
  if (keep) {
    e = cudaMemcpyAsync(fq->text[fq->cur ^ 1].get(), text + ext.consumed, keep, cudaMemcpyDeviceToDevice, st);
    FQ_CHECK("window tail");
    fq->cur ^= 1;
  }
  fq->used = keep;
  e = cudaStreamSynchronize(st);
  FQ_CHECK("cut");
#undef FQ_CHECK
  float a = 0, b = 0, c = 0;
  cudaEventElapsedTime(&a, fq->ev[1], fq->ev[2]);
  cudaEventElapsedTime(&b, fq->ev[3], fq->ev[4]);
  cudaEventElapsedTime(&c, fq->ev[5], fq->ev[6]);
  fq->ms[0] = a + b + c;
  cudaEventRecord(fq->ev[1], st);
  cudaEventSynchronize(fq->ev[1]);
  cudaEventElapsedTime(&fq->ms[1], fq->ev[0], fq->ev[1]);

  res->n_records = R;
  res->name_off = tab;
  res->nib_off = tab + R + 1;
  res->seq_len = tab + 2 * R + 2;
  res->names = (const char *)os.names.p;
  res->nibbles = (const uint8_t *)os.nibbles.p;
  res->consumed = ext.consumed;
  res->ended = ext.ended;
  fq->out_next ^= 1;
  return MM_OK;
}

}  // extern "C"
