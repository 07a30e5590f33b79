// kaminpar_b200: what the graph readers (kmp_metis.cuh, kmp_parhip.cuh) share: the input file, its stream to the
// device through pinned staging buffers, the prefix fetch of device bytes, the check of a caller's device bytes and
// the prelude of a reader call. Included at the end of kmp_lp.cu before both readers.
#pragma once

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

namespace {

constexpr uint64_t kReadChunk = 32ull << 20; // bytes per pinned staging buffer of stream_file

// An input file opened read-only, closed with the object.
struct InputFile {
  const char *path = nullptr;
  int fd = -1;
  uint64_t len = 0;
  ~InputFile() {
    if (fd >= 0) {
      close(fd);
    }
  }
  // opens `p` and takes its size; files of 2^56 bytes or more are refused (len is set before)
  int open(const char *p) {
    path = p;
    fd = ::open(p, O_RDONLY);
    struct stat info {};
    if (fd < 0 || fstat(fd, &info) != 0) {
      return fail(KMP_ERR_INVALID, std::string("cannot open ") + p);
    }
    len = static_cast<uint64_t>(info.st_size);
    if (len >= (1ull << 56)) {
      return fail(KMP_ERR_UNSUPPORTED, "files of 2^56 bytes or more are not supported");
    }
    return KMP_OK;
  }
  // pread until the `size` bytes at `off` are in dst; a read error or an early end is refused
  int read(uint8_t *dst, uint64_t size, uint64_t off) const {
    while (size > 0) {
      const ssize_t got = pread(fd, dst, size, static_cast<off_t>(off));
      if (got <= 0) {
        return fail(KMP_ERR_INVALID, std::string("cannot read ") + path);
      }
      dst += got;
      size -= static_cast<uint64_t>(got);
      off += static_cast<uint64_t>(got);
    }
    return KMP_OK;
  }
};

// the two pinned staging buffers of stream_file and the events of the copies out of them
struct FileStaging {
  cudaStream_t st = nullptr;
  uint8_t *buf[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  ~FileStaging() {
    if (st != nullptr) {
      cudaStreamSynchronize(st); // no copy reads a buffer any more
    }
    for (int b = 0; b < 2; ++b) {
      if (buf[b] != nullptr) {
        cudaFreeHost(buf[b]);
      }
      if (ev[b] != nullptr) {
        cudaEventDestroy(ev[b]);
      }
    }
  }
};

// Streams the file's bytes into dst (device) on h's stream through the two pinned buffers of `stage` (the caller's,
// so that they outlive the work it queues after), kReadChunk bytes each: reading one chunk overlaps the copy of the
// previous one. Starts h's call clock. queued(end) runs once the copy of bytes [0, end) is queued, to launch the work
// on them; its error ends the stream.
template <typename Queued> int stream_file(kmp_lp_handle *h, FileStaging &stage, const InputFile &f, uint8_t *dst,
                                           Queued &&queued) {
  const cudaStream_t st = h->stream;
  stage.st = st;
  const uint64_t len = f.len, chunk = std::min<uint64_t>(len, kReadChunk);
  for (int b = 0; b < 2; ++b) {
    KMP_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&stage.buf[b]), chunk, cudaHostAllocDefault));
    KMP_CUDA(cudaEventCreateWithFlags(&stage.ev[b], cudaEventDisableTiming));
  }
  KMP_CUDA(call_clock_start(h, st));
  for (uint64_t off = 0, idx = 0; off < len; off += chunk, ++idx) {
    const int b = static_cast<int>(idx & 1u);
    const uint64_t size = std::min<uint64_t>(chunk, len - off);
    if (idx >= 2) {
      KMP_CUDA(cudaEventSynchronize(stage.ev[b])); // the copy of chunk idx - 2 is out of this buffer
    }
    int rc = f.read(stage.buf[b], size, off);
    if (rc != KMP_OK) {
      return rc;
    }
    KMP_CUDA(cudaMemcpyAsync(dst + off, stage.buf[b], size, cudaMemcpyHostToDevice, st));
    KMP_CUDA(cudaEventRecord(stage.ev[b], st));
    rc = queued(off + size);
    if (rc != KMP_OK) {
      return rc;
    }
  }
  return KMP_OK;
}

// the first `size` of the device bytes d_bytes into dst, copied on h's stream and waited for
int fetch_device_prefix(kmp_lp_handle *h, uint8_t *dst, const uint8_t *d_bytes, uint64_t size) {
  KMP_CUDA(cudaMemcpyAsync(dst, d_bytes, size, cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  return KMP_OK;
}

// The bytes of a parse call: non-null unless empty, 16-byte aligned, below 2^56 bytes and device memory on h's device.
int check_device_bytes(const kmp_lp_handle *h, const void *d_bytes, uint64_t len) {
  if (d_bytes == nullptr && len > 0) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if ((reinterpret_cast<uintptr_t>(d_bytes) & 15u) != 0) {
    return fail(KMP_ERR_INVALID, "the device bytes must be 16-byte aligned");
  }
  if (len >= (1ull << 56)) {
    return fail(KMP_ERR_UNSUPPORTED, "inputs of 2^56 bytes or more are not supported");
  }
  if (len > 0) { // host memory or another device's memory would reach the kernels as a raw pointer
    cudaPointerAttributes attr{};
    const bool on_device = cudaPointerGetAttributes(&attr, d_bytes) == cudaSuccess &&
                           (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) &&
                           attr.device == h->device;
    cudaGetLastError(); // an unregistered host pointer leaves no sticky error
    if (!on_device) {
      return fail(KMP_ERR_INVALID, "the bytes must be device memory on the handle's device");
    }
  }
  return KMP_OK;
}

// The prelude of a reader call: null arguments are refused, the report is zeroed and given the reader's fields by
// fill(*report), a handle inside a stepping call is refused, then the reader's own checks() run and h's device is
// selected.
template <typename Report, typename Fill, typename Checks>
int reader_begin(kmp_lp_handle *h, const void *out, Report *report, Fill &&fill, Checks &&checks) {
  if (h == nullptr || out == nullptr || report == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  std::memset(report, 0, sizeof(*report));
  fill(*report);
  if (h->step.open) {
    return fail(KMP_ERR_INVALID, "the handle is inside a stepping call");
  }
  const int rc = checks();
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaSetDevice(h->device));
  return KMP_OK;
}

} // namespace
