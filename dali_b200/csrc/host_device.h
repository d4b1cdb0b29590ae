// dali_b200/csrc/host_device.h -- what the kernel cores share between their two builds: nvcc compiles them for the device, a host
// compiler for tools/emul and the CPU tests.  Plain C++ with no CUDA header, so that the host builds can include it.
#ifndef DALI_B200_CSRC_HOST_DEVICE_H_
#define DALI_B200_CSRC_HOST_DEVICE_H_

#if defined(__CUDACC__)
#define DB_HD __host__ __device__ __forceinline__
#else
#define DB_HD inline
#endif

namespace dalib200 {

struct Identity {
  template <class T> DB_HD const T &operator()(const T &x) const { return x; }
};

// The last index i in [lo, hi] with key(d[i]) <= v, or lo when there is none; lo <= hi.
//
// This is how a batched kernel maps a flat work item v to its sample: key(d[i]) is the first item of sample i, so the keys ascend, and a
// sample with no work shares its first item with the next sample.  Taking the *last* match skips such empty samples.  The comparison is
// made in the types of key(d[i]) and v, which the caller picks.
template <class T, class V, class Key = Identity>
DB_HD int last_at_most(const T *d, int lo, int hi, V v, const Key &key = {}) {
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (key(d[mid]) <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_HOST_DEVICE_H_
