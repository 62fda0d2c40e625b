// The data-parallel exchange step of the path as a C-ABI entry (SURVEY.md section 8b / 8e): ONE all-reduce (average) over
// the flat fp32 gradient bucket on the caller's NCCL communicator and stream.
//
// Replaces: the gradient bucketing + all-reduce of the DistributedDataParallel wrapper slowfast/models/build.py:66-76 puts
// around the model (one ncclAllReduce per 25 MB bucket, sum, then a division kernel per bucket).  The engine's backward has
// already written every gradient into one contiguous bucket, so the exchange is a single in-place ncclAllReduce with
// ncclAvg (NCCL >= 2.10).  NCCL is resolved at run time (dlopen of the libnccl the process already loaded - torch's bundled
// one in a torch process): the library has no link-time NCCL dependency and still loads on a box without NCCL.
#include <cstdint>
#include <cstdio>
#include <dlfcn.h>

#include "../../include/slowfast_b200.h"
#include "runtime.h"

namespace sfb {
// the two NCCL enums used (nccl.h: ncclFloat = 7, ncclSum = 0, ncclAvg = 4) and entry points, resolved lazily
typedef int (*nccl_allreduce_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef const char* (*nccl_errstr_fn)(int);
static nccl_allreduce_fn g_allreduce = nullptr;
static nccl_errstr_fn g_errstr = nullptr;

static int resolve_nccl() {
  if (g_allreduce) return 0;
  void* h = nullptr;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  // RTLD_NOLOAD first: use the copy this process already holds (torch's), never a second NCCL beside it
  for (const char* n : names)
    if (!h) h = dlopen(n, RTLD_NOW | RTLD_NOLOAD);
  if (!h) h = dlopen(nullptr, RTLD_NOW);  // symbols may be in the global namespace already
  void* f = h ? dlsym(h, "ncclAllReduce") : nullptr;
  if (!f) {
    for (const char* n : names) {
      if (f) break;
      void* h2 = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (h2) {
        f = dlsym(h2, "ncclAllReduce");
        h = h2;
      }
    }
  }
  if (!f) {
    set_error("sfb_allreduce_flat: ncclAllReduce not found (no libnccl.so.2 loaded or loadable)");
    return -30;
  }
  g_allreduce = reinterpret_cast<nccl_allreduce_fn>(f);
  g_errstr = reinterpret_cast<nccl_errstr_fn>(dlsym(h, "ncclGetErrorString"));
  return 0;
}
}  // namespace sfb

extern "C" int sfb_allreduce_flat(float* buf, int64_t count, void* nccl_comm, int32_t average, void* stream) {
  if (count <= 0) return 0;
  if (!nccl_comm || !buf) {
    sfb::set_error("sfb_allreduce_flat: null communicator or buffer");
    return -10;
  }
  if (int rc = sfb::resolve_nccl()) return rc;
  const int ncclFloat = 7, ncclSum = 0, ncclAvg = 4;
  const int rc = sfb::g_allreduce(buf, buf, size_t(count), ncclFloat, average ? ncclAvg : ncclSum, nccl_comm,
                                  (cudaStream_t)stream);
  if (rc != 0) {
    sfb::set_error("sfb_allreduce_flat: ncclAllReduce failed: %s", sfb::g_errstr ? sfb::g_errstr(rc) : "?");
    return -31;
  }
  return 0;
}
