// Host program over 6dpose_b200/csrc/lm_buffer.h (tests/test_device_buffer.py).  "nodevice": run where every allocation
// fails; "device": run on a GPU.  Prints one line per failed check and exits non-zero if there was one.
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <utility>

#include "lm_buffer.h"

static int failures = 0;
#define CHECK(c)                                                 \
  do {                                                           \
    if (!(c)) {                                                  \
      printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c);        \
      ++failures;                                                \
    }                                                            \
  } while (0)

template <typename A>
static bool holds_nothing(const A& a) { return a.empty() && a.size() == 0 && a.get() == nullptr; }

static void without_device() {
  DeviceArray<int> a;
  CHECK(a.reserve(16) != cudaSuccess);
  CHECK(holds_nothing(a));
  CHECK(a.assign(8) != cudaSuccess);
  CHECK(holds_nothing(a));
  a.reset();
  CHECK(holds_nothing(a));
  PinnedArray<double> p;
  CHECK(p.reserve(4) != cudaSuccess);
  CHECK(holds_nothing(p));
  Stream s;
  CHECK(s.create(cudaStreamNonBlocking) != cudaSuccess);
  CHECK(s.get() == nullptr);
  Event e;
  CHECK(e.create(cudaEventDisableTiming) != cudaSuccess);
  CHECK(e.get() == nullptr);
  cudaGetLastError();
}  // the failed owners are destroyed here

static void with_device() {
  DeviceArray<int> a;
  CHECK(a.reserve(100) == cudaSuccess && a.size() == 100 && a.get() != nullptr);
  int* p = a.get();
  CHECK(a.reserve(100) == cudaSuccess && a.get() == p && a.size() == 100);
  CHECK(a.reserve(50) == cudaSuccess && a.get() == p && a.size() == 100);  // never shrinks
  CHECK(a.reserve(0) == cudaSuccess && a.get() == p && a.size() == 100);
  CHECK(a.reserve(200) == cudaSuccess && a.size() == 200 && a.get() != nullptr);
  CHECK(a.assign(10) == cudaSuccess && a.size() == 10);
  CHECK(a.assign(10) == cudaSuccess && a.size() == 10);
  CHECK(a.assign(0) == cudaSuccess && holds_nothing(a));
  CHECK(a.assign(10) == cudaSuccess);
  p = a.get();
  DeviceArray<int> b(std::move(a));
  CHECK(holds_nothing(a) && b.get() == p && b.size() == 10);
  DeviceArray<int> c;
  CHECK(c.reserve(3) == cudaSuccess);
  c = std::move(b);
  CHECK(holds_nothing(b) && c.get() == p && c.size() == 10);

  PinnedArray<int> h;
  CHECK(h.reserve(4) == cudaSuccess && h.size() == 4);
  for (int i = 0; i < 4; ++i) h[i] = 7 * i;
  CHECK(cudaMemcpy(c.get(), h.get(), 4 * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess);
  int back[4] = {0, 0, 0, 0};
  CHECK(cudaMemcpy(back, c.get(), sizeof(back), cudaMemcpyDeviceToHost) == cudaSuccess);
  CHECK(back[0] == 0 && back[1] == 7 && back[2] == 14 && back[3] == 21);

  // growing past the whole device: the allocator's ordinary error, and the array holds nothing (not its old size)
  size_t free_b = 0, total_b = 0;
  CHECK(cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && total_b > 0);
  DeviceArray<uint8_t> big;
  CHECK(big.reserve(1024) == cudaSuccess && big.size() == 1024);
  CHECK(big.reserve(total_b + ((size_t)1 << 30)) == cudaErrorMemoryAllocation);
  CHECK(holds_nothing(big));
  cudaGetLastError();
  CHECK(big.reserve(1024) == cudaSuccess && big.size() == 1024);

  Stream s;
  CHECK(s.create(cudaStreamNonBlocking) == cudaSuccess && s.get() != nullptr);
  Event e;
  CHECK(e.create(cudaEventDisableTiming) == cudaSuccess && e.get() != nullptr);
  CHECK(cudaEventRecord(e.get(), s.get()) == cudaSuccess && cudaStreamSynchronize(s.get()) == cudaSuccess);
  cudaEvent_t raw = e.get();
  Event f(std::move(e));
  CHECK(e.get() == nullptr && f.get() == raw);
  CHECK(cudaGetLastError() == cudaSuccess);
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  if (!strcmp(argv[1], "nodevice")) without_device();
  else if (!strcmp(argv[1], "device")) with_device();
  else return 2;
  if (failures == 0) printf("OK\n");
  return failures ? 1 : 0;
}
