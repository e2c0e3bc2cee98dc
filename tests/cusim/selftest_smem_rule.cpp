// Self-test of the emulation's dynamic shared memory launch rule (48 KB unless cudaFuncSetAttribute raised it, 227 KB at most),
// of CUSIM_SMEM_MONOTONIC=1 (a call that lowers a kernel's limit fails) and of the per-thread last-error word.
#include "cuda_runtime.h"
#include <stdio.h>
#include <stdlib.h>
#include <thread>
static int ran = 0;
__global__ void k(int) { ran = 1; }
int main() {
  ::cusim::launch(dim3(1), dim3(32), 60000, [&]() { k(0); }, reinterpret_cast<const void*>(+k));
  int e1 = cudaGetLastError(); int r1 = ran;
  int a = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 60000);
  ::cusim::launch(dim3(1), dim3(32), 60000, [&]() { k(0); }, reinterpret_cast<const void*>(+k));
  int e2 = cudaGetLastError();
  int b = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 300000);
  printf("first: err %d ran %d | attr %d second: err %d ran %d | too large attr %d\n", e1, r1, a, e2, ran, b);
  int ok = e1 == 1 && r1 == 0 && a == 0 && e2 == 0 && ran == 1 && b == 1;
  // lowering the limit: allowed, except in the monotonic mode
  const bool monotonic = getenv("CUSIM_SMEM_MONOTONIC") && getenv("CUSIM_SMEM_MONOTONIC")[0] == '1';
  const int lower = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 50000);
  const int raise = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 70000);
  printf("lower: %d raise: %d (monotonic %d)\n", lower, raise, monotonic ? 1 : 0);
  ok = ok && lower == (monotonic ? 1 : 0) && raise == 0;
  // a failed launch on another host thread leaves this thread's error word alone, and the other thread sees its own
  int other = -1;
  std::thread t([&] {
    ::cusim::launch(dim3(1), dim3(32), 100000, [&]() { k(0); }, reinterpret_cast<const void*>(+k));
    other = cudaGetLastError();
  });
  t.join();
  const int mine = cudaGetLastError();
  printf("other thread: err %d, this thread: err %d\n", other, mine);
  ok = ok && other == 1 && mine == 0;
  return !ok;
}
