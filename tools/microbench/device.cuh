// Geometry of the current device, so that the microbenchmarks fill every SM and convert times to clocks on any part.
#pragma once
#include <cuda_runtime.h>

static inline int dev_sms() {
  int d = 0, v = 0;
  cudaGetDevice(&d);
  cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d);
  return v;
}
// maximum SM clock in Hz (the clock the timings are converted with; a power-capped part may run below it)
static inline double dev_clock_hz() {
  int d = 0, khz = 0;
  cudaGetDevice(&d);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, d);
  return khz * 1e3;
}
