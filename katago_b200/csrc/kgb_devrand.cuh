// The reference's Rand on the device (core/rand.h:149-185, 245-298; core/rand.cpp:335-363; core/rand_helpers.h:29-66):
// PCG32 + XorShift1024* for the integers, 53-bit doubles, polar-method Gaussians with the cached second value,
// Marsaglia-Tsang gamma draws - SURVEY.md §8a rows a22/a25.  One thread drives a generator; its state lives in global memory
// (one per game) and is initialised on the host from a seed string exactly like Rand::init (kgb_rand.cpp).
#pragma once
#include <stdint.h>

namespace kgb {

struct DevRandState {
  unsigned long long a[16];
  unsigned long long aIdx;
  unsigned long long pcg;
  double storedGaussian;
  int hasGaussian;
  int pad;
};

struct DevRand {
  DevRandState s;
  __device__ __forceinline__ uint32_t nextUInt() {
    s.pcg = s.pcg * 6364136223846793005ULL + 1442695040888963407ULL;
    const uint32_t x = (uint32_t)(((s.pcg >> 18) ^ s.pcg) >> 27);
    const int rot = (int)(s.pcg >> 59);
    const uint32_t p = rot == 0 ? x : ((x >> rot) | (x << (32 - rot)));
    unsigned long long a0 = s.a[s.aIdx];
    s.aIdx = (s.aIdx + 1) & 15;
    unsigned long long a1 = s.a[s.aIdx];
    a1 ^= a1 << 31;
    a1 ^= a1 >> 11;
    a0 ^= a0 >> 30;
    s.a[s.aIdx] = a0 ^ a1;
    const unsigned long long res = s.a[s.aIdx] * 1181783497276652981ULL;
    return p + (uint32_t)(res >> 32);
  }
  __device__ __forceinline__ unsigned long long nextUInt64() {
    const unsigned long long lo = nextUInt();
    const unsigned long long hi = (unsigned long long)nextUInt() << 32;
    return lo | hi;
  }
  __device__ __forceinline__ double nextDouble() {
    double x;
    do {
      const unsigned long long bits = nextUInt64() & ((1ULL << 53) - 1ULL);
      x = (double)bits / (double)(1ULL << 53);
    } while(!(x >= 0.0 && x < 1.0));
    return x;
  }
  __device__ double nextGaussian() {
    if(s.hasGaussian) { s.hasGaussian = 0; return s.storedGaussian; }
    double v1, v2, q;
    do {
      v1 = nextDouble() * 2.0 - 1.0;
      v2 = nextDouble() * 2.0 - 1.0;
      q = v1 * v1 + v2 * v2;
    } while(q >= 1 || q == 0);
    const double multiplier = sqrt(-2 * log(q) / q);
    s.storedGaussian = v2 * multiplier;
    s.hasGaussian = 1;
    return v1 * multiplier;
  }
  // A gamma draw without its final scaling: the Marsaglia-Tsang draw and, for shape a <= 1 (drawn with shape a + 1 and scaled by
  // U^(1/a)), the uniform U.  Returns the unscaled draw; boostU >= 0 means the result still has to be multiplied by pow(boostU, inva) - a pure function
  // that a caller holding many draws can evaluate in parallel (the stream of random numbers is consumed in exactly the reference's order).
  __device__ double nextGammaCore(double a, double& boostU, double& inva) {
    bool small = false;
    inva = 0.0; boostU = -1.0;
    if(a <= 1.0) { small = true; inva = 1.0 / a; a = a + 1.0; }
    const double dd = a - 1.0 / 3.0;
    const double c = (1.0 / 3.0) / sqrt(dd);
    double r;
    while(true) {
      const double x = nextGaussian();
      const double vtmp = 1.0 + c * x;
      if(vtmp <= 0.0) continue;
      const double v = vtmp * vtmp * vtmp;
      const double u = nextDouble();
      const double xx = x * x;
      if(u < 1.0 - 0.0331 * xx * xx) { r = dd * v; break; }
      if(u == 0.0 || log(u) < 0.5 * xx + dd * (1.0 - v + log(v))) { r = dd * v; break; }
    }
    if(small && inva != 0.0) boostU = nextDouble();   // drawn AFTER the inner gamma, like the recursion in the reference
    return r;
  }
};

}  // namespace kgb
