// The DDPM step's Gaussian noise: a pure function of (task seed, frame's index in its task, frame's timestep index,
// element), so that every multi-GPU mode draws the same bits as one GPU (DESIGN.md section 7).  Shared by
// cfg_ddpm_kernel and the d4d_op_ddpm_noise kernel; oracle/ddpm_oracle.py restates it on the host.
//
// Element e of a frame's [4, h, w] NCHW latent takes word e % 4 of Philox4x32-10 (Random123) with key = seed (low word
// first) and counter (e / 4, frame, timestep index, 0).  A word x maps to u = (x + 0.5) * 2^-32 in (0, 1); Box-Muller
// on (u0, u1) gives z0, z1 and on (u2, u3) gives z2, z3, in fp64, rounded once to the sample's type.
#pragma once
#include <cstdint>

namespace d4d {

__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c[0], hi0 = __umulhi(0xD2511F53u, c[0]);
    const uint32_t lo1 = 0xCD9E8D57u * c[2], hi1 = __umulhi(0xCD9E8D57u, c[2]);
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
  }
}

// z[0..3] of elements 4q .. 4q + 3, in fp64
__device__ __forceinline__ void ddpm_normal4(unsigned long long seed, uint32_t q, uint32_t frame, uint32_t ts_index,
                                             double z[4]) {
  uint32_t c[4] = {q, frame, ts_index, 0u};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  const double two_pi = 6.283185307179586, scale = 2.3283064365386963e-10;  // 2 pi (the double nearest), 2^-32
  for (int p = 0; p < 2; ++p) {
    const double u0 = (c[2 * p] + 0.5) * scale, u1 = (c[2 * p + 1] + 0.5) * scale;
    const double r = sqrt(-2.0 * log(u0)), a = two_pi * u1;
    z[2 * p] = r * cos(a);
    z[2 * p + 1] = r * sin(a);
  }
}

// fp64 -> bf16 rounded once (round to nearest even on the 45 dropped mantissa bits; |z| is far from bf16's subnormals
// and overflow), returned as the fp32 that holds it exactly
__device__ __forceinline__ float round_to_bf16(double z) {
  unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(z));
  b += ((1ull << 44) - 1) + ((b >> 45) & 1);
  b &= ~((1ull << 45) - 1);
  return __double2float_rn(__longlong_as_double(static_cast<long long>(b)));
}

// the noise sample in the step's arithmetic: bf16 in the bf16-emulating step (upstream draws it in the model output's
// dtype), fp32 otherwise
template <bool BF16>
__device__ __forceinline__ float round_noise(double z) {
  return BF16 ? round_to_bf16(z) : __double2float_rn(z);
}

}  // namespace d4d
