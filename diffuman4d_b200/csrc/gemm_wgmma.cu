// Warpgroup-MMA (wgmma) GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M, N] = A[M, K] * W[N, K]^T  (+bias[N]) (+rowvec[image(m), N]) (+residual[M, N])   -> bf16
//
// * operands are bf16, K-major, staged by TMA into 128B-swizzled shared memory (mbarrier ring, as deep as fits)
// * three warpgroups: warpgroup 0 is the TMA producer (one thread; it hands most of its registers to the others), and
//   warpgroups 1 and 2 each own 64 rows of the 128-row tile and issue wgmma.m64nBNk16 with fp32 accumulators in
//   registers.  The kernel is persistent (grid = #SMs) and walks tiles n-fastest, so CTAs that run concurrently share
//   the same A rows through L2; the producer runs ahead into the next tile while the MMA warpgroups run the epilogue.
// * "conv" mode turns the A loader into an implicit-GEMM gather: the A tile for k-block (tap, c0) is a 4-D TMA box
//   {64 ch, BW, BH, BN} of the NHWC activation at spatial offset (ky-1, kx-1); out-of-bounds rows/cols are zero-filled
//   by TMA, which is exactly the conv's zero padding.  K = 9*Cin, weights are pre-laid-out as [Cout][tap][Cin].
// * "two-source" mode reads the first kb_split k-blocks from A and the rest from A2 (a channel concat that is never
//   materialised: resnet shortcut 1x1 conv over [hidden | skip]).
// * epilogue options: +bias (fp32), +per-image row vector (time-embedding projection), SiLU / scale, +residual, fused
//   GroupNorm statistics, fused K/V all-gather, GEGLU (a * gelu_erf(g); weight rows interleaved in groups of 8, so that
//   each thread holds matching a / g accumulators).
//
// Replaces, on the reference path: F.linear / 1x1 conv / 3x3 conv calls of diffusers ResnetBlock2D, Attention,
// FeedForward, Transformer2DModel (reference call sites: unet_multiview_blocks.py:274,423,585,
// transformer_multiview.py:46-77, attention.py:73,116,142).
#include "kernels.h"
#include "wgmma.cuh"

namespace d4d {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int BAR_BYTES = 1024;                 // barrier block in front of the ring keeps the stages 1024-B aligned
constexpr int NUM_THREADS = 384;                // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int MAX_SMEM = 227 * 1024;

// Tile width BN (the wgmma N) is a template parameter; the ring takes as many stages as fit (at most 8).
template <int BN>
struct GemmCfg {
  static constexpr int STAGE_BYTES = A_BYTES + BN * BLOCK_K * 2;
  static constexpr int STAGES_FIT = (MAX_SMEM - 1024 - BAR_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  static constexpr int SMEM = 1024 + BAR_BYTES + STAGES * STAGE_BYTES;
};

struct TileCoord {
  int m0;          // plain: first row.  conv: unused
  int n_img0, y0, x0;
  int pa, pb;      // conv, n_phases == 4: sub-pixel phase of this tile (0 otherwise)
};

template <bool kConv>
__device__ __forceinline__ void tile_coords(const GemmKernelArgs& a, int m_tile, TileCoord& t) {
  if (!kConv) {
    t.m0 = m_tile * BLOCK_M;
    t.n_img0 = t.y0 = t.x0 = 0;
    t.pa = t.pb = 0;
  } else {
    const int ph = a.n_phases > 1 ? m_tile / a.tiles_per_phase : 0;  // phases outermost: concurrent CTAs share a weight slab
    m_tile -= ph * a.tiles_per_phase;
    t.pa = ph >> 1;
    t.pb = ph & 1;
    int tx = m_tile % a.tiles_x;
    int r = m_tile / a.tiles_x;
    int ty = r % a.tiles_y;
    int tn = r / a.tiles_y;
    t.m0 = 0;
    t.x0 = tx * a.BW;
    t.y0 = ty * a.BH;
    t.n_img0 = tn * a.BN;
  }
}

// output row (pixel / token index) of tile row rr, the image it belongs to, and whether it exists
template <bool kConv>
__device__ __forceinline__ void row_of(const GemmKernelArgs& a, const TileCoord& tc, int rr, long long& row, int& img,
                                       bool& valid) {
  if (!kConv) {
    row = static_cast<long long>(tc.m0) + rr;
    valid = row < a.M;
    img = a.rows_per_image > 0 ? static_cast<int>(row / a.rows_per_image) : 0;
  } else {
    const int bx = rr % a.BW;
    const int r2 = rr / a.BW;
    const int by = r2 % a.BH;
    const int bn = r2 / a.BH;
    const int x = tc.x0 + bx, y = tc.y0 + by, n = tc.n_img0 + bn;
    valid = (x < a.W) && (y < a.H) && (n < a.n_img);
    row = (static_cast<long long>(n) * a.out_H + (y * a.out_sy + a.out_oy + tc.pa)) * a.out_W + (x * a.out_sx + a.out_ox + tc.pb);
    img = n;
  }
}

// Epilogue feature bits of the kernel template: a CLEAR bit compiles the feature out, a set bit is still checked at run
// time.  gemm_run picks the instantiation whose bits equal the launch's features, or the E_ALL one.
enum : int { E_BIAS = 1, E_ROWVEC = 2, E_ACT = 4, E_RES = 8, E_STATS = 16, E_KV = 32, E_ALL = 63 };

template <int BN, bool kGeglu, bool kConv, int kEpi>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2,
                  const __grid_constant__ CUtensorMap tmap_b, const GemmKernelArgs a) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);  // [STAGES]
  uint64_t* empty = full + STAGES;                      // [STAGES]
  uint8_t* ring = smem + BAR_BYTES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // tells the compiler the role branches are warp-uniform
  const int lane = threadIdx.x & 31;
  const int total_tiles = a.m_tiles * a.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (a.kb_split < a.k_blocks) tma_prefetch_desc(&tmap_a2);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // barriers are set up while the previous kernel drains
  pdl_launch_dependents();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const uint32_t tx_bytes = A_BYTES + static_cast<uint32_t>(a.block_n) * BLOCK_K * 2;
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_tile = tile / a.n_tiles;
        const int n_tile = tile % a.n_tiles;
        TileCoord tc;
        tile_coords<kConv>(a, m_tile, tc);
        const int n0 = n_tile * a.block_n;
        for (int kb = 0; kb < a.k_blocks; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = ring + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full[stage], tx_bytes);
          if (!kConv) {
            if (kb < a.kb_split) tma_load_2d(sa, &tmap_a, &full[stage], kb * BLOCK_K, tc.m0);
            else tma_load_2d(sa, &tmap_a2, &full[stage], (kb - a.kb_split) * BLOCK_K, tc.m0);
            tma_load_2d(sb, &tmap_b, &full[stage], kb * BLOCK_K, n0);
          } else {
            const int tap = kb / a.cin_blocks;
            const int cb = kb - tap * a.cin_blocks;
            tma_load_4d(sa, &tmap_a, &full[stage], cb * BLOCK_K, tc.x0 * a.in_stride + a.tap_dx[tap] + tc.pb,
                        tc.y0 * a.in_stride + a.tap_dy[tap] + tc.pa, tc.n_img0);
            tma_load_2d(sb, &tmap_b, &full[stage], tap * a.Cin + cb * BLOCK_K, n0 + (tc.pa * 2 + tc.pb) * a.N);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== MMA warpgroups + epilogue =====================
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;   // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp & 3;          // warp within the warpgroup: rows 16 wq .. 16 wq + 15 of the warpgroup's 64
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int r_base = wg * 64 + wq * 16 + (lane >> 2);  // tile rows r_base and r_base + 8 belong to this thread
  const int c_base = 2 * (lane & 3);                   // columns 8j + c_base, +1 of fragment j
  const uint32_t ring_u32 = smem_u32(ring);

  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int m_tile = tile / a.n_tiles;
    const int n_tile = tile % a.n_tiles;
    TileCoord tc;
    tile_coords<kConv>(a, m_tile, tc);
    const int n0 = n_tile * a.block_n;

    // ---- main loop: one k-block in flight behind the one being issued; a stage is released once its MMAs retired
    int prev_stage = -1;
    for (int kb = 0; kb < a.k_blocks; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = ring_u32 + stage * Cfg::STAGE_BYTES + wg * 64 * 128;
      const uint32_t sb = ring_u32 + stage * Cfg::STAGE_BYTES + A_BYTES;
      const uint64_t adesc = make_wgmma_desc(sa, 16, 1024);
      const uint64_t bdesc = make_wgmma_desc(sb, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
        // advancing 16 bf16 along K inside the 128B swizzle atom = +32 bytes = +2 in the (addr >> 4) field
        const int scale_d = (kb | k) != 0 ? 1 : 0;
        if constexpr (BN == 64) wgmma_ss_n64(acc, adesc + 2 * k, bdesc + 2 * k, scale_d);
        else if constexpr (BN == 128) wgmma_ss_n128(acc, adesc + 2 * k, bdesc + 2 * k, scale_d);
        else wgmma_ss_n256(acc, adesc + 2 * k, bdesc + 2 * k, scale_d);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (wg_leader) mbar_arrive(&empty[prev_stage]);

    // ---- epilogue: straight from the accumulator registers
    long long rows[2];
    int imgs[2];
    bool valid[2];
    row_of<kConv>(a, tc, r_base, rows[0], imgs[0], valid[0]);
    row_of<kConv>(a, tc, r_base + 8, rows[1], imgs[1], valid[1]);

    if constexpr (kGeglu) {
      // tile columns 16p .. 16p+7 are the a half, 16p+8 .. 16p+15 the g half of output columns n0/2 + 8p .. + 7
      const bool has_bias = (kEpi & E_BIAS) && a.bias != nullptr;
#pragma unroll
      for (int p = 0; p < BN / 16; ++p) {
        if (16 * p >= a.block_n || n0 + 16 * p >= a.N) break;
        float2 ba = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
        if (has_bias) {
          ba = __ldg(reinterpret_cast<const float2*>(a.bias + n0 + 16 * p + c_base));
          bg = __ldg(reinterpret_cast<const float2*>(a.bias + n0 + 16 * p + 8 + c_base));
        }
        const int ocol = n0 / 2 + 8 * p + c_base;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!valid[h]) continue;
          const float a0 = acc[8 * p + 2 * h] + ba.x, a1 = acc[8 * p + 2 * h + 1] + ba.y;
          const float g0 = acc[8 * p + 4 + 2 * h] + bg.x, g1 = acc[8 * p + 4 + 2 * h + 1] + bg.y;
          *reinterpret_cast<uint32_t*>(a.out + static_cast<size_t>(rows[h]) * a.ldo + ocol) =
              pack_bf16x2(a0 * gelu_erf_f(g0), a1 * gelu_erf_f(g1));
        }
      }
    } else {
      const bool has_bias = (kEpi & E_BIAS) && a.bias != nullptr, has_rv = (kEpi & E_ROWVEC) && a.rowvec != nullptr;
      const bool has_res = (kEpi & E_RES) && a.residual != nullptr, has_stats = (kEpi & E_STATS) && a.stats != nullptr;
      const bool has_act = (kEpi & E_ACT) && a.act == 1, has_scale = (kEpi & E_ACT) && a.out_scale != 1.0f;
      const bool has_kv = (kEpi & E_KV) && a.kv_world > 0;
      // statistics: the 16 rows of a warp lie in ONE image (gemm_prepare checks it); the warp's first row has the
      // smallest (x, y, image) / token index, so when it is outside the tensor the whole warp is
      const long long row0 = __shfl_sync(0xffffffffu, rows[0], 0);
      const bool stats_on = has_stats && __shfl_sync(0xffffffffu, valid[0] ? 1 : 0, 0);
      const int stats_img = !kConv ? static_cast<int>(row0 / a.stats_rows) : __shfl_sync(0xffffffffu, imgs[0], 0);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int cl = 8 * j + c_base;
        const int col = n0 + cl;
        if (8 * j >= a.block_n || n0 + 8 * j >= a.N) break;  // (warp-uniform: N and block_n are multiples of 16)
        float2 b2 = make_float2(0.f, 0.f);
        if (has_bias) b2 = __ldg(reinterpret_cast<const float2*>(a.bias + col));
        float sv[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          sv[h][0] = sv[h][1] = 0.f;
          if (!valid[h]) continue;
          float f0 = acc[4 * j + 2 * h] + b2.x, f1 = acc[4 * j + 2 * h + 1] + b2.y;
          if (has_rv) {
            const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.rowvec + static_cast<size_t>(imgs[h]) * a.ld_rowvec + col));
            f0 += v.x; f1 += v.y;
          }
          if (has_act) { f0 = silu_f(f0); f1 = silu_f(f1); }
          if (has_scale) { f0 *= a.out_scale; f1 *= a.out_scale; }
          if (has_res) {  // plain load: the residual may alias the output (in-place add)
            const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.residual + static_cast<size_t>(rows[h]) * a.ld_res + col));
            f0 += v.x; f1 += v.y;
          }
          const uint32_t o = pack_bf16x2(f0, f1);
          if (has_stats) {  // statistics of what is stored: the rounded values
            const float2 rv = unpack_bf16x2(o);
            sv[h][0] = rv.x; sv[h][1] = rv.y;
          }
          if (has_kv && col >= a.kv_col0) {
            // fused all-gather: the K|V columns of the QKV projection go straight into every rank's gathered K/V buffer
            // (peer memory over NVLink; own rank included) at this rank's global token rows
            const long long half = rows[h] / a.kv_rows_local;
            const long long grow = half * a.kv_rows_global + a.kv_row_offset + (rows[h] - half * a.kv_rows_local);
            const size_t off = static_cast<size_t>(grow) * a.kv_ld + (col - a.kv_col0);
#pragma unroll 1
            for (int rk = 0; rk < a.kv_world; ++rk) *reinterpret_cast<uint32_t*>(a.kv_dst[rk] + off) = o;
          } else {
            *reinterpret_cast<uint32_t*>(a.out + static_cast<size_t>(rows[h]) * a.ldo + col) = o;
          }
        }
        if (has_stats) {
          // column sums over the warp's 16 rows: lanes with equal lane % 4 hold the same two columns
          float s0 = sv[0][0] + sv[1][0], s1 = sv[0][1] + sv[1][1];
          float q0 = sv[0][0] * sv[0][0] + sv[1][0] * sv[1][0], q1 = sv[0][1] * sv[0][1] + sv[1][1] * sv[1][1];
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, m);
            s1 += __shfl_xor_sync(0xffffffffu, s1, m);
            q0 += __shfl_xor_sync(0xffffffffu, q0, m);
            q1 += __shfl_xor_sync(0xffffffffu, q1, m);
          }
          if (stats_on && lane < 4) {  // fixed point: integer adds commute, the result is independent of tile order
            unsigned long long* st = reinterpret_cast<unsigned long long*>(a.stats) + (static_cast<size_t>(stats_img) * a.N + col) * 2;
            atomicAdd(st + 0, static_cast<unsigned long long>(__float2ll_rn(s0 * kGnSumScale)));
            atomicAdd(st + 1, static_cast<unsigned long long>(__float2ll_rn(q0 * kGnSqScale)));
            atomicAdd(st + 2, static_cast<unsigned long long>(__float2ll_rn(s1 * kGnSumScale)));
            atomicAdd(st + 3, static_cast<unsigned long long>(__float2ll_rn(q1 * kGnSqScale)));
          }
        }
      }
    }
  }
}

}  // namespace

int gemm_prepare(const GemmDesc& d, GemmLaunch* L) {
  D4D_REQUIRE(d.N % 16 == 0, "GEMM N must be a multiple of 16");
  D4D_REQUIRE(d.out != nullptr && d.A != nullptr && d.Wt != nullptr, "null operand");
  GemmKernelArgs& a = L->args;
  memset(&a, 0, sizeof(a));
  int dev = 0, sms = 0;
  D4D_CUDA_OK(cudaGetDevice(&dev));
  D4D_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int bn = d.block_n;
  if (bn <= 0) {
    // tile width 64, 128 or 256 (the last N tile may overhang; its extra columns are not stored): the widest one unless a
    // narrower one wastes fewer SM-waves of the persistent grid (cost ~ waves * (block_n + fixed per-tile work))
    const long long rows = d.conv ? static_cast<long long>(d.n_img) * d.H * d.W : d.M;
    const long long m_tiles_est = (rows + BLOCK_M - 1) / BLOCK_M;
    long long best_cost = -1;
    for (int c = 64; c <= 256; c *= 2) {
      const long long tiles = m_tiles_est * ((d.N + c - 1) / c);
      const long long waves = (tiles + sms - 1) / sms;
      const long long cost = waves * (c + 64) + (static_cast<long long>((d.N + c - 1) / c) * c - d.N) / 4;
      if (best_cost < 0 || cost <= best_cost) { best_cost = cost; bn = c; }
    }
  }
  D4D_REQUIRE(bn >= 16 && bn <= 256 && bn % 16 == 0 && (d.block_n <= 0 || d.N % bn == 0), "no valid block_n");
  a.block_n = bn;
  a.n_tiles = (d.N + bn - 1) / bn;
  a.N = d.N;
  a.bias = d.bias;
  a.rowvec = d.rowvec;
  a.ld_rowvec = d.ld_rowvec;
  a.rows_per_image = d.rows_per_image;
  a.residual = d.residual;
  a.ld_res = d.ld_res;
  a.out = d.out;
  a.ldo = d.ldo;
  a.geglu = d.geglu;
  a.act = d.act;
  a.out_scale = d.out_scale;
  a.stats = d.stats;
  a.stats_rows = d.stats_rows > 0 ? d.stats_rows : 1;
  D4D_REQUIRE(d.stats == nullptr || (!d.geglu && d.kv_world == 0), "GroupNorm statistics: plain / conv epilogue only");
  D4D_REQUIRE(d.stats == nullptr || d.conv || (d.stats_rows > 0 && d.stats_rows % 32 == 0), "statistics need rows-per-image % 32 == 0");
  a.kv_world = d.kv_world;
  a.kv_col0 = d.kv_col0;
  a.kv_ld = d.kv_ld;
  a.kv_rows_local = d.kv_rows_local > 0 ? d.kv_rows_local : 1;
  a.kv_rows_global = d.kv_rows_global;
  a.kv_row_offset = d.kv_row_offset;
  for (int i = 0; i < 8; ++i) a.kv_dst[i] = d.kv_dst[i];
  D4D_REQUIRE(d.kv_world >= 0 && d.kv_world <= 8 && (d.kv_world == 0 || (d.kv_col0 % 16 == 0 && d.kv_ld % 8 == 0 && !d.geglu)), "K/V scatter arguments");
  D4D_REQUIRE(d.ldo % 8 == 0 && (d.residual == nullptr || d.ld_res % 8 == 0) &&
              (d.rowvec == nullptr || d.ld_rowvec % 8 == 0), "leading dimensions must be multiples of 8");

  if (!d.conv) {
    D4D_REQUIRE(d.K1 > 0 && d.K1 % 8 == 0 && d.K2 % 8 == 0, "K must be a multiple of 8");
    D4D_REQUIRE(d.A2 == nullptr || d.K1 % BLOCK_K == 0, "two-source GEMM needs K1 % 64 == 0");
    a.mode = 0;
    a.M = d.M;
    a.m_tiles = (d.M + BLOCK_M - 1) / BLOCK_M;
    a.kb_split = (d.K1 + BLOCK_K - 1) / BLOCK_K;
    const int kb2 = d.A2 ? (d.K2 + BLOCK_K - 1) / BLOCK_K : 0;
    a.k_blocks = a.kb_split + kb2;
    const int K = d.K1 + (d.A2 ? d.K2 : 0);
    if (int rc = make_tmap_2d(&L->tmap_a, d.A, d.M, d.K1, d.lda, BLOCK_K, BLOCK_M, 128)) return rc;
    if (d.A2) {
      if (int rc = make_tmap_2d(&L->tmap_a2, d.A2, d.M, d.K2, d.lda2, BLOCK_K, BLOCK_M, 128)) return rc;
    } else {
      L->tmap_a2 = L->tmap_a;
    }
    if (int rc = make_tmap_2d(&L->tmap_b, d.Wt, d.N, K, K, BLOCK_K, bn, 128)) return rc;
  } else {
    D4D_REQUIRE(d.Cin % 8 == 0, "conv Cin must be a multiple of 8");
    D4D_REQUIRE(d.conv_kind >= 0 && d.conv_kind <= 3, "conv_kind");
    D4D_REQUIRE(d.conv_kind != 1 || (d.H % 2 == 0 && d.W % 2 == 0), "stride-2 conv needs even H, W");
    a.mode = 1;
    a.n_img = d.n_img; a.Cin = d.Cin;
    // tap table, grid of output positions, output pixel mapping (GemmKernelArgs)
    a.in_stride = 1; a.out_sy = a.out_sx = 1; a.out_oy = a.out_ox = 0;
    a.n_phases = 1;
    if (d.conv_kind >= 2) {  // sub-pixel phase (a, b): rows {-1, 0} for a = 0, {0, +1} for a = 1 (same for columns)
      const int pa = d.conv_kind == 3 ? 0 : d.up_a, pb = d.conv_kind == 3 ? 0 : d.up_b;  // kind 3: the tile adds its phase
      a.n_taps = 4;
      for (int t = 0; t < 4; ++t) {
        a.tap_dy[t] = static_cast<signed char>((t >> 1) + pa - 1);
        a.tap_dx[t] = static_cast<signed char>((t & 1) + pb - 1);
      }
      a.H = d.H; a.W = d.W; a.out_H = 2 * d.H; a.out_W = 2 * d.W;
      a.out_sy = a.out_sx = 2; a.out_oy = pa; a.out_ox = pb;
      if (d.conv_kind == 3) a.n_phases = 4;
    } else {
      a.n_taps = 9;
      for (int t = 0; t < 9; ++t) {
        a.tap_dy[t] = static_cast<signed char>(t / 3 - 1);
        a.tap_dx[t] = static_cast<signed char>(t % 3 - 1);
      }
      if (d.conv_kind == 1) { a.in_stride = 2; a.H = d.H / 2; a.W = d.W / 2; }
      else { a.H = d.H; a.W = d.W; }
      a.out_H = a.H; a.out_W = a.W;
    }
    a.M = d.n_img * a.H * a.W;
    a.cin_blocks = (d.Cin + BLOCK_K - 1) / BLOCK_K;
    a.k_blocks = a.n_taps * a.cin_blocks;
    a.kb_split = a.k_blocks;
    // spatial tile: BW x BH x BN = 128 output positions
    int bw = 16; while (bw > a.W) bw >>= 1;
    int bh = 128 / bw; while (bh > a.H && bh > 1) bh >>= 1;
    // H, W need not be powers of two: the tile may overhang, TMA zero-fills and the epilogue masks
    int bnimg = 128 / (bw * bh);
    D4D_REQUIRE(bw * bh * bnimg == 128 && bnimg <= 256, "conv tile shape");
    D4D_REQUIRE(d.stats == nullptr || (bw * bh) % 32 == 0, "statistics need 32-row warps inside one image");
    a.BW = bw; a.BH = bh; a.BN = bnimg;
    a.tiles_x = (a.W + bw - 1) / bw;
    a.tiles_y = (a.H + bh - 1) / bh;
    const int tiles_n = (d.n_img + bnimg - 1) / bnimg;
    a.tiles_per_phase = a.tiles_x * a.tiles_y * tiles_n;
    a.m_tiles = a.tiles_per_phase * a.n_phases;
    a.M *= a.n_phases;  // output positions of the launch (FLOP count)
    if (int rc = make_tmap_nhwc(&L->tmap_a, d.A, d.n_img, d.H, d.W, d.Cin, BLOCK_K, bw, bh, bnimg, 128, a.in_stride)) return rc;
    L->tmap_a2 = L->tmap_a;
    const uint64_t kw = static_cast<uint64_t>(a.n_taps) * d.Cin;
    if (int rc = make_tmap_2d(&L->tmap_b, d.Wt, static_cast<uint64_t>(d.N) * a.n_phases, kw, kw, BLOCK_K, bn, 128)) return rc;
  }
  const int total = a.m_tiles * a.n_tiles;
  L->grid = total < sms ? total : sms;
  return 0;
}

namespace {

using GemmKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const GemmKernelArgs);
struct GemmVariant {
  int bn;
  bool geglu, conv;
  int epi;
  GemmKernelFn fn;
  int smem;
};
#define D4D_GV(BN, G, C, E) {BN, G, C, E, gemm_wgmma_kernel<BN, G, C, E>, GemmCfg<BN>::SMEM}
#define D4D_GV_SET(BN)                                                                                                \
  /* plain GEMM: qkv | proj_in, shortcut | attn out, ff2 | proj_out, conv_in */                                       \
  D4D_GV(BN, false, false, 0), D4D_GV(BN, false, false, E_BIAS), D4D_GV(BN, false, false, E_BIAS | E_RES),           \
  D4D_GV(BN, false, false, E_BIAS | E_RES | E_STATS), D4D_GV(BN, false, false, E_ALL),                                \
  /* 3x3 convs: resnet conv1 | conv2 | down / up sampling */                                                          \
  D4D_GV(BN, false, true, E_BIAS | E_ROWVEC | E_STATS), D4D_GV(BN, false, true, E_BIAS | E_RES | E_STATS),           \
  D4D_GV(BN, false, true, E_BIAS | E_STATS), D4D_GV(BN, false, true, E_ALL),                                          \
  /* GEGLU projection (only the bias bit matters) */                                                                  \
  D4D_GV(BN, true, false, E_BIAS)
// the feature sets the UNet plan launches (csrc/unet.cu) at the tile widths it picks, plus E_ALL kernels for the rest
const GemmVariant kGemmVariants[] = {
    D4D_GV_SET(128), D4D_GV_SET(256),
    D4D_GV(64, false, false, E_ALL), D4D_GV(64, false, true, E_ALL), D4D_GV(64, true, false, E_BIAS),
};
#undef D4D_GV_SET
#undef D4D_GV
constexpr int kNumGemmVariants = sizeof(kGemmVariants) / sizeof(kGemmVariants[0]);

int gemm_variant_of(const GemmKernelArgs& a) {
  const bool conv = a.mode != 0, geglu = a.geglu != 0;
  const int bn = a.block_n <= 64 ? 64 : a.block_n <= 128 ? 128 : 256;  // narrower tiles run on a wider kernel, masked
  int need = 0;
  if (a.bias) need |= E_BIAS;
  if (!geglu) {
    if (a.rowvec) need |= E_ROWVEC;
    if (a.act == 1 || a.out_scale != 1.0f) need |= E_ACT;
    if (a.residual) need |= E_RES;
    if (a.stats) need |= E_STATS;
    if (a.kv_world > 0) need |= E_KV;
  }
  int generic = -1;
  for (int i = 0; i < kNumGemmVariants; ++i) {
    const GemmVariant& v = kGemmVariants[i];
    if (v.bn != bn || v.geglu != geglu || v.conv != conv) continue;
    if (v.epi == need) return i;
    if ((v.epi & need) == need && (generic < 0 || v.epi == E_ALL)) generic = i;  // geglu: E_BIAS covers {} as well
  }
  return generic;
}

}  // namespace

int gemm_run(const GemmLaunch& L, cudaStream_t stream) {
  static PerDeviceOnce attr_once[kNumGemmVariants];
  const int vi = gemm_variant_of(L.args);
  D4D_REQUIRE(vi >= 0, "no GEMM kernel instantiation covers this launch");
  const GemmVariant& v = kGemmVariants[vi];
  if (int rc = ensure_dyn_smem(v.fn, v.smem, attr_once[vi])) return rc;
  D4D_CUDA_OK(launch_pdl(v.fn, dim3(L.grid), dim3(NUM_THREADS), v.smem, stream, L.tmap_a, L.tmap_a2, L.tmap_b, L.args));
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

double gemm_flops(const GemmLaunch& L) {
  return 2.0 * static_cast<double>(L.args.M) * L.args.N * (static_cast<double>(L.args.k_blocks) * BLOCK_K);
}

}  // namespace d4d
