// Warpgroup-MMA (wgmma) GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M, N] = A[M, K] * W[N, K]^T  (+bias[N]) (+rowvec[image(m), N]) (+residual[M, N])   -> bf16
//
// * operands are bf16, K-major, staged by TMA into 128B-swizzled shared memory (mbarrier ring, as deep as fits)
// * three warpgroups: warpgroup 0 is the TMA producer (one thread; it hands most of its registers to the others), and
//   warpgroups 1 and 2 each own 64 MI rows of the 128 MI-row tile (MI = 1, or 2 for the larger convs) and issue MI
//   wgmma.m64nBNk16 per k16 slice against one B descriptor, with fp32 accumulators in registers: at MI = 2 a weight tile
//   feeds twice the rows, which cuts the operand bytes a CTA pulls from L2 per FLOP from 1/128 + 1/BN to 1/256 + 1/BN and
//   halves the TMA issues and mbarrier round trips per FLOP.  The kernel is persistent (grid = #SMs) and walks tiles n-fastest, so CTAs that run concurrently share
//   the same A rows through L2; the producer runs ahead into the next tile while the MMA warpgroups run the epilogue.
// * plain GEMMs stage the epilogue in shared memory: each MMA warpgroup writes its finished 64 x BN bf16 rows into 32-column
//   slabs (64B-swizzled, conflict-free), and one thread TMA-stores them and goes on into the next tile's MMAs while the
//   stores drain.  The residual tile is TMA-loaded into the same slabs during the first k-block.
// * ping-pong schedule (plain staged GEMMs, chosen per shape): each MMA warpgroup owns whole 128-row tiles, as two 64-row
//   blocks (MI = 2, staging slabs for 128 rows each), and the two take turns: warpgroup i & 1 runs the i-th tile of the
//   CTA's sequence.  Two named barriers order the main loops (tile i's MMAs are all issued before tile i + 1's start), so
//   one warpgroup's epilogue runs while the other's MMAs keep the tensor cores busy.  The epilogue body is the same per
//   64-row block, so outputs and statistics are bit-identical to the cooperative schedule.
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
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB per 128 rows; a stage holds MI of them
constexpr int BAR_BYTES = 1024;                 // barrier block in front of the ring keeps the stages 1024-B aligned
constexpr int NUM_THREADS = 384;                // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int MAX_SMEM = 227 * 1024;

// staged epilogue: a slab is 64 rows x 32 columns of bf16 (64 B per row, TMA box {32, 64}, 64-byte swizzle)
constexpr int SLAB_COLS = 32;
constexpr int SLAB_BYTES = 64 * SLAB_COLS * 2;

// Tile width BN (the wgmma N) and the m64 blocks per warpgroup MI (tile rows = 128 MI, or 128 under ping-pong, where one
// warpgroup owns the whole tile) are template parameters; after the staging slabs of both warpgroups (64 MI rows each;
// plain GEMM only), the ring takes as many stages as fit (at most 8).
template <int BN, int MI, bool kStaged, bool kPingPong>
struct GemmCfg {
  static constexpr int TILE_A_BYTES = kPingPong ? A_BYTES : MI * A_BYTES;
  static constexpr int STAGE_BYTES = TILE_A_BYTES + BN * BLOCK_K * 2;
  static constexpr int STAGING_BYTES = kStaged ? 2 * 64 * MI * BN * 2 : 0;
  static constexpr int STAGES_FIT = (MAX_SMEM - 1024 - BAR_BYTES - STAGING_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  static constexpr int SMEM = 1024 + BAR_BYTES + STAGES * STAGE_BYTES + STAGING_BYTES;
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
enum : int { E_BIAS = 1, E_ROWVEC = 2, E_ACT = 4, E_RES = 8, E_STATS = 16, E_KV = 32, E_ALL = 63, E_STAGED_ALL = E_ALL & ~E_KV };
// Instantiations with the staged epilogue: plain GEMMs.  Convs store from registers (their output pixels are not a row
// range), and so do the E_KV kernels (they serve the K/V scatter and, as E_ALL, the rare feature sets no other kernel has).
__host__ __device__ constexpr bool gemm_staged(bool conv, int epi) { return !conv && !(epi & E_KV); }

// ping-pong: hardware barriers 3 and 4 hand the turn to issue MMAs to warpgroup 0 / 1 (1 and 2 are the epilogue barriers)
constexpr int ORDER_BAR = 3;

template <int BN, int MI, bool kGeglu, bool kConv, int kEpi, bool kPingPong>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2,
                  const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_c,
                  const __grid_constant__ CUtensorMap tmap_r, const GemmKernelArgs a) {
  constexpr bool kStaged = gemm_staged(kConv, kEpi);
  static_assert(MI == 1 || (kConv && MI == 2) || kPingPong, "256-row tiles: conv mode only (a plain tile is 128 rows)");
  static_assert(!kPingPong || (kStaged && MI == 2), "ping-pong: staged plain GEMMs, one warpgroup per 128-row tile");
  using Cfg = GemmCfg<BN, MI, kStaged, kPingPong>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);  // [STAGES]
  uint64_t* empty = full + STAGES;                      // [STAGES]
  uint64_t* res_full = empty + STAGES;                  // [2]: residual tile of MMA warpgroup 0 / 1 landed
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
      mbar_init(&empty[i], kPingPong ? 1 : 2);  // one arrival per MMA warpgroup that reads the stage
    }
    mbar_init(&res_full[0], 1);
    mbar_init(&res_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // barriers are set up while the previous kernel drains
  pdl_launch_dependents();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      const uint32_t tx_bytes = Cfg::TILE_A_BYTES + static_cast<uint32_t>(a.block_n) * BLOCK_K * 2;
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_tile = tile / a.n_tiles;
        const int n_tile = tile % a.n_tiles;
        TileCoord tc;
        tile_coords<kConv>(a, m_tile, tc);
        const int n0 = n_tile * a.block_n;
        for (int kb = 0; kb < a.k_blocks; ++kb) {
          mbar_wait_nocall(&empty[stage], phase ^ 1);
          uint8_t* sa = ring + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::TILE_A_BYTES;
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
  const int wg = (warp >> 2) - 1;   // 0 / 1: rows [64 MI wg, 64 MI (wg + 1)) of the tile (ping-pong: all rows of every
                                    // other tile), as MI blocks of 64
  const int wq = warp & 3;          // warp within the warpgroup: rows 16 wq .. 16 wq + 15 of each 64-row block
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int wg_row0 = kPingPong ? 0 : wg * 64 * MI;          // the warpgroup's first tile row
  const int r_base = wg_row0 + wq * 16 + (lane >> 2);       // tile rows r_base + 64 mi and + 8 belong to this thread
  const int c_base = 2 * (lane & 3);                   // columns 8j + c_base, +1 of fragment j
  const uint32_t ring_u32 = smem_u32(ring);
  // staged epilogue: this warpgroup's slabs (64 rows x BN per 64-row block), and the offset of this thread's (row r_base,
  // columns c_base, +1) in a slab; the 64-byte swizzle moves the 16-byte chunk c of row r to c ^ ((r >> 1) & 3), which for
  // rows r_base, r_base + 8 is (lane >> 3) & 3: the 8 rows of a warp store land in 8 different chunks, 32 different banks
  constexpr int STG_BLOCK = 64 * BN * 2;
  const bool staged = kStaged && a.staged;
  uint8_t* stg = ring + STAGES * Cfg::STAGE_BYTES + wg * MI * STG_BLOCK;
  const uint32_t stg_u32 = smem_u32(stg) + (r_base - wg_row0) * 64 + c_base * 2;
  const int stg_xor = (lane >> 3) & 3;
  const bool has_res = (kEpi & E_RES) && !kGeglu && a.residual != nullptr;
  const int out_cols = kGeglu ? a.N / 2 : a.N;
  uint32_t res_phase = 0;

  int stage = 0;
  uint32_t phase = 0;
  // ping-pong: the k-blocks of the other warpgroup's tiles pass this warpgroup's ring counters by
  const auto skip_stages = [&](int n) {
    stage += n;
    while (stage >= STAGES) { stage -= STAGES; phase ^= 1; }
  };
  if (kPingPong && wg == 1) {
    skip_stages(a.k_blocks);
    named_barrier_arrive(ORDER_BAR, 256);  // warpgroup 0 issues the MMAs of the first tile
  }
  const int tile_step = kPingPong ? 2 * gridDim.x : gridDim.x;
  float acc[MI][BN / 2];
  for (int tile = blockIdx.x + (kPingPong ? wg * gridDim.x : 0); tile < total_tiles; tile += tile_step) {
    const int m_tile = tile / a.n_tiles;
    const int n_tile = tile % a.n_tiles;
    TileCoord tc;
    tile_coords<kConv>(a, m_tile, tc);
    const int n0 = n_tile * a.block_n;
    // staged: the output columns and slabs of this tile, and whether this warpgroup has any rows inside the tensor
    const int ocol0 = kGeglu ? n0 / 2 : n0;
    const int ocols = min(kGeglu ? a.block_n / 2 : a.block_n, out_cols - ocol0);
    const int n_slabs = (ocols + SLAB_COLS - 1) / SLAB_COLS;
    // staged: this warpgroup's 64-row blocks of the tile that lie inside the tensor, from output row orow0 on
    const int orow0 = tc.m0 + wg_row0;
    const int live_blocks = staged ? max(0, min(MI, (a.M - orow0 + 63) / 64)) : 0;

    // ---- main loop: one k-block in flight behind the one being issued; a stage is released once its MMAs retired
    if (kPingPong) named_barrier_sync(ORDER_BAR + wg, 256);  // the previous tile's MMAs are all issued
    int prev_stage = -1;
    for (int kb = 0; kb < a.k_blocks; ++kb) {
      mbar_wait_nocall(&full[stage], phase);
      const uint32_t sa = ring_u32 + stage * Cfg::STAGE_BYTES + wg_row0 * 128;
      const uint32_t sb = ring_u32 + stage * Cfg::STAGE_BYTES + Cfg::TILE_A_BYTES;
      const uint64_t adesc = make_wgmma_desc(sa, 16, 1024);
      const uint64_t bdesc = make_wgmma_desc(sb, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
        // advancing 16 bf16 along K inside the 128B swizzle atom = +32 bytes = +2 in the (addr >> 4) field
        const int scale_d = (kb | k) != 0 ? 1 : 0;
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) {
          // the warpgroup's next 64 rows: + 64 * 128 bytes = + 512 in the (addr >> 4) field; same B descriptor
          const uint64_t ad = adesc + 512 * mi + 2 * k, bd = bdesc + 2 * k;
          if constexpr (BN == 64) wgmma_ss_n64(acc[mi], ad, bd, scale_d);
          else if constexpr (BN == 128) wgmma_ss_n128(acc[mi], ad, bd, scale_d);
          else if constexpr (BN == 160) wgmma_ss_n160(acc[mi], ad, bd, scale_d);
          else if constexpr (BN == 192) wgmma_ss_n192(acc[mi], ad, bd, scale_d);
          else wgmma_ss_n256(acc[mi], ad, bd, scale_d);
        }
      }
      wgmma_commit();
      if (kb == 0 && staged && wg_leader) {
        // the previous tile's stores must have read the slabs before they are refilled (or rewritten by the epilogue,
        // after the barrier there); then the residual tile comes in under this tile's MMAs.  A tile reads only the
        // residual rows and columns it stores itself, so the residual may alias the output.
        bulk_wait_group_read<0>();
        if (has_res && live_blocks > 0) {
          mbar_expect_tx(&res_full[wg], live_blocks * n_slabs * SLAB_BYTES);
          for (int mi = 0; mi < live_blocks; ++mi)
            for (int s = 0; s < n_slabs; ++s)
              tma_load_2d(stg + mi * STG_BLOCK + s * SLAB_BYTES, &tmap_r, &res_full[wg], ocol0 + s * SLAB_COLS, orow0 + 64 * mi);
        }
      }
      wgmma_wait<1>();
      if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty[prev_stage]);
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    // ping-pong: hand the tensor cores to the other warpgroup (if the CTA has a next tile), run this tile's epilogue under
    // its MMAs, and let the ring counters pass its k-blocks
    if (kPingPong) {
      if (tile + gridDim.x < total_tiles) named_barrier_arrive(ORDER_BAR + (wg ^ 1), 256);
      skip_stages(a.k_blocks);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int mi = 0; mi < MI; ++mi) wgmma_fence_regs(acc[mi]);
    if (wg_leader) mbar_arrive(&empty[prev_stage]);

    // ---- epilogue: into the staging slabs, or straight from the accumulator registers to global memory
    if (staged) {
      named_barrier_sync(1 + wg, 128);  // orders the slab writes below after the leader's bulk_wait_group_read
      if (has_res && live_blocks > 0) {
        mbar_wait_nocall(&res_full[wg], res_phase);
        res_phase ^= 1;
      }
    }
    // one pass per 64-row block of the warpgroup; a warp's 16 rows and their statistics are those of a 128-row tile
#pragma unroll
    for (int mi = 0; mi < MI; ++mi) {
      // shared address of this thread's pair (fragment j, row half h) in the slabs of this block
      auto stg_addr = [&](int j, int h) {
        return stg_u32 + mi * STG_BLOCK + h * 8 * 64 + (j >> 2) * SLAB_BYTES + (((j & 3) ^ stg_xor) << 4);
      };
      float (&accm)[BN / 2] = acc[mi];
      long long rows[2];
      int imgs[2];
      bool valid[2];
      row_of<kConv>(a, tc, r_base + 64 * mi, rows[0], imgs[0], valid[0]);
      row_of<kConv>(a, tc, r_base + 64 * mi + 8, rows[1], imgs[1], valid[1]);
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
            const float a0 = accm[8 * p + 2 * h] + ba.x, a1 = accm[8 * p + 2 * h + 1] + ba.y;
            const float g0 = accm[8 * p + 4 + 2 * h] + bg.x, g1 = accm[8 * p + 4 + 2 * h + 1] + bg.y;
            const uint32_t o = pack_bf16x2(a0 * gelu_erf_f(g0), a1 * gelu_erf_f(g1));
            if (staged) st_shared_u32(stg_addr(p, h), o);  // output column 8p + c_base of the tile: fragment p
            else *reinterpret_cast<uint32_t*>(a.out + static_cast<size_t>(rows[h]) * a.ldo + ocol) = o;
          }
        }
      } else {
        const bool has_bias = (kEpi & E_BIAS) && a.bias != nullptr, has_rv = (kEpi & E_ROWVEC) && a.rowvec != nullptr;
        const bool has_stats = (kEpi & E_STATS) && a.stats != nullptr;
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
            float f0 = accm[4 * j + 2 * h] + b2.x, f1 = accm[4 * j + 2 * h + 1] + b2.y;
            if (has_rv) {
              const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.rowvec + static_cast<size_t>(imgs[h]) * a.ld_rowvec + col));
              f0 += v.x; f1 += v.y;
            }
            if (has_act) { f0 = silu_f(f0); f1 = silu_f(f1); }
            if (has_scale) { f0 *= a.out_scale; f1 *= a.out_scale; }
            if (has_res) {  // plain load: the residual may alias the output (in-place add)
              const float2 v = unpack_bf16x2(staged ? ld_shared_u32(stg_addr(j, h))
                                                    : *reinterpret_cast<const uint32_t*>(a.residual + static_cast<size_t>(rows[h]) * a.ld_res + col));
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
            } else if (staged) {
              st_shared_u32(stg_addr(j, h), o);
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
    if (staged) {
      // the slab writes (generic proxy) become visible to the TMA store (async proxy); TMA clips rows >= M, columns >= N
      fence_proxy_async_smem();
      named_barrier_sync(1 + wg, 128);
      if (wg_leader && live_blocks > 0) {
        for (int mi = 0; mi < live_blocks; ++mi)
          for (int s = 0; s < n_slabs; ++s)
            tma_store_2d(&tmap_c, stg + mi * STG_BLOCK + s * SLAB_BYTES, ocol0 + s * SLAB_COLS, orow0 + 64 * mi);
        bulk_commit_group();
      }
    }
  }
  // no bulk store may still be reading the shared memory of an exited CTA
  if (staged && wg_leader) bulk_wait_group<0>();
}

}  // namespace

namespace {

// conv: the grid of output positions per image and the sub-pixel phases of one launch
void conv_out_grid(const GemmDesc& d, int* oh, int* ow, int* phases) {
  *oh = d.conv_kind == 1 ? d.H / 2 : d.H;
  *ow = d.conv_kind == 1 ? d.W / 2 : d.W;
  *phases = d.conv_kind == 3 ? 4 : 1;
}

// conv: the spatial tile BW x BH x BN_img = `rows` output positions on an oh x ow grid, and the tiles per phase.  H, W need
// not be powers of two: the tile may overhang, TMA zero-fills and the epilogue masks
struct ConvTile { int bw, bh, bn_img; long long tiles; };
ConvTile conv_tile(int rows, int n_img, int oh, int ow) {
  ConvTile t;
  t.bw = 16; while (t.bw > ow) t.bw >>= 1;
  t.bh = rows / t.bw; while (t.bh > oh && t.bh > 1) t.bh >>= 1;
  t.bn_img = rows / (t.bw * t.bh);
  t.tiles = static_cast<long long>((ow + t.bw - 1) / t.bw) * ((oh + t.bh - 1) / t.bh) * ((n_img + t.bn_img - 1) / t.bn_img);
  return t;
}

}  // namespace

// A k-block of a rows x bn tile does rows * bn * 64 multiply-adds on (rows + bn) * 128 operand bytes from L2, so the time of
// a tile goes as rows * bn + kOperandWeight * (rows + bn); at 128 rows that is 256 * (bn + 64).  The weight is fitted to
// the per-tile times of tools/conv_tile_sweep.py (DESIGN section 5).
constexpr int kOperandWeight = 128;
constexpr int kMinKBlocks256 = 16;
// Schedule of a plain GEMM: a tile's main loop costs k_blocks * (128 bn + kOperandWeight (128 + bn)) and its epilogue
// kEpilogueWeight * bn in the same units.  Cooperative CTAs run main loop and epilogue in turn; a ping-pong CTA overlaps
// each epilogue with the next tile's main loop, so only the longer of the two counts, plus the last tile's epilogue.
// The weight is fitted to the per-shape times of tools/gemm_schedule_sweep.py (DESIGN section 5).
constexpr int kEpilogueWeight = 3072;

namespace {
bool pingpong_width(int bn, bool geglu) { return bn == 128 || (bn == 64 && !geglu); }
}  // namespace

int gemm_choose_tile(const GemmDesc& d, int sms, int* block_m, int* block_n, int* schedule) {
  D4D_REQUIRE(d.block_m == 0 || d.block_m == 128 || d.block_m == 256, "block_m must be 0 (automatic), 128 or 256");
  D4D_REQUIRE(d.block_m != 256 || d.conv, "256-row tiles: convolutions only (a plain GEMM stages a 128-row tile for its TMA store)");
  D4D_REQUIRE(d.block_m != 256 || d.block_n <= 0 || d.block_n == 128 || d.block_n == 160,
              "256-row tiles run at block_n 128 or 160 (the accumulators of wider tiles do not fit the register file)");
  D4D_REQUIRE(d.schedule == 0 || d.schedule == kSchedCooperative || d.schedule == kSchedPingPong,
              "schedule must be 0 (automatic), 1 (cooperative) or 2 (ping-pong)");
  const bool pp_ok = !d.conv && d.kv_world == 0;
  D4D_REQUIRE(d.schedule != kSchedPingPong || pp_ok, "ping-pong: plain GEMMs without the K/V scatter only");
  D4D_REQUIRE(d.schedule != kSchedPingPong || d.block_n <= 0 || pingpong_width(d.block_n, d.geglu),
              "ping-pong runs at block_n 64 or 128 (GEGLU: 128; wider accumulators do not fit the register file)");
  int oh = 0, ow = 0, phases = 1;
  if (d.conv) conv_out_grid(d, &oh, &ow, &phases);
  D4D_REQUIRE(!d.conv || (d.n_img > 0 && oh > 0 && ow > 0), "empty conv");
  // rows 128 or 256 (convs at widths 128 / 160 with at least one tile per SM and at least kMinKBlocks256 k-blocks per tile:
  // a shorter tile is bound by its register epilogue, and 64 -> 128 channels at 64x64 ran 40% slower at 256 rows), width 64, 128, 160, 192 or 256 (the last N
  // tile may overhang; its extra columns are not stored): the pair with the fewest SM-waves of the persistent grid, weighted
  // by the tile's time, plus the work of the padded columns; ties to the larger tile.  GEGLU keeps to widths whose halves
  // fill whole 32-column store slabs.  The same choice among the ping-pong widths gives that schedule's tile.
  const auto best_tile = [&](bool pingpong, int* bm, int* bn) {
    long long best_cost = -1;
    for (int r : {128, 256}) {
      if (d.block_m > 0 ? r != d.block_m : (r == 256 && !d.conv)) continue;
      if (pingpong && r != 128) continue;
      const int k_blocks = d.conv ? (d.conv_kind >= 2 ? 4 : 9) * ((d.Cin + BLOCK_K - 1) / BLOCK_K) : 0;
      const long long m_tiles = d.conv ? conv_tile(r, d.n_img, oh, ow).tiles * phases : (static_cast<long long>(d.M) + r - 1) / r;
      for (int c : {64, 128, 160, 192, 256}) {
        if (d.block_n > 0) c = d.block_n;
        else if ((d.geglu && c % 64 != 0) || (pingpong && !pingpong_width(c, d.geglu))) continue;
        const long long n_tiles = (d.N + c - 1) / c, tiles = m_tiles * n_tiles;
        const bool fits = r == 128 || ((c == 128 || c == 160) && (d.block_m == 256 || (tiles >= sms && k_blocks >= kMinKBlocks256)));
        if (fits) {
          const long long waves = (tiles + sms - 1) / sms;
          const long long cost = waves * (static_cast<long long>(r) * c + kOperandWeight * (r + c)) + (n_tiles * c - d.N) * (r / 2);
          if (best_cost < 0 || cost <= best_cost) { best_cost = cost; *bm = r; *bn = c; }
        }
        if (d.block_n > 0) break;
      }
    }
    return best_cost >= 0;
  };
  // the time of the tiles an SM runs on either schedule (gemm_choose_tile's header comment), ping-pong strictly faster
  const auto plain_time = [&](bool pingpong, int bn) {
    const long long k_blocks = (d.K1 + BLOCK_K - 1) / BLOCK_K + (d.A2 ? (d.K2 + BLOCK_K - 1) / BLOCK_K : 0);
    const long long tiles = ((static_cast<long long>(d.M) + BLOCK_M - 1) / BLOCK_M) * ((d.N + bn - 1) / bn);
    const long long per_sm = (tiles + sms - 1) / sms;
    const long long main = k_blocks * (static_cast<long long>(BLOCK_M) * bn + kOperandWeight * (BLOCK_M + bn));
    const long long epi = static_cast<long long>(kEpilogueWeight) * bn;
    return pingpong ? per_sm * std::max(main, epi) + std::min(main, epi) : per_sm * (main + epi);
  };
  int sched = d.schedule;
  if (sched == 0) {
    int pbm = 0, pbn = 0, cbm = 0, cbn = 0;
    // an overhanging last N tile costs ping-pong more than the overlap saves (N = 320 at width 128, DESIGN section 5)
    const bool pp_fits = pp_ok && (d.block_n <= 0 || pingpong_width(d.block_n, d.geglu)) && best_tile(true, &pbm, &pbn) &&
                         d.N % pbn == 0;
    D4D_REQUIRE(best_tile(false, &cbm, &cbn), "no tile for this block_m / block_n");
    sched = pp_fits && plain_time(true, pbn) < plain_time(false, cbn) ? kSchedPingPong : kSchedCooperative;
  }
  D4D_REQUIRE(best_tile(sched == kSchedPingPong, block_m, block_n), "no tile for this block_m / block_n");
  if (schedule) *schedule = sched;
  return 0;
}

bool gemm_stats_fusable(const GemmDesc& d, int sms, const char** why) {
  const auto refuse = [&](const char* msg) {
    if (why) *why = msg;
    return false;
  };
  if (d.geglu || d.kv_world != 0) return refuse("GroupNorm statistics: plain / conv epilogue only");
  if (!d.conv) {
    if (d.stats_rows <= 0 || d.stats_rows % 32 != 0) return refuse("statistics need rows-per-image % 32 == 0");
    // rows past the last whole image would add into image M / stats_rows, past the [M / stats_rows][N][2] workspace
    if (d.M % d.stats_rows != 0) return refuse("statistics need M % rows-per-image == 0");
    return true;
  }
  int bm = 0, bn = 0, oh = 0, ow = 0, phases = 1;
  if (gemm_choose_tile(d, sms, &bm, &bn)) return refuse("no tile for this block_m / block_n");
  conv_out_grid(d, &oh, &ow, &phases);
  const ConvTile t = conv_tile(bm, d.n_img, oh, ow);
  if ((t.bw * t.bh) % 32 != 0) return refuse("statistics need 32-row warps inside one image");
  return true;
}

int gemm_prepare(const GemmDesc& d, GemmLaunch* L) {
  D4D_REQUIRE(d.N % 16 == 0, "GEMM N must be a multiple of 16");
  D4D_REQUIRE(d.out != nullptr && d.A != nullptr && d.Wt != nullptr, "null operand");
  // K/V scatter: every rank's buffer exists, and local row m of CFG half m / rows_local lands inside that half's
  // [rows_global] rows of the gathered buffer (the kernel writes without bounds checks)
  D4D_REQUIRE(d.kv_world >= 0 && d.kv_world <= 8, "K/V scatter: world must be in [1, 8]");
  if (d.kv_world > 0) {
    D4D_REQUIRE(!d.conv && !d.geglu && d.kv_col0 >= 0 && d.kv_col0 < d.N && d.kv_col0 % 16 == 0 && d.kv_ld % 8 == 0 &&
                d.kv_ld >= d.N - d.kv_col0, "K/V scatter arguments");
    for (int r = 0; r < d.kv_world; ++r) D4D_REQUIRE(d.kv_dst[r] != nullptr, "K/V scatter: null destination buffer");
    D4D_REQUIRE(d.kv_rows_local > 0 && d.M % d.kv_rows_local == 0, "K/V scatter: M must be a multiple of rows_local");
    D4D_REQUIRE(d.kv_row_offset >= 0 && d.kv_row_offset + d.kv_rows_local <= d.kv_rows_global,
                "K/V scatter: row_offset + rows_local exceeds rows_global");
  }
  GemmKernelArgs& a = L->args;
  memset(&a, 0, sizeof(a));
  int dev = 0, sms = 0;
  D4D_CUDA_OK(cudaGetDevice(&dev));
  D4D_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  D4D_REQUIRE(d.block_n <= 0 || (d.block_n >= 16 && d.block_n <= 256 && d.block_n % 16 == 0 && d.N % d.block_n == 0),
              "no valid block_n");
  D4D_REQUIRE(!d.conv || (d.conv_kind >= 0 && d.conv_kind <= 3), "conv_kind");
  int bm = 0, bn = 0, sched = 0;
  if (int rc = gemm_choose_tile(d, sms, &bm, &bn, &sched)) return rc;
  a.block_m = bm;
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
  const char* no_stats = nullptr;
  D4D_REQUIRE(d.stats == nullptr || gemm_stats_fusable(d, sms, &no_stats), no_stats);
  a.kv_world = d.kv_world;
  a.kv_col0 = d.kv_col0;
  a.kv_ld = d.kv_ld;
  a.kv_rows_local = d.kv_rows_local > 0 ? d.kv_rows_local : 1;
  a.kv_rows_global = d.kv_rows_global;
  a.kv_row_offset = d.kv_row_offset;
  for (int i = 0; i < 8; ++i) a.kv_dst[i] = d.kv_dst[i];
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
    // staged epilogue unless the K/V scatter writes elsewhere, a tile's columns do not fill whole slabs (narrow block_n:
    // a slab would store into the next tile's columns) or an operand is not 16-byte aligned for TMA
    const auto aligned16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    a.staged = d.kv_world == 0 && (d.geglu ? bn % (2 * SLAB_COLS) : bn % SLAB_COLS) == 0 && aligned16(d.out) &&
               (d.residual == nullptr || aligned16(d.residual));
    // ping-pong stages its epilogue; an automatic launch that cannot runs cooperatively from registers
    D4D_REQUIRE(d.schedule != kSchedPingPong || a.staged, "ping-pong needs the staged epilogue (16-byte aligned out / residual)");
    a.pingpong = a.staged && sched == kSchedPingPong;
    L->tmap_c = L->tmap_r = L->tmap_a;
    if (a.staged) {
      if (int rc = make_tmap_2d(&L->tmap_c, d.out, d.M, d.geglu ? d.N / 2 : d.N, d.ldo, SLAB_COLS, 64, 64)) return rc;
      if (d.residual && !d.geglu)
        if (int rc = make_tmap_2d(&L->tmap_r, d.residual, d.M, d.N, d.ld_res, SLAB_COLS, 64, 64)) return rc;
    }
  } else {
    D4D_REQUIRE(d.Cin % 8 == 0, "conv Cin must be a multiple of 8");
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
    // spatial tile: BW x BH x BN = block_m output positions, one 4-D TMA box
    const ConvTile ct = conv_tile(bm, d.n_img, a.H, a.W);
    const int bw = ct.bw, bh = ct.bh, bnimg = ct.bn_img;
    D4D_REQUIRE(bw * bh * bnimg == bm && bnimg <= 256, "conv tile shape");
    a.BW = bw; a.BH = bh; a.BN = bnimg;
    a.tiles_x = (a.W + bw - 1) / bw;
    a.tiles_y = (a.H + bh - 1) / bh;
    a.tiles_per_phase = static_cast<int>(ct.tiles);
    a.m_tiles = a.tiles_per_phase * a.n_phases;
    a.M *= a.n_phases;  // output positions of the launch (FLOP count)
    if (int rc = make_tmap_nhwc(&L->tmap_a, d.A, d.n_img, d.H, d.W, d.Cin, BLOCK_K, bw, bh, bnimg, 128, a.in_stride)) return rc;
    L->tmap_a2 = L->tmap_c = L->tmap_r = L->tmap_a;
    const uint64_t kw = static_cast<uint64_t>(a.n_taps) * d.Cin;
    if (int rc = make_tmap_2d(&L->tmap_b, d.Wt, static_cast<uint64_t>(d.N) * a.n_phases, kw, kw, BLOCK_K, bn, 128)) return rc;
  }
  const int total = a.m_tiles * a.n_tiles;
  L->grid = total < sms ? total : sms;
  return 0;
}

namespace {

using GemmKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                              const CUtensorMap, const GemmKernelArgs);
struct GemmVariant {
  int bn, bm;
  bool geglu, conv;
  int epi;
  bool pingpong;
  GemmKernelFn fn;
  int smem;
};
#define D4D_GV_M(BN, MI, G, C, E) \
  {BN, 128 * MI, G, C, E, false, gemm_wgmma_kernel<BN, MI, G, C, E, false>, GemmCfg<BN, MI, gemm_staged(C, E), false>::SMEM}
#define D4D_GV(BN, G, C, E) D4D_GV_M(BN, 1, G, C, E)
#define D4D_GV_PP(BN, G, E) \
  {BN, 128, G, false, E, true, gemm_wgmma_kernel<BN, 2, G, false, E, true>, GemmCfg<BN, 2, true, true>::SMEM}
#define D4D_GV_PLAIN(BN, GV)                                                                                          \
  /* plain GEMM: qkv | proj_in, shortcut | attn out, ff2 | proj_out, conv_in */                                       \
  GV(BN, false, 0), GV(BN, false, E_BIAS), GV(BN, false, E_BIAS | E_RES), GV(BN, false, E_BIAS | E_RES | E_STATS),     \
  GV(BN, false, GV##_ALL)
#define D4D_GV_COOP_ALL E_ALL
#define D4D_GV_PP_ALL E_STAGED_ALL
#define D4D_GV_COOP(BN, G, E) D4D_GV(BN, G, false, E)
#define D4D_GV_CONV(BN, MI)                                                                                           \
  /* 3x3 convs: resnet conv1 | conv2 | down / up sampling */                                                          \
  D4D_GV_M(BN, MI, false, true, E_BIAS | E_ROWVEC | E_STATS), D4D_GV_M(BN, MI, false, true, E_BIAS | E_RES | E_STATS), \
  D4D_GV_M(BN, MI, false, true, E_BIAS | E_STATS), D4D_GV_M(BN, MI, false, true, E_ALL)
// the feature sets the UNet plan launches (csrc/unet.cu) at the tile widths it picks, plus E_ALL kernels for the rest.
// GEGLU (only the bias bit matters) runs at widths whose output halves fill whole store slabs; no conv picks 192.
// 256-row conv tiles (MI = 2) exist where 2 * BN / 2 accumulators per thread fit the 232 registers: widths 128 and 160.
// Ping-pong kernels (MI = 2 as well) exist at width 128, plain and GEGLU, and at 64 for the all-features set (all but the
// K/V scatter: ping-pong stages its epilogue).  At 160 the staged epilogue of two 64-row blocks spills.
const GemmVariant kGemmVariants[] = {
    D4D_GV_PLAIN(128, D4D_GV_COOP), D4D_GV_CONV(128, 1), D4D_GV_CONV(128, 2), D4D_GV(128, true, false, E_BIAS),
    D4D_GV_PLAIN(160, D4D_GV_COOP), D4D_GV_CONV(160, 1), D4D_GV_CONV(160, 2),
    D4D_GV_PLAIN(192, D4D_GV_COOP),
    D4D_GV_PLAIN(256, D4D_GV_COOP), D4D_GV_CONV(256, 1), D4D_GV(256, true, false, E_BIAS),
    D4D_GV(64, false, false, E_ALL), D4D_GV(64, false, true, E_ALL), D4D_GV(64, true, false, E_BIAS),
    D4D_GV_PLAIN(128, D4D_GV_PP), D4D_GV_PP(128, true, E_BIAS), D4D_GV_PP(64, false, E_STAGED_ALL),
};
#undef D4D_GV_COOP
#undef D4D_GV_COOP_ALL
#undef D4D_GV_PP_ALL
#undef D4D_GV_CONV
#undef D4D_GV_PLAIN
#undef D4D_GV_PP
#undef D4D_GV
#undef D4D_GV_M
constexpr int kNumGemmVariants = sizeof(kGemmVariants) / sizeof(kGemmVariants[0]);

// the instantiation of kernel width bn (and the launch's tile rows) whose feature bits equal the launch's, else the E_ALL one (-1: none)
int gemm_variant_at(const GemmKernelArgs& a, int bn) {
  const bool conv = a.mode != 0, geglu = a.geglu != 0;
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
    if (v.bn != bn || v.bm != a.block_m || v.geglu != geglu || v.conv != conv || v.pingpong != (a.pingpong != 0)) continue;
    if (v.epi == need) return i;
    if ((v.epi & need) == need && (generic < 0 || v.epi == E_ALL)) generic = i;  // geglu: E_BIAS covers {} as well
  }
  return generic;
}

// The instantiation that runs a launch: the narrowest kernel width >= block_n that has the launch's feature set (a narrower
// block_n runs on a wider kernel with the extra columns masked).
int gemm_variant_of(const GemmKernelArgs& a) {
  for (int bn : {64, 128, 160, 192, 256}) {
    if (bn < a.block_n) continue;
    const int vi = gemm_variant_at(a, bn);
    if (vi >= 0) return vi;
  }
  return -1;
}

}  // namespace

int gemm_run(const GemmLaunch& L, cudaStream_t stream) {
  static PerDeviceOnce attr_once[kNumGemmVariants];
  const int vi = gemm_variant_of(L.args);
  D4D_REQUIRE(vi >= 0, "no GEMM kernel instantiation covers this launch");
  const GemmVariant& v = kGemmVariants[vi];
  if (int rc = ensure_dyn_smem(v.fn, v.smem, attr_once[vi])) return rc;
  D4D_CUDA_OK(launch_pdl(v.fn, dim3(L.grid), dim3(NUM_THREADS), v.smem, stream, L.tmap_a, L.tmap_a2, L.tmap_b, L.tmap_c, L.tmap_r,
                         L.args));
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

double gemm_flops(const GemmLaunch& L) {
  return 2.0 * static_cast<double>(L.args.M) * L.args.N * (static_cast<double>(L.args.k_blocks) * BLOCK_K);
}

}  // namespace d4d
