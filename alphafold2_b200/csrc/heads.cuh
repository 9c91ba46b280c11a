// Angle heads of Alphafold2(predict_angles=True) (alphafold2.py:559-562, 813-836) in one pass over the fp32 trunk output
// x [B][n][n][d], token-major:
//
//   theta[b,i,j] = W_t x[b,i,j] + b_t        phi[b,i,j] = W_p x[b,i,j] + b_p
//   omega[b,i,j] = W_o s + b_o,   s = (x[b,i,j] + x[b,j,i]) * 0.5  (SYM, in the reference's order)   or   s = x[b,i,j]
//
// Work item: an unordered pair of 8 x 8 token tiles {(I, J), (J, I)}, I <= J (a diagonal tile alone).  One producer thread
// TMA-loads both tiles chunk by chunk (32 channels, fp32, 8 KB per tile) through an mbarrier ring, so every element of x
// crosses HBM once, with or without SYM.  Per chunk the MMA warpgroup splits each tile into three bf16 planes in shared
// memory (p0 = bf16(v), p1 = bf16(v - p0), p2 = bf16(v - p0 - p1): strict mode's encoding, ops.split_weight) and runs the six
// plane-pair passes (0,2) (2,0) (1,1) (0,1) (1,0) (0,0) against the weight planes, smallest first, on `wgmma`:
//   tile (I, J) and tile (J, I): m64n64 over all 64 output columns [theta | phi | omega | 0] (a diagonal tile runs both on the
//   same data and stores one: a branch between the wgmmas makes ptxas wait for each one before issuing the next);
//   SYM: s of tile (I, J) is formed in fp32 from both tiles, and the 32 weight rows from omega_row0 (which hold omega's rows,
//   inside the 64-row block) run on it (m64n32).
//   omega is then stored at (i, j) and (j, i) from the same value, so it is bitwise symmetric.
// Row variant (ROWS, one batch element): the output rows are a shard [row0, row0 + rows) of the pair rows.  Work item: (row
// tile I of the shard, column tile J), every J; tile (I, J) comes from the shard's rows x_rows [rows][n][d] and, with SYM, the
// transposed tile from the shard's columns x_cols [n][rows][d] (x_cols[j][i - row0] = x[j][i]) through the second tensor map,
// loaded exactly like the whole kernel's tile (J, I).  Only tile (I, J) is stored (omega at (i, j) alone): every value is
// formed from the same operands in the same order as the whole kernel's value at (row0 + i, j), so the shard is bitwise its
// rows.  Row tiles start at the shard's first row, whatever row0 is.
// Each chunk accumulates into a fresh fp32 register accumulator that is then added (IEEE, round to nearest) to the item's
// running sum, so the tensor cores' accumulation only ever sums 32 channels; bias last.  The next chunk is split into the
// second plane buffer while the tensor cores run the current one.
#pragma once
#include "common.cuh"

namespace af2 {

constexpr int AH_TILE = 8;                     // tokens per side of a square tile: 64 pair tokens = the m64 rows of a wgmma
constexpr int AH_KC = 32;                      // channels per chunk
constexpr int AH_BOX = 64 * AH_KC * 4;         // one tile's chunk in fp32 (TMA box [1][8][8][32]): 8 KB
constexpr int AH_PLANE = 64 * AH_KC * 2;       // one bf16 plane of 64 rows x 32 channels, 64-byte swizzled rows: 4 KB
constexpr int AH_THREADS = 160;                // warps 0-3: the MMA warpgroup; warp 4: the TMA producer
constexpr int AH_COLS = 64;                    // output columns of the tile: theta | phi | omega | zero rows
constexpr int AH_SMEM_MAX = 232448;

struct AngleHeadsParams {
  const uint4* wplanes;   // bf16 [d / 32][3][64][32]: the split planes of the concatenated weight, rows theta | phi | omega | 0
  const float* bias;      // [64], zero beyond the buckets
  float* theta;           // [B][n][n][nt]
  float* phi;             // [B][n][n][np]
  float* omega;           // [B][n][n][no]
  int B, n, d;
  int rows;               // output rows per batch element: n, or the shard's rows (ROWS)
  int nt, np, no;
  int omega_row0;         // SYM: first weight row of the 32-row window that holds omega's rows (a multiple of 8, <= 32)
  int tiles;              // ceil(n / 8)
  long long items;        // B * tiles * (tiles + 1) / 2;  ROWS: ceil(rows / 8) * tiles
  int stages;             // TMA ring depth
};

template <bool SYM>
struct AngleHeadsSmem {
  static constexpr int TILES = SYM ? 3 : 2;                          // planes per chunk: tile (I, J), tile (J, I), s
  static constexpr int PLANES_BYTES = 2 * TILES * 3 * AH_PLANE;      // two buffers
  __host__ __device__ static int weights_bytes(int d) { return d / AH_KC * 3 * AH_PLANE; }
  __host__ __device__ static int ring_off(int d) { return weights_bytes(d) + PLANES_BYTES; }
  static int stages(int d) {
    const int s = (AH_SMEM_MAX - ring_off(d) - 256) / (2 * AH_BOX);
    return s > 6 ? 6 : s;
  }
  static int total(int d, int stages) { return ring_off(d) + stages * 2 * AH_BOX + 256; }
};

// byte offset of 16-byte chunk `chunk` (0..3) of row `row` in a 64B-swizzled tile whose rows are 64 bytes (wgmma SWZ_64)
__device__ __forceinline__ uint32_t swz64_off(uint32_t row, uint32_t chunk) {
  return row * 64u + ((chunk ^ ((row >> 1) & 3u)) << 4);
}

// item -> (b, I, J), items of a batch element in row-major order over I <= J
__device__ __forceinline__ void ah_item(long long item, int tiles, int& b, int& I, int& J) {
  const long long per = static_cast<long long>(tiles) * (tiles + 1) / 2;
  b = static_cast<int>(item / per);
  const long long q = item - static_cast<long long>(b) * per;
  auto off = [&](long long r) { return r * tiles - r * (r - 1) / 2; };      // first item of row r
  const double t2 = 2.0 * tiles + 1.0;
  long long r = static_cast<long long>((t2 - sqrt(t2 * t2 - 8.0 * static_cast<double>(q))) * 0.5);
  if (r < 0) r = 0;
  while (r > 0 && off(r) > q) --r;
  while (r + 1 < tiles && off(r + 1) <= q) ++r;
  I = static_cast<int>(r);
  J = static_cast<int>(r + (q - off(r)));
}

// the three split planes of 4 consecutive channels (4 q .. 4 q + 3) of row t, 8 bytes per plane
__device__ __forceinline__ void ah_split_store(uint8_t* planes, int t, int q, float4 v) {
  const uint32_t off = swz64_off(t, q >> 1) + (q & 1) * 8;
  float r0 = v.x, r1 = v.y, r2 = v.z, r3 = v.w;
#pragma unroll
  for (int pl = 0; pl < 3; ++pl) {
    const uint32_t lo = pack_bf16x2(r0, r1), hi = pack_bf16x2(r2, r3);
    *reinterpret_cast<uint2*>(planes + pl * AH_PLANE + off) = make_uint2(lo, hi);
    r0 -= bf16lo_to_f32(lo);
    r1 -= bf16hi_to_f32(lo);
    r2 -= bf16lo_to_f32(hi);
    r3 -= bf16hi_to_f32(hi);
  }
}

template <int R>
__device__ __forceinline__ void ah_accumulate(float (&tot)[R], const float (&acc)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) tot[i] += acc[i];
}

// item -> (b, I, J) of either variant; diag: a diagonal tile of the whole kernel (one tile, stored once)
template <bool ROWS>
__device__ __forceinline__ void ah_decode(long long it, int tiles, int& b, int& I, int& J, bool& diag) {
  if constexpr (ROWS) {
    b = 0;
    I = static_cast<int>(it / tiles);
    J = static_cast<int>(it - static_cast<long long>(I) * tiles);
    diag = false;
  } else {
    ah_item(it, tiles, b, I, J);
    diag = I == J;
  }
}

// tmX: x [B][n][n][d] (ROWS: x_rows [1][rows][n][d]); tmC: the tensor the transposed tile comes from, x itself (ROWS:
// x_cols [1][n][rows][d])
template <bool SYM, bool ROWS>
__global__ void __launch_bounds__(AH_THREADS, 1)
angle_heads_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmC,
                   const __grid_constant__ AngleHeadsParams p) {
  using L = AngleHeadsSmem<SYM>;
  constexpr int NT = L::TILES;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const int nk = p.d / AH_KC;
  uint8_t* wsm = smem;
  uint8_t* planes = smem + L::weights_bytes(p.d);
  uint8_t* ring = smem + L::ring_off(p.d);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + p.stages * 2 * AH_BOX);
  uint64_t* empty_bar = full_bar + p.stages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmC);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      int slot = 0;
      uint32_t phase = 0;
      for (long long it = blockIdx.x; it < p.items; it += gridDim.x) {
        int b, I, J;
        bool diag;
        ah_decode<ROWS>(it, p.tiles, b, I, J, diag);
        const bool two = ROWS ? SYM : !diag;                  // the transposed tile is loaded
        for (int kc = 0; kc < nk; ++kc) {
          mbar_wait(&empty_bar[slot], phase ^ 1);
          uint8_t* dst = ring + slot * 2 * AH_BOX;
          mbar_arrive_expect_tx(&full_bar[slot], two ? 2 * AH_BOX : AH_BOX);
          // box [1][8 i][8 j][32 c] at (c, j, i, b): rows of the box are tokens t = 8 (i - i0) + (j - j0); out-of-range i / j
          // are zero-filled and never stored
          tma_load_4d(dst, &tmX, &full_bar[slot], kc * AH_KC, J * AH_TILE, I * AH_TILE, b);
          if (two) tma_load_4d(dst + AH_BOX, &tmC, &full_bar[slot], kc * AH_KC, I * AH_TILE, J * AH_TILE, b);
          if (++slot == p.stages) { slot = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ============================ MMA warpgroup (threads 0-127) ============================
  const int tid = threadIdx.x;
  // weight planes -> shared memory, 64B-swizzled: block (kc, plane) = 64 rows x 32 channels
  for (int c = tid; c < nk * 3 * 64 * 4; c += 128) {
    const int blk = c >> 8, r = (c >> 2) & 63, ch = c & 3;
    *reinterpret_cast<uint4*>(wsm + blk * AH_PLANE + swz64_off(r, ch)) = __ldg(p.wplanes + c);
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 128);

  const uint32_t wsm_u = smem_u32(wsm);
  auto desc = [](uint32_t addr) { return wgmma_desc(addr, 16, 512, SWZ_64); };
  const int q = tid & 7;          // split: channel quad
  const int t0 = tid >> 3;        // split: tokens t0 + 16 u
  const int wq = tid >> 5;
  const int r_lo = wq * 16 + (lane >> 2);
  const int q2 = 2 * (lane & 3);
  const int o0 = p.nt + p.np;     // first omega column

  int slot = 0;
  uint32_t phase = 0;
  float accA[32], accC[32], accS[SYM ? 16 : 1];
  float totA[32], totC[32], totS[SYM ? 16 : 1];

  for (long long it = blockIdx.x; it < p.items; it += gridDim.x) {
    int b, I, J;
    bool diag;
    ah_decode<ROWS>(it, p.tiles, b, I, J, diag);
    const bool two = ROWS ? SYM : !diag;
#pragma unroll
    for (int i = 0; i < 32; ++i) totA[i] = totC[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (SYM ? 16 : 1); ++i) totS[i] = 0.f;

    for (int kc = 0; kc < nk; ++kc) {
      mbar_wait(&full_bar[slot], phase);
      const uint8_t* xa = ring + slot * 2 * AH_BOX;
      const uint8_t* xc = two ? xa + AH_BOX : xa;
      uint8_t* pl = planes + (kc & 1) * (NT * 3 * AH_PLANE);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int t = t0 + 16 * u;
        const float4 a = *reinterpret_cast<const float4*>(xa + t * 128 + q * 16);
        ah_split_store(pl, t, q, a);
        if constexpr (!ROWS) ah_split_store(pl + 3 * AH_PLANE, t, q, *reinterpret_cast<const float4*>(xc + t * 128 + q * 16));
        if constexpr (SYM) {
          // s at token t = (ii, jj) of tile (I, J) pairs with token (jj, ii) of tile (J, I)
          const int tt = (t & 7) * 8 + (t >> 3);
          const float4 c = *reinterpret_cast<const float4*>(xc + tt * 128 + q * 16);
          const float4 s = make_float4((a.x + c.x) * 0.5f, (a.y + c.y) * 0.5f, (a.z + c.z) * 0.5f, (a.w + c.w) * 0.5f);
          ah_split_store(pl + 6 * AH_PLANE, t, q, s);
        }
      }
      fence_proxy_async_smem();
      if (kc > 0) {                     // the previous chunk's passes ran while this chunk was split
        wgmma_wait<0>();
        reg_fence(accA);
        reg_fence(accS);
        ah_accumulate(totA, accA);
        if constexpr (!ROWS) {
          reg_fence(accC);
          ah_accumulate(totC, accC);
        }
        if constexpr (SYM) ah_accumulate(totS, accS);
      }
      // every warp has split this chunk and waited for the previous chunk's passes: the next chunk may rewrite their plane
      // buffer, and the ring slot is free
      named_bar_sync(1, 128);
      if (tid == 0) mbar_arrive(&empty_bar[slot]);
      if (++slot == p.stages) { slot = 0; phase ^= 1; }
      wgmma_fence();
      const uint32_t pa_u = smem_u32(pl);
      const uint32_t wb = wsm_u + kc * 3 * AH_PLANE;
      constexpr int PA[6] = {0, 2, 1, 0, 1, 0};
      constexpr int PB[6] = {2, 0, 1, 1, 0, 0};
#pragma unroll
      for (int ps = 0; ps < 6; ++ps) {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          const uint32_t scale_d = (ps | ks) != 0 ? 1u : 0u;
          const uint64_t bdesc = desc(wb + PB[ps] * AH_PLANE + ks * 32);
          wgmma_m64n64k16_ss<0, 0>(accA, desc(pa_u + PA[ps] * AH_PLANE + ks * 32), bdesc, scale_d);
          if constexpr (!ROWS) wgmma_m64n64k16_ss<0, 0>(accC, desc(pa_u + (3 + PA[ps]) * AH_PLANE + ks * 32), bdesc, scale_d);
          if constexpr (SYM)
            wgmma_m64n32k16_ss<0, 0>(accS, desc(pa_u + (6 + PA[ps]) * AH_PLANE + ks * 32),
                                     desc(wb + PB[ps] * AH_PLANE + p.omega_row0 * 64 + ks * 32), scale_d);
        }
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    reg_fence(accA);
    reg_fence(accS);
    ah_accumulate(totA, accA);
    if constexpr (!ROWS) {
      reg_fence(accC);
      ah_accumulate(totC, accC);
    }
    if constexpr (SYM) ah_accumulate(totS, accS);
    named_bar_sync(1, 128);             // every warp has seen the item's last passes retire before any splits the next item

    // ---- epilogue: + bias, rows r_lo and r_lo + 8 of each tile; columns 8 j + q2 + {0, 1} ----
    const long long bn = static_cast<long long>(b) * p.rows;
    auto store_tile = [&](const float (&tot)[32], int h, int i, int j) {
      if (i >= p.rows || j >= p.n) return;
      const long long tok = (bn + i) * p.n + j;
#pragma unroll
      for (int jx = 0; jx < 8; ++jx) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * jx + q2 + e;
          const float v = tot[4 * jx + 2 * h + e] + __ldg(p.bias + col);
          if (col < p.nt) p.theta[tok * p.nt + col] = v;
          else if (col < o0) p.phi[tok * p.np + (col - p.nt)] = v;
          else if (!SYM && col < o0 + p.no) p.omega[tok * p.no + (col - o0)] = v;
        }
      }
    };
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = r_lo + 8 * h;
      const int ii = m >> 3, jj = m & 7;
      store_tile(totA, h, I * AH_TILE + ii, J * AH_TILE + jj);
      if (!ROWS && !diag) store_tile(totC, h, J * AH_TILE + ii, I * AH_TILE + jj);
      if constexpr (SYM) {
        // omega of s at (i, j) and (j, i); within a diagonal tile each unordered pair once
        const int i = I * AH_TILE + ii, j = J * AH_TILE + jj;
        if (i < p.rows && j < p.n && (!diag || ii <= jj)) {
          const long long t1 = (bn + i) * p.n + j, t2 = (bn + j) * p.n + i;
#pragma unroll
          for (int jx = 0; jx < 4; ++jx) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = p.omega_row0 + 8 * jx + q2 + e;
              if (col >= o0 && col < o0 + p.no) {
                const float v = totS[4 * jx + 2 * h + e] + __ldg(p.bias + col);
                p.omega[t1 * p.no + (col - o0)] = v;
                if constexpr (!ROWS) p.omega[t2 * p.no + (col - o0)] = v;
              }
            }
          }
        }
      }
    }
  }
}

}  // namespace af2
