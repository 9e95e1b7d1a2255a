// mlp_tc.cu -- Hopper tensor-core path of usip_layer_fwd (precision == 1): 3xTF32 error-compensated GEMM
//
//     Y[P,Cout] = act(X)[P,Cin] * W[Cout,Cin]^T (+bias, +addend),     act = folded BN affine + ReLU
//
// with  a = a_hi + a_lo (a_hi = rna_tf32(a), a_lo = rna_tf32(a - a_hi)) and likewise for W:
//     D += a_lo*w_hi + a_hi*w_lo + a_hi*w_hi        (dropped term a_lo*w_lo ~ 2^-22 relative)
// which keeps fp32-level accuracy (the 1e-4 parity bar) at 1/3 of the TF32 tensor rate.
//
// Persistent CTA (one per SM) of two consumer warpgroups and one producer warpgroup.  A CTA keeps one BN-wide column tile and
// walks its row tiles base, base + stride, ...  Each warpgroup accumulates 64-row x BN tiles in registers with
// wgmma.mma_async (m64 x BN x k8): it takes every other 64-row tile of the CTA's sequence, or, with COMBINE (group-128
// max/min), one 64-row half of every 128-row tile.
//   * A comes from registers.  Each consumer warpgroup has its own ring of raw fp32 activation stages ([64 rows x 32
//     floats], SWIZZLE_128B), filled by one producer lane with tensor-map TMA loads in the warpgroup's own (tile, K chunk)
//     order, across tile boundaries: the ring runs ahead through the epilogue, and rows past P arrive as zeros.  A thread
//     reads its fragment's 8 floats of each of its two rows from the stage, applies the folded BN affine + ReLU and
//     splits hi/lo; the stage is released when the chunk's wgmma retired.  Two fragment buffers alternate; a buffer is
//     rewritten only after wgmma.wait_group retired the chunk that read it.
//   * B (the pre-split, pre-swizzled weight tile of one K chunk) streams through one shared-memory ring that both
//     warpgroups read, since they run through the same column tile's chunks.  The producer lane refills a stage with one
//     bulk-TMA copy once both warpgroups arrived on its empty barrier; the full barrier counts the copy's bytes.  When the
//     whole K panel fits in the ring (KC <= stages) it is loaded once and never recycled.
//   * Nothing in the main loop couples the two warpgroups, so one runs its tensor work while the other is in its epilogue.
// Epilogue per warpgroup tile, one 64-column half at a time: accumulators (+addend, +bias) -> the warpgroup's XOR-swizzled
// [64 x 64] fp32 staging tile -> four warps on 32-row x 32-column chunks: coalesced Y stores, BN statistics, per-group
// max/min (+arg).  A lane owns the same <= 2 columns in every tile and keeps their running (sum, sum^2) in registers.
//
// K order inside a 32-float chunk: the wgmma fragment holds k = l%4 and l%4 + 4 of each k-step, so logical position p of
// k-step s reads physical column 8*(p%4) + 2s + p/4.  Thread quad position t then owns physical columns 8t..8t+7 of both of
// its rows (two float4 each), and a quad reads one contiguous 128-byte row segment.  In 16-byte-chunk terms the logical
// column 4c + j holds physical column 8j + c; the weight pack applies the same map, and a dot product ignores K order.
//
// B tiles and A stages are K-major, SWIZZLE_128B: row r (128 B = 32 floats) at r*128, 16-byte chunk c stored at chunk
// (c ^ (r & 7)); 8-row groups 1024 B apart.  One K chunk = 32 floats = 4 wgmma k-steps of 8.
#include "tc_common.cuh"

namespace usip {

constexpr int TC_CONSUMERS = 256;                    // two consumer warpgroups
// + a producer warpgroup (warp 0: weights, warps 1 and 2: activations of consumer warpgroup 0 and 1): with 384 threads a
// thread starts with 168 registers; the producer gives most of its share to the consumers (40 + 2 x 232 per 128 threads),
// whose accumulators and two 3xTF32 A-fragment buffers need about 170
constexpr int TC_THREADS = TC_CONSUMERS + 128;
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;
constexpr int TC_EPI_COLS = 64;                      // columns of the epilogue staging tile

// ------------------------------------------------------------------------------------------------
// weight pre-pack: W[Cout,Cin] (row stride ldw) -> per (n_tile, k_chunk) one contiguous, pre-swizzled block
// [w_hi | w_lo] (TF32, BN x 128 B each, SWIZZLE_128B), K permuted as in the header, so a stage's B operand is a single
// bulk copy.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tc_pack_one(const float* __restrict__ W, int ldw, int transposed, int Cout, int Cin, int BN,
                                            uint32_t* __restrict__ out, int t) {
  const int KC = Cin / TC_BK;
  const int total = Cout * (Cin / 4);                 // one thread per 16-byte chunk of the packed row
  if (t >= total) return;
  const int n = t / (Cin / 4), k4 = t - n * (Cin / 4);
  const int kc = k4 / 8, c = k4 & 7;                  // 16-byte chunk c of K chunk kc
  const int nt = n / BN, r = n - nt * BN;
  float w[4];
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = kc * TC_BK + 8 * j + c;             // logical column 4c + j <- physical column 8j + c
    w[j] = transposed ? W[(size_t)k * ldw + n] : W[(size_t)n * ldw + k];
    split_tf32(w[j], hi[j], lo[j]);
  }
  const size_t blk = ((size_t)nt * KC + kc) * 2 * (size_t)BN * TC_BK;     // in 32-bit words
  const size_t off = (size_t)r * TC_BK + (size_t)((c ^ (r & 7)) * 4);
  *reinterpret_cast<uint4*>(out + blk + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(out + blk + (size_t)BN * TC_BK + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

__global__ void tc_pack_weights_kernel(const float* __restrict__ W, int ldw, int transposed, int Cout, int Cin, int BN,
                                       uint32_t* __restrict__ out) {
  tc_pack_one(W, ldw, transposed, Cout, Cin, BN, out, blockIdx.x * blockDim.x + threadIdx.x);
}

// Many layers in ONE launch (the train step re-packs all 26 weight matrices after every Adam update): the block index is
// mapped to (layer, block of that layer) through a prefix table that travels in the kernel parameters.
constexpr int TC_PACK_MANY = 32;
struct TcPackMany {
  int n;
  int blk0[TC_PACK_MANY + 1];
  const float* W[TC_PACK_MANY];
  uint32_t* out[TC_PACK_MANY];
  int ldw[TC_PACK_MANY], transposed[TC_PACK_MANY], Cout[TC_PACK_MANY], Cin[TC_PACK_MANY], BN[TC_PACK_MANY];
};
__global__ void tc_pack_many_kernel(const __grid_constant__ TcPackMany pm) {
  int i = 0;
  while (i + 1 < pm.n && (int)blockIdx.x >= pm.blk0[i + 1]) ++i;
  tc_pack_one(pm.W[i], pm.ldw[i], pm.transposed[i], pm.Cout[i], pm.Cin[i], pm.BN[i], pm.out[i],
              ((int)blockIdx.x - pm.blk0[i]) * (int)blockDim.x + (int)threadIdx.x);
}


// ------------------------------------------------------------------------------------------------
template <int BN>
struct TcSmem {
  static constexpr int STAGES = BN == 128 ? 4 : 8;               // weight ring: 128 KB of stages
  static constexpr int B_STAGE = 2 * BN * 128;                   // [w_hi | w_lo] of one K chunk
  static constexpr int A_STAGES = 3;                             // activation ring of each consumer warpgroup (what fits)
  static constexpr int A_STAGE = TC_WG_ROWS * TC_BK * 4;         // 64 rows x one K chunk
  static constexpr int TILE = TC_WG_ROWS * TC_EPI_COLS * 4;      // epilogue staging tile of one warpgroup
  static constexpr int COMB = 4 * 4 * BN * 4;                    // max, min, argmax, argmin per 32-row quarter (group > 32)
  static constexpr int BARS = 16 * (STAGES + 2 * A_STAGES);      // full + empty barrier per stage
  static constexpr int BYTES = STAGES * B_STAGE + 2 * A_STAGES * A_STAGE + 2 * TILE + 2 * COMB + BARS + 1024;  // +1024: alignment
};

// SINGLE: plain TF32, hi x hi only (the backward-precision option, usip_layer_desc.debug_flags & 8)
// COMBINE: group-128 max/min; both warpgroups work on the halves of one 128-row tile and combine through shared memory
template <int BN, bool COMBINE, bool SINGLE>
__global__ void __launch_bounds__(TC_THREADS, 1)
layer_fwd_tc_kernel(const usip_layer_desc d, const uint32_t* __restrict__ wpack, const __grid_constant__ CUtensorMap xmap) {
  using SM = TcSmem<BN>;
  constexpr int S = SM::STAGES, SA = SM::A_STAGES;
  constexpr int BK = TC_BK;                          // 32 floats per K chunk
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;       // SWIZZLE_128B needs 1024-B alignment
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  // [B ring | A ring of warpgroup 0 | of warpgroup 1 | 2 staging tiles | 2 comb areas | barriers]
  const uint32_t a_base = S * SM::B_STAGE;           // byte offsets from smem_base
  const uint32_t tile_base = a_base + 2 * SA * SM::A_STAGE;
  const uint32_t comb_base = tile_base + 2 * SM::TILE;
  const uint32_t bar_base = smem_base + comb_base + 2 * SM::COMB;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };
  auto a_stage = [&](int w, int s) { return a_base + (uint32_t)(w * SA + s) * SM::A_STAGE; };
  auto a_full_bar = [&](int w, int s) { return bar_base + 8u * (2 * S + w * SA + s); };
  auto a_empty_bar = [&](int w, int s) { return bar_base + 8u * (2 * S + 2 * SA + w * SA + s); };

  // warp index via a shuffle: the compiler then knows the role branches are warp-uniform (a branch it cannot prove uniform
  // makes it serialise the wgmma)
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int P = d.P, Cout = d.Cout;
  const int KC = d.Cin / BK;
  const bool ring = KC > S;                          // else the K panel is loaded once and stays resident
  const int n_tiles = Cout / BN;
  const int base = blockIdx.x / n_tiles, stride = gridDim.x / n_tiles;     // the grid is a multiple of n_tiles
  const int nt = blockIdx.x - base * n_tiles, n0 = nt * BN;
  // row tiles of this CTA: base, base + stride, ... (128-row tiles with COMBINE, else 64-row tiles)
  const int cta_tiles = cdiv(cdiv(P, COMBINE ? TC_BM : TC_WG_ROWS) - base, stride);
  // tiles of consumer warpgroup w, and the first row of its jt-th tile
  auto wg_tiles = [&](int w) { return COMBINE ? cta_tiles : (cta_tiles + 1 - w) / 2; };
  auto tile_row0 = [&](int w, int jt) {
    return COMBINE ? (base + jt * stride) * TC_BM + TC_WG_ROWS * w : (base + (2 * jt + w) * stride) * TC_WG_ROWS;
  };

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);                    // one arrival per warpgroup
    }
    for (int w = 0; w < 2; ++w)
      for (int s = 0; s < SA; ++s) {
        mbar_init(a_full_bar(w, s), 1);
        mbar_init(a_empty_bar(w, s), 1);             // the consumer warpgroup, once the chunk's wgmma retired
      }
    fence_barrier_init();
  }
  __syncthreads();

  // ================= producer warpgroup
  if (warp >= TC_CONSUMERS / 32) {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    const int pw = warp - TC_CONSUMERS / 32;
    if (pw > 0 && pw <= 2 && lane == 0) {
      // activations of consumer warpgroup w: its tiles' K chunks in the order it consumes them, so the ring runs ahead
      // across tile boundaries (through the warpgroup's epilogue)
      const int w = pw - 1, tiles = wg_tiles(w);
      prefetch_tensor_map(&xmap);
      for (int jt = 0, it = 0; jt < tiles; ++jt) {
        const int row0 = tile_row0(w, jt);
        for (int kc = 0; kc < KC; ++kc, ++it) {
          const int s = it % SA;
          if (it >= SA) mbar_wait_sleep(a_empty_bar(w, s), ((it / SA) & 1) ^ 1);
          mbar_arrive_expect_tx(a_full_bar(w, s), SM::A_STAGE);
          tma_load_2d(smem_base + a_stage(w, s), &xmap, kc * BK, row0, a_full_bar(w, s));
        }
      }
    }
    // weights: one lane streams the column tile's K chunks through the ring, round after round (a round = one tile of
    // each warpgroup; both read the same chunks).  In a round that only warpgroup 0 has a tile for, the producer arrives
    // in warpgroup 1's place, after the stage's previous phase completed.
    if (pw == 0 && lane == 0) {
      const int rounds = COMBINE ? cta_tiles : (cta_tiles + 1) / 2;
      const int both = COMBINE ? cta_tiles : cta_tiles / 2;
      const uint32_t* src = wpack + (size_t)nt * KC * 2 * BN * BK;
      const int chunks = ring ? rounds * KC : KC;
      for (int it = 0; it < chunks; ++it) {
        const int s = it % S, kc = it % KC;
        if (it >= S) mbar_wait_sleep(empty_bar(s), ((it / S) & 1) ^ 1);
        mbar_arrive_expect_tx(full_bar(s), SM::B_STAGE);
        bulk_g2s(smem_base + s * SM::B_STAGE, src + (size_t)kc * 2 * BN * BK, SM::B_STAGE, full_bar(s));
        if (ring && it / KC >= both) mbar_arrive(empty_bar(s));
      }
    }
    return;
  }

  // ================= consumer warpgroup wg
  setmaxnreg_inc<TC_CONSUMER_REGS>();
  const int wg = warp >> 2, wwarp = warp & 3, wtid = tid & 127;
  const int my_tiles = wg_tiles(wg);

  // ---- A fragment: rows ra and ra + 8 of the tile, physical columns kq..kq+7 (16-byte chunks 2t, 2t+1) of each K chunk.
  // In the swizzled stage they lie at chunk slots (2t, 2t+1) ^ (ra & 7) of rows ra and ra + 8 ((ra + 8) & 7 == ra & 7):
  // the 8 lanes of a quarter-warp phase read 8 distinct slots of two rows, without bank conflicts.
  const int ra = 16 * wwarp + (lane >> 2), t4 = lane & 3, kq = 8 * t4;
  const uint32_t a_off0 = ra * 128 + (((2 * t4) ^ (ra & 7)) << 4), a_off1 = ra * 128 + (((2 * t4 + 1) ^ (ra & 7)) << 4);
  const bool has_aff = d.in_scale != nullptr;
  const float relu_floor = d.in_relu ? 0.f : -INFINITY;
  float4 sc[2] = {make_float4(1.f, 1.f, 1.f, 1.f), make_float4(1.f, 1.f, 1.f, 1.f)};
  float4 sh[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  // the folded BN affine of this thread's 8 input channels, loaded one chunk ahead
  auto fetch_affine = [&](int kc) {
    if (has_aff) {
      const int k = kc * BK + kq;
      sc[0] = __ldg(reinterpret_cast<const float4*>(d.in_scale + k)); sc[1] = __ldg(reinterpret_cast<const float4*>(d.in_scale + k + 4));
      sh[0] = __ldg(reinterpret_cast<const float4*>(d.in_shift + k)); sh[1] = __ldg(reinterpret_cast<const float4*>(d.in_shift + k + 4));
    }
  };
  // hi = rna_tf32(v), lo = rna_tf32(v - hi): (bits + 0x1000) & ~0x1fff IS cvt.rna.tf32.f32 for finite inputs (round to
  // nearest, ties away, on the magnitude), without the inf/nan guard nvcc wraps around the cvt; activations here are finite.
  // xr: raw X of the chunk, row ra (xr[0..1]) and row ra + 8 (xr[2..3]); rows past P are zeros, accumulator rows the
  // epilogue never reads.
  auto make_frag = [&](const float4 (&xr)[4], uint32_t (&hi)[16], uint32_t (&lo)[16]) {
    const float s8[8] = {sc[0].x, sc[0].y, sc[0].z, sc[0].w, sc[1].x, sc[1].y, sc[1].z, sc[1].w};
    const float h8[8] = {sh[0].x, sh[0].y, sh[0].z, sh[0].w, sh[1].x, sh[1].y, sh[1].z, sh[1].w};
    const float x16[16] = {xr[0].x, xr[0].y, xr[0].z, xr[0].w, xr[1].x, xr[1].y, xr[1].z, xr[1].w,
                           xr[2].x, xr[2].y, xr[2].z, xr[2].w, xr[3].x, xr[3].y, xr[3].z, xr[3].w};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      // physical column 2s + b of row half h is k-step s, register 2b + h
      const int h = i >> 3, s = (i & 7) >> 1, b = i & 1;
      const float v = fmaxf(fmaf(x16[i], s8[i & 7], h8[i & 7]), relu_floor);
      const uint32_t vh = (__float_as_uint(v) + 0x1000u) & 0xffffe000u;
      hi[4 * s + 2 * b + h] = vh;
      lo[4 * s + 2 * b + h] = (__float_as_uint(v - __uint_as_float(vh)) + 0x1000u) & 0xffffe000u;
    }
  };

  // ---- epilogue role: warp -> 32-row quarter q of the warpgroup tile, column chunks with (ch & 1) == half
  const int q = wwarp & 1, half = wwarp >> 1;
  const int g = d.group;
  const bool want_stats = d.stat_partial != nullptr;
  const bool want_grp = (d.gmax != nullptr) || (d.gmin != nullptr);
  float* tile_s = reinterpret_cast<float*>(smem + tile_base + wg * SM::TILE);
  // BN statistics: ONE partial row per (CTA, warpgroup, row quarter), accumulated over the warpgroup's tiles.  A CTA keeps
  // its column tile, so column 64 hf + 32 half + lane of the tile belongs to this lane for the whole kernel: its running
  // (sum, sum^2) stays in registers, as tile + previous, and is stored once at the end.
  float st_s[BN / TC_EPI_COLS], st_q[BN / TC_EPI_COLS];
#pragma unroll
  for (int hf = 0; hf < BN / TC_EPI_COLS; ++hf) st_s[hf] = st_q[hf] = 0.f;

  float acc[BN / 2];
  uint32_t fh0[16], fl0[16], fh1[16], fl1[16];       // A fragments of even / odd chunks
  if (my_tiles > 0) fetch_affine(0);
  for (int jt = 0; jt < my_tiles; ++jt) {
    const int row0 = tile_row0(wg, jt);
    // ================= main loop over the tile's K chunks
    auto step = [&](uint32_t (&fh)[16], uint32_t (&fl)[16], int kc) {
      const int ia = jt * KC + kc;                   // activation ring position: stage ia % SA, phase parity (ia / SA) & 1
      const int sa = ia % SA;
      mbar_wait(a_full_bar(wg, sa), (ia / SA) & 1);
      const uint8_t* st = smem + a_stage(wg, sa);
      const float4 xr[4] = {*reinterpret_cast<const float4*>(st + a_off0), *reinterpret_cast<const float4*>(st + a_off1),
                            *reinterpret_cast<const float4*>(st + a_off0 + 1024),
                            *reinterpret_cast<const float4*>(st + a_off1 + 1024)};
      make_frag(xr, fh, fl);                         // the last reader of fh / fl, chunk kc - 2, retired
      if (kc + 1 < KC) fetch_affine(kc + 1);
      else if (jt + 1 < my_tiles) fetch_affine(0);
      const int it = ring ? jt * KC + kc : kc;       // ring position: stage it % S, phase parity (it / S) & 1
      mbar_wait(full_bar(it % S), (it / S) & 1);
      wgmma_chunk_rs<BN, SINGLE>(acc, fh, fl, smem_base + (it % S) * SM::B_STAGE, kc == 0);
      wgmma_wait<1>();                               // chunk kc - 1 retired
      // its activation stage is free: the retired wgmma read registers computed from every thread's loads of it.  (An
      // arrive right after the loads let the TMA refill land before some of them had read the stage.)
      if (kc > 0 && wtid == 0) mbar_arrive(a_empty_bar(wg, (ia - 1) % SA));
      if (ring && kc > 0 && wtid == 0) mbar_arrive(empty_bar((it - 1) % S));
    };
#pragma unroll 1
    for (int kc = 0; kc < KC; kc += 2) {
      step(fh0, fl0, kc);
      if (kc + 1 < KC) step(fh1, fl1, kc + 1);
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (wtid == 0) mbar_arrive(a_empty_bar(wg, (jt * KC + KC - 1) % SA));
    if (ring && wtid == 0) mbar_arrive(empty_bar((jt * KC + KC - 1) % S));

    // group > 32: per-quarter results go to comb[kind][quarter of the 128-row tile][column]; with COMBINE the buffer
    // alternates with the tile so that one warpgroup's next tile cannot overwrite what the other still reads
    float* comb = reinterpret_cast<float*>(smem + comb_base + (COMBINE ? (jt & 1) : 0) * SM::COMB);
    const int cq = 2 * wg + q;                       // quarter slot in comb
    const int wrow0 = row0 + q * 32;                 // first row of this warp
    const int nvalid = min(32, max(0, P - wrow0));   // valid rows of this warp
    const float* addp[2];                            // addend rows of this thread's accumulator rows ra, ra + 8
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + ra + 8 * h;
      addp[h] = nullptr;
      if (d.addend && row < P) {
        const int gi = d.add_index ? __ldg(d.add_index + row) : row / d.add_group;
        addp[h] = d.addend + (size_t)gi * d.ld_add + n0;
      }
    }
    constexpr int EC = TC_EPI_COLS;
#pragma unroll
    for (int hf = 0; hf < BN / EC; ++hf) {
      // ================= accumulators of columns 64 hf .. 64 hf + 63 (+addend, +bias) -> staging tile,
      // element (r, c) at r*64 + (((c>>2) ^ (r&7))<<2) + (c&3)
      named_bar_sync(1 + wg, 128);                   // this warpgroup finished reading the staging tile's previous contents
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = ra + 8 * h;
        float* trow = tile_s + (size_t)r * EC;
#pragma unroll
        for (int j = 0; j < EC / 8; ++j) {
          const int cc = 8 * j + 2 * (lane & 3), ct = hf * EC + cc;     // column in the staging tile / in the BN tile
          float v0 = acc[4 * (hf * EC / 8 + j) + 2 * h], v1 = acc[4 * (hf * EC / 8 + j) + 2 * h + 1];
          if (addp[h]) { const float2 a = __ldg(reinterpret_cast<const float2*>(addp[h] + ct)); v0 += a.x; v1 += a.y; }
          if (d.bias) { const float2 b = __ldg(reinterpret_cast<const float2*>(d.bias + n0 + ct)); v0 += b.x; v1 += b.y; }
          *reinterpret_cast<float2*>(trow + ((((cc >> 2) ^ (r & 7))) << 2) + (cc & 3)) = make_float2(v0, v1);
        }
      }
      named_bar_sync(1 + wg, 128);

      // ================= epilogue: warp (q, half) on the 32 x 32 chunk ch of rows 32q..32q+31 of the warpgroup tile
      const int ch = 2 * hf + half;
      const int cb = n0 + ch * 32;
      // element (r, c) of the chunk: tw[r*64 + (((c>>2) ^ (r&7))<<2) + (c&3)]
      const float* tw = tile_s + (size_t)(q * 32) * EC + half * 32;
      const int l8 = lane & 7, rsub = lane >> 3;
      if (d.Y) {
        // coalesced stores: 8 lanes cover one 128-byte row segment, a warp instruction writes 4 full lines
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = 4 * i + rsub;
          if (r < nvalid)
            *reinterpret_cast<float4*>(d.Y + (size_t)(wrow0 + r) * d.ldy + cb + l8 * 4) =
                *reinterpret_cast<const float4*>(tw + r * EC + ((l8 ^ (r & 7)) << 2));
        }
      }
      // column view: lane owns column cb + lane
      const int cl = ch * 32 + lane;                 // column inside the tile
      const int csub = lane & 3, cchunk = lane >> 2;
      if (want_stats && !want_grp) {
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
        if (nvalid == 32) {
#pragma unroll
          for (int r = 0; r < 32; r += 2) {
            const float x0 = tw[r * EC + ((cchunk ^ (r & 7)) << 2) + csub];
            const float x1 = tw[(r + 1) * EC + ((cchunk ^ ((r + 1) & 7)) << 2) + csub];
            s0 += x0; q0 = fmaf(x0, x0, q0); s1 += x1; q1 = fmaf(x1, x1, q1);
          }
        } else {
          for (int r = 0; r < nvalid; ++r) { const float x0 = tw[r * EC + ((cchunk ^ (r & 7)) << 2) + csub]; s0 += x0; q0 = fmaf(x0, x0, q0); }
        }
        st_s[hf] = jt ? (s0 + s1) + st_s[hf] : s0 + s1;
        st_q[hf] = jt ? (q0 + q1) + st_q[hf] : q0 + q1;
      } else if (want_grp) {
        float s = 0.f, ss = 0.f;
        float mx0 = -INFINITY, mn0 = INFINITY, mx1 = -INFINITY, mn1 = INFINITY;
        int ax0 = 0, an0 = 0, ax1 = 0, an1 = 0;
        const int hrows = (g == 16) ? 16 : 32;      // rows per in-warp group segment
        if (nvalid == 32 && !d.garg_max && !d.garg_min) {
          // forward-only fast path (full slice, no arg outputs): 4 instructions per element instead of ~12
          float s1 = 0.f, q1 = 0.f;
#pragma unroll
          for (int r = 0; r < 16; ++r) {
            const float x0 = tw[r * EC + ((cchunk ^ (r & 7)) << 2) + csub];
            const float x1 = tw[(r + 16) * EC + ((cchunk ^ (r & 7)) << 2) + csub];       // (r + 16) & 7 == r & 7
            s += x0; ss = fmaf(x0, x0, ss); s1 += x1; q1 = fmaf(x1, x1, q1);
            mx0 = fmaxf(mx0, x0); mn0 = fminf(mn0, x0);
            if (hrows == 16) { mx1 = fmaxf(mx1, x1); mn1 = fminf(mn1, x1); }
            else { mx0 = fmaxf(mx0, x1); mn0 = fminf(mn0, x1); }
          }
          s += s1; ss += q1;
        } else {
#pragma unroll 8
          for (int r = 0; r < 32; ++r) {
            const float x = tw[r * EC + ((cchunk ^ (r & 7)) << 2) + csub];
            const bool ok = r < nvalid;
            if (ok) { s += x; ss = fmaf(x, x, ss); }
            if (r < hrows) {
              if (ok && x > mx0) { mx0 = x; ax0 = r; }
              if (ok && x < mn0) { mn0 = x; an0 = r; }
            } else {
              if (ok && x > mx1) { mx1 = x; ax1 = r; }
              if (ok && x < mn1) { mn1 = x; an1 = r; }
            }
          }
        }
        if (want_stats) {
          st_s[hf] = jt ? s + st_s[hf] : s;
          st_q[hf] = jt ? ss + st_q[hf] : ss;
        }
        if (g == 16) {
          const int grow = wrow0 / 16;
          if (nvalid > 0) {
            if (d.gmax) d.gmax[(size_t)grow * Cout + cb + lane] = mx0;
            if (d.gmin) d.gmin[(size_t)grow * Cout + cb + lane] = mn0;
            if (d.garg_max) d.garg_max[(size_t)grow * Cout + cb + lane] = ax0;
            if (d.garg_min) d.garg_min[(size_t)grow * Cout + cb + lane] = an0;
          }
          if (nvalid > 16) {
            if (d.gmax) d.gmax[(size_t)(grow + 1) * Cout + cb + lane] = mx1;
            if (d.gmin) d.gmin[(size_t)(grow + 1) * Cout + cb + lane] = mn1;
            if (d.garg_max) d.garg_max[(size_t)(grow + 1) * Cout + cb + lane] = ax1 - 16;
            if (d.garg_min) d.garg_min[(size_t)(grow + 1) * Cout + cb + lane] = an1 - 16;
          }
        } else if (g == 32) {
          if (nvalid > 0) {
            const int grow = wrow0 / 32;
            if (d.gmax) d.gmax[(size_t)grow * Cout + cb + lane] = mx0;
            if (d.gmin) d.gmin[(size_t)grow * Cout + cb + lane] = mn0;
            if (d.garg_max) d.garg_max[(size_t)grow * Cout + cb + lane] = ax0;
            if (d.garg_min) d.garg_min[(size_t)grow * Cout + cb + lane] = an0;
          }
        } else {                                     // 64 / 128: combine the row quarters below
          const int qoff = (COMBINE ? cq : q) * 32;  // first row of this quarter inside the group
          comb[(0 * 4 + cq) * BN + cl] = mx0; comb[(1 * 4 + cq) * BN + cl] = mn0;
          reinterpret_cast<int*>(comb)[(2 * 4 + cq) * BN + cl] = qoff + ax0;
          reinterpret_cast<int*>(comb)[(3 * 4 + cq) * BN + cl] = qoff + an0;
        }
      }
    }
    if (want_grp && g > 32) {
      // group 64 is this warpgroup's tile (quarters 2wg, 2wg + 1); group 128 (COMBINE) is both warpgroups' tiles
      if (COMBINE) named_bar_sync(3, TC_CONSUMERS);
      else named_bar_sync(1 + wg, 128);
      const int q0 = COMBINE ? 0 : 2 * wg, nq = COMBINE ? 4 : 2;
      const int grow = row0 / g;
      for (int cl = COMBINE ? tid : wtid; cl < BN; cl += COMBINE ? TC_CONSUMERS : 128) {
        float mx = -INFINITY, mn = INFINITY; int ax = 0, an = 0;
        for (int w = q0; w < q0 + nq; ++w) {
          const float a = comb[(0 * 4 + w) * BN + cl], b = comb[(1 * 4 + w) * BN + cl];
          if (a > mx) { mx = a; ax = reinterpret_cast<int*>(comb)[(2 * 4 + w) * BN + cl]; }
          if (b < mn) { mn = b; an = reinterpret_cast<int*>(comb)[(3 * 4 + w) * BN + cl]; }
        }
        if (d.gmax) d.gmax[(size_t)grow * Cout + n0 + cl] = mx;
        if (d.gmin) d.gmin[(size_t)grow * Cout + n0 + cl] = mn;
        if (d.garg_max) d.garg_max[(size_t)grow * Cout + n0 + cl] = ax;
        if (d.garg_min) d.garg_min[(size_t)grow * Cout + n0 + cl] = an;
      }
    }
  }
  // one store per column; a warpgroup without a tile (a CTA with a single 64-row tile) still owns its statistic slots and
  // writes zeros
  if (want_stats) {
    float* stat_row = d.stat_partial + ((size_t)base * 4 + 2 * wg + q) * 2 * Cout;
#pragma unroll
    for (int hf = 0; hf < BN / TC_EPI_COLS; ++hf) {
      const int col = n0 + hf * TC_EPI_COLS + half * 32 + lane;
      stat_row[col] = st_s[hf];
      stat_row[Cout + col] = st_q[hf];
    }
  }
}

// persistent grid: one CTA per SM, rounded down to a multiple of the column-tile count so that a CTA keeps its column
// tile (BN-statistic slots are per CTA)
static int tc_grid(int P, int Cout, int BN, int sm_count) {
  const int m_tiles = cdiv(P, TC_BM), n_tiles = Cout / BN;
  const int g = min(sm_count, m_tiles * n_tiles);
  return max(n_tiles, g / n_tiles * n_tiles);
}

template <int BN, bool COMBINE, bool SINGLE>
static int launch_tc(const usip_layer_desc& d, const uint32_t* wpack, cudaStream_t st) {
  using SM = TcSmem<BN>;
  static_assert(SM::BYTES <= 232448, "shared memory budget (227 KB per block)");
  static_assert(SM::A_STAGES >= 2, "a chunk's activation stage is released while the next chunk's is in use");
  static bool attr_set = false;
  const int sm_count = device_sm_count();
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(layer_fwd_tc_kernel<BN, COMBINE, SINGLE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::BYTES);
    if (e != cudaSuccess) { set_last_error("layer_fwd_tc smem attr"); return (int)e; }
    attr_set = true;
  }
  // X as a 2-D tensor {Cin, P} with row stride ldx, box = one K chunk of one warpgroup tile; rows past P read as zeros
  // (max(P, 1): a map needs a non-empty tensor, and with P = 0 nothing is loaded)
  CUtensorMap xmap;
  const cuuint64_t dims[2] = {(cuuint64_t)d.Cin, (cuuint64_t)max(d.P, 1)};
  const cuuint64_t strides[1] = {(cuuint64_t)d.ldx * 4};
  const cuuint32_t box[2] = {TC_BK, TC_WG_ROWS};
  const cuuint32_t estr[2] = {1, 1};
  int te = encode_tensor_map_tiled(&xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(d.X), dims, strides, box,
                                   estr, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   "layer_fwd_tc: X tensor map");
  if (te) return te;
  const int grid = tc_grid(d.P, d.Cout, BN, sm_count);
  layer_fwd_tc_kernel<BN, COMBINE, SINGLE><<<grid, TC_THREADS, SM::BYTES, st>>>(d, wpack, xmap);
  return check_launch("layer_fwd_tc_kernel");
}

// column-tile width of this layer: 128 (64 accumulator registers per thread) unless Cout needs 64, or the layer has
// fewer row tiles than there are SMs (node-level GEMMs), where narrower column tiles fill more SMs
static int tc_pick_bn(const usip_layer_desc& d) {
  if (d.Cout % 128 == 0 && (long long)cdiv(d.P, TC_BM) * (d.Cout / 128) >= device_sm_count()) return 128;
  return 64;
}

// number of [2, Cout] BN-statistic partial rows usip_layer_fwd writes for this descriptor (tensor-core precisions): one
// per (CTA row base = blockIdx.x / n_tiles, warpgroup, 32-row quarter of the warpgroup tile), slot base*4 + 2*wg + q;
// the n_tiles CTAs of one base fill disjoint column ranges of the same four slots
int tc_stat_slots(const usip_layer_desc& d) {
  const int BN = tc_pick_bn(d);
  return tc_grid(d.P, d.Cout, BN, device_sm_count()) / (d.Cout / BN) * 4;
}

// Packs the weights of n tensor-core layers exactly as layer_fwd_tc() would on a call with tc_weights_packed == 0 (same
// column-tile choice), in ceil(n / 32) launches.
int tc_pack_many(const usip_layer_desc* descs, int n, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += TC_PACK_MANY) {
    TcPackMany pm;
    pm.n = min(TC_PACK_MANY, n - i0);
    int blocks = 0;
    for (int i = 0; i < pm.n; ++i) {
      const usip_layer_desc& d = descs[i0 + i];
      USIP_REQUIRE(d.W && d.tc_workspace && d.Cin % TC_BK == 0 && d.Cout % 64 == 0 &&
                   d.tc_workspace_bytes >= (int64_t)2 * d.Cout * d.Cin * 4, "tc_pack_many: bad descriptor");
      pm.blk0[i] = blocks;
      pm.W[i] = d.W; pm.out[i] = reinterpret_cast<uint32_t*>(d.tc_workspace);
      pm.ldw[i] = d.ldw; pm.transposed[i] = d.w_transposed; pm.Cout[i] = d.Cout; pm.Cin[i] = d.Cin;
      pm.BN[i] = tc_pick_bn(d);
      blocks += cdiv(d.Cout * (d.Cin / 4), 256);
    }
    pm.blk0[pm.n] = blocks;
    tc_pack_many_kernel<<<blocks, 256, 0, st>>>(pm);
    int e = check_launch("tc_pack_many_kernel");
    if (e) return e;
  }
  return 0;
}

int layer_fwd_tc(const usip_layer_desc& d, cudaStream_t st) {
  USIP_REQUIRE(d.Cin % TC_BK == 0 && d.Cout % 64 == 0, "layer_fwd_tc: needs Cin%32==0 and Cout%64==0");
  USIP_REQUIRE((d.ldx % 4) == 0 && (reinterpret_cast<uintptr_t>(d.X) % 16) == 0, "layer_fwd_tc: X must be 16B aligned");
  USIP_REQUIRE(!d.Y || ((d.ldy % 4) == 0 && (reinterpret_cast<uintptr_t>(d.Y) % 16) == 0), "layer_fwd_tc: Y must be 16B aligned");
  USIP_REQUIRE(!d.addend || ((d.ld_add % 4) == 0 && (reinterpret_cast<uintptr_t>(d.addend) % 16) == 0), "layer_fwd_tc: addend alignment");
  USIP_REQUIRE(!d.bias || (reinterpret_cast<uintptr_t>(d.bias) % 16) == 0, "layer_fwd_tc: bias alignment");
  USIP_REQUIRE(!d.in_scale || ((reinterpret_cast<uintptr_t>(d.in_scale) % 16) == 0 && (reinterpret_cast<uintptr_t>(d.in_shift) % 16) == 0),
               "layer_fwd_tc: scale/shift alignment");
  USIP_REQUIRE(d.tc_workspace && d.tc_workspace_bytes >= (int64_t)2 * d.Cout * d.Cin * 4, "layer_fwd_tc: workspace too small");
  if (d.gmax || d.gmin) USIP_REQUIRE(d.group == 16 || d.group == 32 || d.group == 64 || d.group == 128, "layer_fwd_tc: group must be 16/32/64/128");
  const int BN = tc_pick_bn(d);
  uint32_t* wpack = reinterpret_cast<uint32_t*>(d.tc_workspace);
  if (!d.tc_weights_packed) {
    const int total = d.Cout * (d.Cin / 4);
    tc_pack_weights_kernel<<<cdiv(total, 256), 256, 0, st>>>(d.W, d.ldw, d.w_transposed, d.Cout, d.Cin, BN, wpack);
    int e = check_launch("tc_pack_weights_kernel");
    if (e) return e;
  }
  const bool combine = (d.gmax || d.gmin) && d.group == 128;      // groups of 16..64 rows lie inside a warpgroup tile
  if (d.debug_flags & 8) {
    if (combine) return BN == 128 ? launch_tc<128, true, true>(d, wpack, st) : launch_tc<64, true, true>(d, wpack, st);
    return BN == 128 ? launch_tc<128, false, true>(d, wpack, st) : launch_tc<64, false, true>(d, wpack, st);
  }
  if (combine) return BN == 128 ? launch_tc<128, true, false>(d, wpack, st) : launch_tc<64, true, false>(d, wpack, st);
  return BN == 128 ? launch_tc<128, false, false>(d, wpack, st) : launch_tc<64, false, false>(d, wpack, st);
}

}  // namespace usip
