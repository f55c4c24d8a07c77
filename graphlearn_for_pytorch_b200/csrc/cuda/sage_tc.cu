// Fused  gather -> neighbour-mean -> [mean | self] x W -> bias/ReLU  for sm_90a.
//
// This is the headline kernel of the engine: the A operand of the first-layer
// GraphSAGE GEMM is never materialised in HBM.  Producer warps pull feature rows
// straight out of the range-partitioned feature table -- local HBM *or a peer
// GPU's HBM over NVLink* (plain ld.global.nc on IPC-mapped addresses) -- reduce
// them to the neighbour mean in registers and write bf16 tiles into
// SWIZZLE_128B K-major shared memory; warpgroups multiply each tile with wgmma
// (m64n64k16, fp32 accumulators in registers) against the weight image that
// cp.async.bulk (TMA bulk copy) parked in shared memory, add bias, apply ReLU
// and store bf16.
//
// It replaces, in one launch, the reference's GatherTensorKernel
// (csrc/cuda/unified_tensor.cu:47-81) + PyG scatter-mean + two cuBLAS GEMMs +
// bias/ReLU elementwise kernels, and keeps the row count on the device.
#include "launch_utils.h"
#include "tc_utils.cuh"

namespace glt {

namespace {

using namespace tc;

constexpr int kTileM = 128;
constexpr int kProducerWarps = 16;
constexpr int kChunkBytes = 128;                    // 64 bf16 = one SWIZZLE_128B atom row
constexpr int kAChunkTile = kTileM * kChunkBytes;   // 16 KB per K-chunk of an A tile
constexpr int kMmaStageBytes = 16 * 128;            // per-warp epilogue staging: 16 rows x 64 bf16

// One warpgroup's work on half h (rows 64 h .. 64 h + 63) of a 128-row tile:
// Z[row0 + 64 h ...] = act([mean | self] . W^T + b).  It runs in blocks of 64 columns (wgmma.m64n64k16;
// m64n32k16 for a 32-column tail) so that the accumulator takes 32 registers per thread in CTAs of up to 768
// threads.  A: NKC K-chunks of [128 rows x 128 B], W: NKC K-chunks of [N rows x 128 B], both SWIZZLE_128B K-major.
// `release()` runs once the last MMA that reads A has completed.  Every block goes through this warp's staging
// buffer (16 rows x 128 B) and leaves with 8 lanes per row, so each store instruction covers full 128-byte lines.
template <int NKC, typename Release>
__device__ __forceinline__ void wg_mma_half(uint32_t a_u32, uint32_t w_u32, int N, const __nv_bfloat16* bias, int relu,
                                            int h, uint32_t stg_u32, uint8_t* zbase, int row0, int T, Release release) {
  const int lane = threadIdx.x & 31;
  const int wq = (threadIdx.x >> 5) & 3;    // warp inside the warpgroup: fragment rows 16 wq .. 16 wq + 15
  const int cl = 2 * (lane & 3);
  for (int c0 = 0; c0 < N; c0 += 64) {
    const int cw = min(64, N - c0);         // 64 or 32 columns in this block
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < NKC; ++kc) {
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const uint64_t da = make_sw128_desc(a_u32 + kc * kAChunkTile + h * 8192 + k4 * 32);
        const uint64_t db = make_sw128_desc(w_u32 + (kc * N + c0) * kChunkBytes + k4 * 32);
        if (cw == 64) wgmma_m64n64k16_bf16<0, 0>(acc, da, db, (kc | k4) ? 1u : 0u);
        else wgmma_m64n32k16_bf16(acc, da, db, (kc | k4) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (c0 + 64 >= N) release();
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      if (jj * 8 < cw) {
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + c0 + jj * 8 + cl));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float x0 = acc[4 * jj + 2 * i] + b.x, x1 = acc[4 * jj + 2 * i + 1] + b.y;
          if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          const __nv_bfloat162 o = __floats2bfloat162_rn(x0, x1);
          const int lr = (lane >> 2) + 8 * i;
          sts32(stg_u32 + lr * 128 + ((jj ^ (lr & 7)) << 4) + cl * 2, *reinterpret_cast<const int32_t*>(&o));
        }
      }
    }
    __syncwarp();
    const int lpr = cw >> 3;          // 8 (64 columns) or 4 (32 columns) lanes per row
    const int rpi = 32 / lpr;         // rows per store instruction
    const int rl = lane / lpr, ch = lane % lpr;
    for (int rb = 0; rb < 16; rb += rpi) {
      const int row = rb + rl;
      uint4 o;
      asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
                   : "r"(stg_u32 + row * 128 + ((ch ^ (row & 7)) << 4)));
      const int t = row0 + h * 64 + wq * 16 + row;
      if (t < T) *reinterpret_cast<uint4*>(zbase + (static_cast<int64_t>(t) * N + c0) * 2 + ch * 16) = o;
    }
    __syncwarp();                     // the staging buffer is reused by the next block
  }
}

// Decoupled address resolution.  A producer that chases its own pointers (deg/ELL -> node id -> owner shard)
// spends about half of every tile in that dependent chain with no feature bytes in flight.  The chase therefore
// belongs to four dedicated RESOLVER warps (one thread per tile row) that run one tile AHEAD of the loaders and
// publish, per row, 15 neighbour row pointers + the self-row pointer + the degree into a double-buffered
// shared-memory table.  The 16 LOADER warps then do nothing but stream 16-byte feature vectors (6 rows in flight
// per lane: the self row rides in slot 0 of the first batch and goes straight to the A tile) and reduce them.
// Resolver warp 0 also issues the weight bulk copy.  The tile's GEMM + epilogue is split over two warpgroups:
// the last one takes rows 0-63, the resolvers take rows 64-127 once they have published the next tile's table,
// which halves the time the A buffer stays locked.  The CTA stays at 24 warps (80 registers per thread).
//
//   warps 0-15  loaders   (8-lane group per target row, 2 rows per group per tile)
//   warps 16-19 resolvers (warp 16, lane 0: TMA weight load) + wgmma / epilogue of tile rows 64-127
//   warps 20-23 wgmma / epilogue of tile rows 0-63
constexpr int kResolverWarps = 4;
constexpr int kThreads3 = (kProducerWarps + kResolverWarps + 4) * 32;
constexpr int kKP = 15;                      // neighbour handles published per row (+1 self)
constexpr int kTabStageBytes = kTileM * 16 * 4;   // 16 x uint32 row handles per tile row
constexpr int kStageWarpBytes = 2 * kMmaStageBytes;   // epilogue staging of warp w and of resolver warp w
constexpr int kBarBytes = 256;
constexpr uint32_t kNoRow = 0xFFFFFFFFu;

// A row handle is (shard << 28) | row-inside-shard; the loaders turn it into an address with one
// LDS from a 16-entry base table, so a table row costs 64 B instead of 128 B of pointers -- the
// 16 KB this frees hold the epilogue's staging buffers.
// FP8 = true: the feature table holds MXFP8 rows (d e4m3 bytes + d/32 UE8M0 block scales, padded to a multiple
// of 16 bytes; data/quantize.py) -- the loaders move HALF the bytes per row, de-quantise in registers while they
// reduce the neighbour mean in fp32 and still hand bf16 tiles to the tensor core (d = 128 only).
template <int NC, bool FP8>
__global__ void __launch_bounds__(kThreads3, 1) k_sage_fused3(SageFusedArgs f) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int N = f.n_out;
  constexpr int NKC = 2 * NC;
  constexpr int NB = 6;    // first batch: self + 5 neighbour rows in flight per lane
  constexpr int NB2 = 5;   // later batches (fan-out 10 / 15 -> 2 / 3 batches in total)
  uint8_t* smem_w = smem;
  uint8_t* smem_a = smem_w + NKC * N * kChunkBytes;
  uint8_t* tab = smem_a + NKC * kAChunkTile;                  // [2][128][16] uint32
  uint8_t* degtab = tab + 2 * kTabStageBytes;                 // [2][128] int32
  uint8_t* stg = degtab + 2 * kTileM * 4;                     // [4 warps][32 rows][128 B]
  uint8_t* bias_s = stg + 4 * kStageWarpBytes;                // [256] bf16
  uint8_t* base_s = bias_s + 512;                             // [16] shard base pointers
  uint64_t* bars = reinterpret_cast<uint64_t*>(base_s + 128);
  const uint32_t a_u32 = smem_u32(smem_a);
  const uint32_t tab_u32 = smem_u32(tab);
  const uint32_t deg_u32 = smem_u32(degtab);
  const uint32_t base_u32 = smem_u32(base_s);
  const uint32_t bar_w = smem_u32(bars + 0);
  const uint32_t bar_a_full = smem_u32(bars + 1);
  const uint32_t bar_a_empty = smem_u32(bars + 2);
  const uint32_t bar_p_full0 = smem_u32(bars + 3);    // +8: stage 1
  const uint32_t bar_p_empty0 = smem_u32(bars + 5);   // +8: stage 1

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const SageAggArgs& a = f.agg;
  const int64_t row_bytes = FP8 ? static_cast<int64_t>(a.feat.row_bytes) : static_cast<int64_t>(a.d) * 2;
  // Tile order.  Low tile indices hold the early hops (largest fan-out = most neighbour rows per
  // tile); a plain round-robin hands those to the same CTAs that also get a tile of the last,
  // partial wave.  The first wave is therefore dealt in reverse: the CTAs that own an extra tile
  // start on the cheapest tiles and the expensive ones go to CTAs with one tile fewer.
  auto tile_of = [&](int it) -> int {
    return it == 0 ? static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x)
                   : it * static_cast<int>(gridDim.x) + static_cast<int>(blockIdx.x);
  };
  constexpr int kResWarp0 = kProducerWarps;                   // 16
  constexpr int kEpiWarp0 = kProducerWarps + kResolverWarps;  // 20

  if (threadIdx.x == 0) {
    mbar_init(bar_w, 1);
    mbar_init(bar_a_full, kProducerWarps);
    mbar_init(bar_a_empty, 8);
    mbar_init(bar_p_full0, kResolverWarps);
    mbar_init(bar_p_full0 + 8, kResolverWarps);
    mbar_init(bar_p_empty0, kProducerWarps);
    mbar_init(bar_p_empty0 + 8, kProducerWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < kMaxParts) {  // shard base table (one entry for a dense local source)
    const void* b = nullptr;
    if (a.src_local)  // dense local source: "shard" p is the same matrix advanced by p * 2^28 rows, so any
                      // non-negative 32-bit row index decodes correctly
      b = reinterpret_cast<const uint8_t*>(a.src_local) +
          static_cast<int64_t>(threadIdx.x) * (int64_t(1) << 28) * row_bytes;
    else if (static_cast<int>(threadIdx.x) < a.feat.num_parts) b = a.feat.base[threadIdx.x];
    sts64(base_u32 + threadIdx.x * 8, reinterpret_cast<uint64_t>(b));
  }
  // programmatic dependent launch: barrier init and shard base table above overlap with the tail
  // of the previous kernel; global data written by predecessors (bias, counters, ELL, rows) is only read below
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x >= 64 && threadIdx.x < 64 + (N >> 3))  // bias -> smem, 16 B per thread
    *reinterpret_cast<uint4*>(bias_s + (threadIdx.x - 64) * 16) =
        reinterpret_cast<const uint4*>(f.bias)[threadIdx.x - 64];
  __syncthreads();
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int n_tiles = (T + kTileM - 1) / kTileM;

  if (warp < kProducerWarps) {
    // ------------------------------ loaders ------------------------------
    const int gl = lane & 7;
    const int gw = lane >> 3;
    const int group = warp * 4 + gw;  // 0..63
    constexpr int RPG = kTileM / (kProducerWarps * 4);
    auto row_addr = [&](uint32_t h) -> const uint8_t* {
      if (h == kNoRow) return nullptr;
      return reinterpret_cast<const uint8_t*>(lds64(base_u32 + ((h >> 28) << 3))) +
             static_cast<int64_t>(h & 0x0FFFFFFFu) * row_bytes;
    };
    int it = 0;
    for (int tile = tile_of(0); tile < n_tiles; tile = tile_of(++it)) {
      const int stage = it & 1;
      mbar_wait(bar_p_full0 + 8 * stage, (it >> 1) & 1);
      const uint32_t tb = tab_u32 + stage * kTabStageBytes;
      const uint32_t dgt = deg_u32 + stage * (kTileM * 4);
      bool waited = false;
      if constexpr (FP8) {
        static_assert(!FP8 || NC == 2, "the MXFP8 loader is written for d = 128");
        constexpr int NF = 8;              // rows in flight per lane in the first batch (self + 7 neighbours)
        const int cc = gl >> 2;            // bf16 K-chunk that this lane's 16 elements fall into
        const int vv = (gl & 3) * 2;       // first of the two 16-byte bf16 vectors inside that chunk
#pragma unroll 1
        for (int q = 0; q < RPG; ++q) {
          const int r = group + q * (kTileM / RPG);
          const int t = tile * kTileM + r;
          const int dg = lds32(dgt + r * 4);
          const uint32_t trow = tb + r * 64;
          const int sw = r & 15;
          const uint32_t arow = a_u32 + r * kChunkBytes;
          const uint32_t o0 = ((vv ^ (r & 7)) << 4), o1 = (((vv + 1) ^ (r & 7)) << 4);
          uint8_t* save = (t < T && f.a_save)
                              ? reinterpret_cast<uint8_t*>(f.a_save) + static_cast<int64_t>(t) * a.d * 4 + gl * 32
                              : nullptr;
          const int dgt_ = min(dg, kKP);
          float acc[16];
          {
            uint4 v[NF];
            uint32_t sc[NF];
#pragma unroll
            for (int jj = 0; jj < NF; ++jj) {
              const uint8_t* p = nullptr;
              if (jj <= dgt_) p = row_addr(static_cast<uint32_t>(lds32(trow + ((((jj + 15) & 15) ^ sw) << 2))));
              v[jj] = p ? ld_nc_v4(p + gl * 16) : make_uint4(0, 0, 0, 0);
              sc[jj] = p ? ld_nc_u32(p + a.d) : 0u;
            }
            if (!waited) { mbar_wait(bar_a_empty, (it & 1) ^ 1); waited = true; }
            {  // the row itself -> bf16 -> "self" half of the A tile
              float x[16];
#pragma unroll
              for (int i = 0; i < 16; ++i) x[i] = 0.f;
              mxfp8x16_accum(v[0], sc[0], gl, x);
              const uint4 s0 = pack_bf16x8(x, 1.f), s1 = pack_bf16x8(x + 8, 1.f);
              sts128(arow + (NC + cc) * kAChunkTile + o0, s0);
              sts128(arow + (NC + cc) * kAChunkTile + o1, s1);
              if (save) {
                *reinterpret_cast<uint4*>(save + a.d * 2) = s0;
                *reinterpret_cast<uint4*>(save + a.d * 2 + 16) = s1;
              }
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = 0.f;
#pragma unroll
            for (int jj = 1; jj < NF; ++jj) mxfp8x16_accum(v[jj], sc[jj], gl, acc);
          }
          if (dgt_ > NF - 1) {             // neighbours 7..14 in one more batch
            uint4 v[NF];
            uint32_t sc[NF];
#pragma unroll
            for (int jj = 0; jj < NF; ++jj) {
              const int j = NF - 1 + jj;
              const uint8_t* p = nullptr;
              if (j < dgt_) p = row_addr(static_cast<uint32_t>(lds32(trow + ((j ^ sw) << 2))));
              v[jj] = p ? ld_nc_v4(p + gl * 16) : make_uint4(0, 0, 0, 0);
              sc[jj] = p ? ld_nc_u32(p + a.d) : 0u;
            }
#pragma unroll
            for (int jj = 0; jj < NF; ++jj) mxfp8x16_accum(v[jj], sc[jj], gl, acc);
          }
          if (dg > kKP) {  // rows wider than the table (fan-out > 15): chase the rest here
            const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
            const int32_t* ellrow = a.ell[l.hop] + static_cast<int64_t>(l.row) * a.k[l.hop];
#pragma unroll 1
            for (int j = kKP; j < dg; ++j) {
              const int sidx = __ldg(ellrow + j);
              if (sidx < 0) continue;
              const uint8_t* p = src_row(a, sidx);
              if (p == nullptr) continue;  // an id the table does not hold: a zero row, still counted in dg
              mxfp8x16_accum(ld_nc_v4(p + gl * 16), ld_nc_u32(p + a.d), gl, acc);
            }
          }
          const float inv = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
          const uint4 m0 = pack_bf16x8(acc, inv), m1 = pack_bf16x8(acc + 8, inv);
          sts128(arow + cc * kAChunkTile + o0, m0);
          sts128(arow + cc * kAChunkTile + o1, m1);
          if (save) {
            *reinterpret_cast<uint4*>(save) = m0;
            *reinterpret_cast<uint4*>(save + 16) = m1;
          }
        }
      } else {
#pragma unroll 1
      for (int q = 0; q < RPG; ++q) {
        const int r = group + q * (kTileM / RPG);
        const int t = tile * kTileM + r;
        const int dg = lds32(dgt + r * 4);
        const uint32_t trow = tb + r * 64;
        const int sw = r & 15;
        const uint32_t off = r * kChunkBytes + ((gl ^ (r & 7)) << 4);
        uint8_t* save = (t < T && f.a_save)
                            ? reinterpret_cast<uint8_t*>(f.a_save) + static_cast<int64_t>(t) * a.d * 4 + gl * 16
                            : nullptr;
        const int dgt_ = min(dg, kKP);
        float acc[NC][8];
        {
          // first batch (peeled so the accumulators are not live across it): the row itself +
          // neighbours 0..NB-2.  Table entry 15 holds the self handle, entry j neighbour j.
          uint4 v[NB][NC];
#pragma unroll
          for (int jj = 0; jj < NB; ++jj) {
            const uint8_t* p = nullptr;
            if (jj <= dgt_) p = row_addr(static_cast<uint32_t>(lds32(trow + ((((jj + 15) & 15) ^ sw) << 2))));
#pragma unroll
            for (int c = 0; c < NC; ++c)
              v[jj][c] = p ? ld_nc_v4(p + c * kChunkBytes + gl * 16) : make_uint4(0, 0, 0, 0);
          }
          // the single A buffer is free once the previous tile's MMAs have retired; the wait
          // hides behind the loads issued above
          if (!waited) { mbar_wait(bar_a_empty, (it & 1) ^ 1); waited = true; }
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            sts128(a_u32 + (NC + c) * kAChunkTile + off, v[0][c]);
            if (save) *reinterpret_cast<uint4*>(save + a.d * 2 + c * kChunkBytes) = v[0][c];
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
          }
#pragma unroll
          for (int jj = 1; jj < NB; ++jj)
#pragma unroll
            for (int c = 0; c < NC; ++c) bf16x8_accum(v[jj][c], acc[c]);
        }
#pragma unroll 1
        for (int j0 = NB - 1; j0 < dgt_; j0 += NB2) {
          uint4 v[NB2][NC];
#pragma unroll
          for (int jj = 0; jj < NB2; ++jj) {
            const int j = j0 + jj;
            const uint8_t* p = nullptr;
            if (j < dgt_) p = row_addr(static_cast<uint32_t>(lds32(trow + ((j ^ sw) << 2))));
#pragma unroll
            for (int c = 0; c < NC; ++c)
              v[jj][c] = p ? ld_nc_v4(p + c * kChunkBytes + gl * 16) : make_uint4(0, 0, 0, 0);
          }
#pragma unroll
          for (int jj = 0; jj < NB2; ++jj)
#pragma unroll
            for (int c = 0; c < NC; ++c) bf16x8_accum(v[jj][c], acc[c]);
        }
        if (dg > kKP) {  // rows wider than the table (fan-out > 15): chase the rest here
          const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
          const int32_t* ellrow = a.ell[l.hop] + static_cast<int64_t>(l.row) * a.k[l.hop];
#pragma unroll 1
          for (int j = kKP; j < dg; ++j) {
            const int sidx = __ldg(ellrow + j);
            if (sidx < 0) continue;
            const uint8_t* p = src_row(a, sidx);
            if (p == nullptr) continue;  // an id the table does not hold: a zero row, still counted in dg
#pragma unroll
            for (int c = 0; c < NC; ++c) bf16x8_accum(ld_nc_v4(p + c * kChunkBytes + gl * 16), acc[c]);
          }
        }
        const float inv = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const uint4 m = pack_bf16x8(acc[c], inv);
          sts128(a_u32 + c * kAChunkTile + off, m);
          if (save) *reinterpret_cast<uint4*>(save + c * kChunkBytes) = m;
        }
      }
      }  // !FP8
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_p_empty0 + 8 * stage);  // table stage may be refilled
      fence_proxy_async();  // generic-proxy writes -> visible to the tensor-core (async) proxy
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_a_full);
    }
  } else if (warp < kEpiWarp0) {
    // ------------------------------ resolvers (+ weight load) ------------------------------
    const int r = (warp - kResWarp0) * 32 + lane;  // tile row owned by this thread
    const bool w_thread = (warp == kResWarp0) && (lane == 0);
    if (w_thread && tile_of(0) < n_tiles) {  // never leave a bulk copy in flight at exit
      const uint32_t w_bytes = NKC * N * kChunkBytes;
      mbar_expect_tx(bar_w, w_bytes);
      for (int kc = 0; kc < NKC; ++kc)
        bulk_g2s(smem_u32(smem_w + kc * N * kChunkBytes),
                 reinterpret_cast<const uint8_t*>(f.w_packed) + static_cast<size_t>(kc) * N * kChunkBytes,
                 N * kChunkBytes, bar_w);
    }
    // global row id -> (shard, row in shard)
    auto handle_of = [&](int64_t gid) -> uint32_t {
      if (gid < 0) return kNoRow;
#pragma unroll 1
      for (int p = 0; p < a.feat.num_parts; ++p)
        if (gid >= a.feat.row_begin[p] && gid < a.feat.row_begin[p + 1])
          return (static_cast<uint32_t>(p) << 28) | static_cast<uint32_t>(gid - a.feat.row_begin[p]);
      return kNoRow;
    };
    auto resolve = [&](int tile, int stage) {
      const int t = tile * kTileM + r;
      int dg = 0, kk = 0;
      const int32_t* ellp = nullptr;
      int64_t self_gid = -1;
      if (t < T) {
        const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
        kk = min(a.k[l.hop], kKP);
        ellp = a.ell[l.hop] + static_cast<int64_t>(l.row) * a.k[l.hop];
        dg = __ldg(a.deg + t);
        if (!a.src_local) self_gid = __ldg(a.nodes + t);
      }
      int sidx[kKP];
#pragma unroll
      for (int j = 0; j < kKP; ++j) sidx[j] = (j < kk) ? __ldg(ellp + j) : -1;  // independent of dg
      const uint32_t trow = tab_u32 + stage * kTabStageBytes + r * 64;
      const int sw = r & 15;
      if (a.src_local) {
#pragma unroll
        for (int j = 0; j < kKP; ++j)
          sts32(trow + ((j ^ sw) << 2), (j < dg && sidx[j] >= 0) ? sidx[j] : static_cast<int32_t>(kNoRow));
        sts32(trow + ((15 ^ sw) << 2), (t < T) ? t : static_cast<int32_t>(kNoRow));
      } else {
        int64_t gid[kKP];
#pragma unroll
        for (int j = 0; j < kKP; ++j) gid[j] = (j < dg && sidx[j] >= 0) ? __ldg(a.nodes + sidx[j]) : -1;
        uint32_t hnd[kKP + 1];
#pragma unroll
        for (int j = 0; j < kKP; ++j) hnd[j] = handle_of(gid[j]);
        hnd[kKP] = handle_of(self_gid);
#pragma unroll
        for (int j = 0; j < kKP; ++j) sts32(trow + ((j ^ sw) << 2), static_cast<int32_t>(hnd[j]));
        sts32(trow + ((15 ^ sw) << 2), static_cast<int32_t>(hnd[kKP]));
      }
      sts32(deg_u32 + (stage * kTileM + r) * 4, dg);
    };
    int it = 0;
    int tile = tile_of(0);
    if (tile < n_tiles) {
      resolve(tile, 0);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_p_full0);
    }
    for (; tile < n_tiles; tile = tile_of(++it)) {
      const int next = tile_of(it + 1);
      if (next < n_tiles) {
        const int ns = (it + 1) & 1;
        const int nu = (it + 1) >> 1;
        mbar_wait(bar_p_empty0 + 8 * ns, (nu & 1) ^ 1);
        resolve(next, ns);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_p_full0 + 8 * ns);
      }
      if (it == 0) mbar_wait(bar_w, 0);
      mbar_wait(bar_a_full, it & 1);
      wg_mma_half<NKC>(a_u32, smem_u32(smem_w), N, reinterpret_cast<const __nv_bfloat16*>(bias_s), f.relu, 1,
                       smem_u32(stg) + (warp - kResWarp0) * kStageWarpBytes + kMmaStageBytes,
                       reinterpret_cast<uint8_t*>(f.z), tile * kTileM, T, [&] {
                         __syncwarp();
                         if (lane == 0) mbar_arrive(bar_a_empty);   // A buffer reusable
                       });
    }
  } else {
    // ------------------------------ MMA + epilogue warpgroup ------------------------------
    const uint32_t stg_u32 = smem_u32(stg) + (warp - kEpiWarp0) * kStageWarpBytes;
    int it = 0;
    for (int tile = tile_of(0); tile < n_tiles; tile = tile_of(++it)) {
      if (it == 0) mbar_wait(bar_w, 0);
      mbar_wait(bar_a_full, it & 1);
      wg_mma_half<NKC>(a_u32, smem_u32(smem_w), N, reinterpret_cast<const __nv_bfloat16*>(bias_s), f.relu, 0, stg_u32,
                       reinterpret_cast<uint8_t*>(f.z), tile * kTileM, T, [&] {
                         __syncwarp();
                         if (lane == 0) mbar_arrive(bar_a_empty);   // A buffer reusable
                       });
    }
  }
}

// W [N, K] row-major bf16 -> [K/64][N][64] with the SWIZZLE_128B XOR applied, so
// the kernel can bulk-copy it verbatim into 1024-B aligned shared memory.
__global__ void k_pack_weight(const __nv_bfloat16* w, int n, int k, __nv_bfloat16* out) {
  pdl_enter();
  const int64_t total = static_cast<int64_t>(n) * k / 8;  // 16-byte vectors
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int row = static_cast<int>(i / (k / 8));
    const int v = static_cast<int>(i % (k / 8));  // 16-B vector index along K
    const int kc = v >> 3, cv = v & 7;
    const int64_t dst = (static_cast<int64_t>(kc) * n + row) * 64 + ((cv ^ (row & 7)) << 3);
    *reinterpret_cast<uint4*>(out + dst) = *reinterpret_cast<const uint4*>(w + static_cast<int64_t>(row) * k + v * 8);
  }
}

size_t fused3_smem_bytes(int d, int n_out) {
  const int nkc = 2 * (d / 64);
  return static_cast<size_t>(nkc) * n_out * kChunkBytes + static_cast<size_t>(nkc) * kAChunkTile +
         2 * kTabStageBytes + 2 * kTileM * sizeof(int32_t) + 4 * kStageWarpBytes + 512 + 128 + kBarBytes + 1024;
}

constexpr size_t kMaxSmem = 227 * 1024;

template <int NC, bool FP8>
void launch_fused3(const SageFusedArgs& a, int grid, cudaStream_t s) {
  const size_t smem = fused3_smem_bytes(a.agg.d, a.n_out);
  cudaFuncSetAttribute(k_sage_fused3<NC, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  launch_k(k_sage_fused3<NC, FP8>, dim3(grid), dim3(kThreads3), smem, s, a);
}

}  // namespace

int sage_fused_supported(int d, int n_out, const RowTable* feat) {
  if (d != 64 && d != 128) return 0;
  if (n_out % 32 != 0 || n_out < 32 || n_out > 256) return 0;
  if (fused3_smem_bytes(d, n_out) > kMaxSmem) return 0;
  if (feat != nullptr) {  // row handles: 4-bit part, 28-bit row inside the part
    if (feat->num_parts > 16) return 0;
    for (int p = 0; p < feat->num_parts; ++p)
      if (feat->row_begin[p + 1] - feat->row_begin[p] >= (int64_t(1) << 28)) return 0;
  }
  return 1;
}

void launch_sage_fused(const SageFusedArgs& a, int num_sms, cudaStream_t s) {
  const int max_tiles = (a.agg.cap_targets + kTileM - 1) / kTileM;
  const int grid = max_tiles < num_sms ? max_tiles : num_sms;
  if (a.feat_fp8) launch_fused3<2, true>(a, grid, s);  // the MXFP8 loader is written for d = 128
  else if (a.agg.d == 64) launch_fused3<1, false>(a, grid, s);
  else launch_fused3<2, false>(a, grid, s);
}

void launch_pack_weight(const void* w, int n, int k, void* packed, cudaStream_t s) {
  const int64_t total = static_cast<int64_t>(n) * k / 8;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  if (blocks < 1) blocks = 1;
  launch_k(k_pack_weight, dim3(blocks), dim3(256), 0, s, reinterpret_cast<const __nv_bfloat16*>(w), n, k,
           reinterpret_cast<__nv_bfloat16*>(packed));
}

}  // namespace glt
