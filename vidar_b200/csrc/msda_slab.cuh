// Persistent "slab" variants of the SpatialCrossAttention-shaped MSDA kernels (textually included by
// msda.cu inside namespace vidar { namespace { ... } }: they share its helpers).
//
// Why.  msda_backward_kernel is bound by the SM's L1 -> XBAR request path: every corner of every sample leaves the SM as one 128-byte `red.global.add.v4.f32` line
// (~5 request cycles), 277 k lines per SM and launch, while the 15x25 level receives ~3400 of them per
// pixel and head.  One head's slab of the coarsest level is 48 KB, so a block can keep it in SHARED
// MEMORY and send it out once:
//   backward  a persistent block owns one (batch, head) and an interleaved share of its query tiles; the
//             coarsest level's corner contributions are not reduced to HBM but recorded (pixel, weight)
//             in shared memory; after every tile (one query per warp, 16 warps) a barrier hands the 512
//             records over: warp w owns the pixels with (pixel & 15) == w, finds its records with a
//             ballot and adds weight * grad_out_row into the slab (lane = channel: conflict-free, no
//             atomics -- fp32 shared-memory atomics are CAS loops on sm_90a).  The slab is flushed once
//             per unit: 375 lines instead of ~110 k.  The flush is a TMA bulk reduction
//             (cp.reduce.async.bulk.tensor, SASS UTMAREDG) when a tensor map is available.
//   forward   the same decomposition with the coarsest level's value slab STAGED in shared memory by TMA
//             (cp.async.bulk.tensor.2d: one [rows x 32 floats] box per 256 rows out of the
//             [B*K, H*C] value matrix -- the head's 128-byte column slice of every pixel row), its samples
//             read with LDS.128 instead of L1 lookups (north_star's "TMA-staged image feature tiles").
// Both fall back to plain loads / reductions when the tensor map cannot be built (driver entry point
// missing): selected on the host, same arithmetic.
// Shapes: head dim 32 (lane = channel in the hand-over), L*P == 32 (one sample per lane), coarsest level
// <= 384 pixels, its points a multiple of 4.  Everything else runs the non-persistent kernels.
#include <cuda.h>

constexpr int kSlabWarps = 16;
constexpr int kSlabMaxRows = 384;
constexpr int kSlabRecords = kSlabWarps * 32;

constexpr int kSlabBoxRows = 128;     // TMA box: 128 pixel rows x 32 floats (16 KB); the level is covered by <= 3 boxes

struct SlabGeo {      // host-side part; the level's size and start are read from spatial_shapes / level_start on the device
  int first_it;       // first inner-loop iteration (of 8) whose samples sit on the coarsest level
  int pix_shift;      // log2(H*C)
  int parts;          // interleaved shares of a (batch, head)'s query tiles
  int tiles;          // ceil(Q / kSlabWarps)
  int use_tma;        // tensor map valid: stage / flush the slab with bulk tensor copies
};
// device-side part: the coarsest level of the pyramid and whether its per-head slab fits the shared-memory budget
struct SlabLevel {
  int start, rows, first_it, box_rows;
};
__device__ __forceinline__ SlabLevel slab_level(const MsdaParams& p, const SlabGeo& sg) {
  SlabLevel lv;
  lv.rows = (int)(__ldg(p.shapes + 2 * (p.L - 1)) * __ldg(p.shapes + 2 * (p.L - 1) + 1));
  lv.start = (int)__ldg(p.lsi + (p.L - 1));
  const bool fits = lv.rows <= kSlabMaxRows;
  lv.first_it = fits ? sg.first_it : 1 << 20;          // too large: nothing is privatised (plain reductions / loads)
  lv.box_rows = (fits && sg.use_tma) ? kSlabBoxRows : 0;
  if (!fits) lv.rows = 0;
  return lv;
}

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// one [box_rows x 32 floats] tile of the [B*K, H*C] matrix -> dense shared memory (row = 128 bytes)
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int col, int row, unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(col), "r"(row), "r"(smem_u32(bar)) : "memory");
}
// shared tile += into the global matrix (bulk tensor reduction; completes through the bulk async-group)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, int col, int row, const void* src) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%1, %2}], [%3];"
               ::"l"(map), "r"(col), "r"(row), "r"(smem_u32(src)) : "memory");
}

// ----------------------------------------------------------------------------------------------
// backward
// ----------------------------------------------------------------------------------------------
template <bool EPI, bool IDX>
__global__ void __launch_bounds__(kSlabWarps * 32, 2)
msda_backward_slab_kernel(const MsdaParams p, const SlabGeo sg, const __grid_constant__ CUtensorMap gmap,
                          const float* __restrict__ grad_out, float* __restrict__ grad_value,
                          float* __restrict__ grad_loc, float* __restrict__ grad_attn) {
  constexpr int CV = 8, NG = 4, ITERS = 8;
  extern __shared__ __align__(128) unsigned char slab_smem[];
  float* slab = reinterpret_cast<float*>(slab_smem);                       // [kSlabMaxRows][32]
  float* go_s = slab + kSlabMaxRows * 32;                                  // [2][16 warps][32]
  float* rec_w = go_s + 2 * kSlabRecords;                                  // [2][512]
  unsigned short* rec_p = reinterpret_cast<unsigned short*>(rec_w + 2 * kSlabRecords);   // [2][512]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane / CV, cl = lane % CV;
  const unsigned pix = (unsigned)p.pix_stride;
  const int units = p.B * p.H * sg.parts;
  const SlabLevel lv = slab_level(p, sg);

  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int nh = u / sg.parts, part = u % sg.parts;
    const int n = nh / p.H, h = nh % p.H;
    for (int i = tid; i < kSlabMaxRows * 8; i += kSlabWarps * 32) reinterpret_cast<float4*>(slab)[i] = f4_zero();
    __syncthreads();

    int round = 0;
    for (int qt = part; qt < sg.tiles; qt += sg.parts, ++round) {
      const int buf = round & 1;
      float* rw = rec_w + buf * kSlabRecords + warp * 32;
      unsigned short* rp = rec_p + buf * kSlabRecords + warp * 32;
      const int q = qt * kSlabWarps + warp;
      const long long item0 = ((long long)n * p.Q + q) * p.H + h;
      Row row;
      const bool item_live = q < p.Q && resolve_row<IDX>(p, item0, row);
      rw[lane] = 0.f;                      // dead rows / levels with fewer than 8 samples leave zero records
      __syncwarp();
      if (item_live) {
        const long long prow = (EPI && IDX) ? row.dense : item0;
        const float* loc0 = p.loc + (size_t)prow * 64;
        const float* att0 = p.attn + (size_t)prow * 32;
        float* gloc0 = grad_loc + (size_t)prow * 64;
        float* gatt0 = grad_attn + (size_t)prow * 32;
        const size_t slab_g = slab_offset(p, item0) + cl * 4;
        const float4 go = IDX ? f4_scale(row.inv, ldg4(grad_out + (size_t)row.dense * 32 + cl * 4))
                              : ldg4(grad_out + (size_t)item0 * 32 + cl * 4);
        if (g == 0) *reinterpret_cast<float4*>(go_s + buf * kSlabRecords + warp * 32 + cl * 4) = go;

        // ---- lane s decodes sample s (identical to msda_backward_kernel)
        const int s = lane;
        int base = 0, meta = 0;
        float lh = 0.f, lw = 0.f, aw = 0.f, fH = 0.f, fW = 0.f;
        float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
        {
          const int l = s / p.P;
          const int Hl = (int)__ldg(p.shapes + 2 * l), Wl = (int)__ldg(p.shapes + 2 * l + 1);
          float2 xy;
          if (EPI) {
            epi_decode(p, row.refrow, s, (float)Wl, (float)Hl, loc0, att0, xy, aw);
          } else {
            xy = __ldg(reinterpret_cast<const float2*>(loc0) + s);
            aw = __ldg(att0 + s);
          }
          decode_sample(xy.x, xy.y, Hl, Wl, (int)__ldg(p.lsi + l), base, meta, lh, lw, p.pix_stride);
          fH = (float)Hl;
          fW = (float)Wl;
          const float hh = 1.f - lh, hw = 1.f - lw;
          w1 = (meta & 1) ? aw * (hh * hw) : 0.f;
          w2 = (meta & 2) ? aw * (hh * lw) : 0.f;
          w3 = (meta & 4) ? aw * (lh * hw) : 0.f;
          w4 = (meta & 8) ? aw * (lh * lw) : 0.f;
        }
        float r1 = 0.f, r2 = 0.f, r3 = 0.f, r4 = 0.f;
#pragma unroll
        for (int it = 0; it < ITERS; ++it) {
          const int src = it * NG + g;
          const int sbase = __shfl_sync(0xffffffffu, base, src);
          const int smeta = __shfl_sync(0xffffffffu, meta, src);
          const float a1 = __shfl_sync(0xffffffffu, w1, src);
          const float a2 = __shfl_sync(0xffffffffu, w2, src);
          const float a3 = __shfl_sync(0xffffffffu, w3, src);
          const float a4 = __shfl_sync(0xffffffffu, w4, src);
          float d1 = 0.f, d2 = 0.f, d3 = 0.f, d4 = 0.f;
          const bool coarse = it >= lv.first_it;             // warp-uniform
          if (smeta & 15) {
            const unsigned o1 = (unsigned)sbase;
            const unsigned o2 = o1 + ((smeta & 16) ? pix : 0u);
            const unsigned o3 = o1 + (unsigned)(smeta >> 5);
            const unsigned o4 = o3 + (o2 - o1);
            const float* vs = p.value + slab_g;
            float* gs = grad_value + slab_g;
            asm volatile("" : "+l"(vs), "+l"(gs));
            const float4 v1 = ldg4(vs + o1);
            const float4 v2 = ldg4(vs + o2);
            const float4 v3 = ldg4(vs + o3);
            const float4 v4 = ldg4(vs + o4);
            if (!coarse) {
              red_add_v4(gs + o1, f4_scale(a1, go));
              red_add_v4(gs + o2, f4_scale(a2, go));
              red_add_v4(gs + o3, f4_scale(a3, go));
              red_add_v4(gs + o4, f4_scale(a4, go));
            } else if (cl == 0) {
              // coarsest level: record (pixel, weight) per corner; the owners add weight * grad_out row
              const int sl = ((it - lv.first_it) * NG + g) * 4;
              rw[sl + 0] = a1; rw[sl + 1] = a2; rw[sl + 2] = a3; rw[sl + 3] = a4;
              rp[sl + 0] = (unsigned short)((o1 >> sg.pix_shift) - lv.start);
              rp[sl + 1] = (unsigned short)((o2 >> sg.pix_shift) - lv.start);
              rp[sl + 2] = (unsigned short)((o3 >> sg.pix_shift) - lv.start);
              rp[sl + 3] = (unsigned short)((o4 >> sg.pix_shift) - lv.start);
            }
            d1 = f4_dot(go, v1); d2 = f4_dot(go, v2); d3 = f4_dot(go, v3); d4 = f4_dot(go, v4);
          }
          const bool up1 = (cl & (CV / 2)) != 0;
          const float e0 = __shfl_xor_sync(0xffffffffu, up1 ? d1 : d3, CV / 2);
          const float e1 = __shfl_xor_sync(0xffffffffu, up1 ? d2 : d4, CV / 2);
          const float k0 = (up1 ? d3 : d1) + e0;
          const float k1 = (up1 ? d4 : d2) + e1;
          const bool up2 = (cl & (CV / 4)) != 0;
          const float eb = __shfl_xor_sync(0xffffffffu, up2 ? k0 : k1, CV / 4);
          float k = (up2 ? k1 : k0) + eb;
          k += __shfl_xor_sync(0xffffffffu, k, 1);
          const int back = (lane & (NG - 1)) * CV;
          const float t1 = __shfl_sync(0xffffffffu, k, back);
          const float t2 = __shfl_sync(0xffffffffu, k, back + CV / 4);
          const float t3 = __shfl_sync(0xffffffffu, k, back + CV / 2);
          const float t4 = __shfl_sync(0xffffffffu, k, back + CV / 2 + CV / 4);
          if ((lane / NG) == it) { r1 = t1; r2 = t2; r3 = t3; r4 = t4; }
        }
        {
          const float hh = 1.f - lh, hw = 1.f - lw;
          if (!(meta & 1)) r1 = 0.f;
          if (!(meta & 2)) r2 = 0.f;
          if (!(meta & 4)) r3 = 0.f;
          if (!(meta & 8)) r4 = 0.f;
          const bool ok = (meta & 15) != 0;
          const float ga = ok ? (hh * hw) * r1 + (hh * lw) * r2 + (lh * hw) * r3 + (lh * lw) * r4 : 0.f;
          const float gx = ok ? fW * aw * (hh * (r2 - r1) + lh * (r4 - r3)) : 0.f;
          const float gy = ok ? fH * aw * (hw * (r3 - r1) + lw * (r4 - r2)) : 0.f;
          if (EPI) {
            const float dot = warp_sum(aw * ga);
            if (IDX) {
              red_add_f32(gatt0 + s, aw * (ga - dot));
              red_add_v2(gloc0 + 2 * s, __fdiv_rn(gx, fW), __fdiv_rn(gy, fH));
            } else {
              gatt0[s] = aw * (ga - dot);
              reinterpret_cast<float2*>(gloc0)[s] = make_float2(__fdiv_rn(gx, fW), __fdiv_rn(gy, fH));
            }
          } else {
            gatt0[s] = ga;
            reinterpret_cast<float2*>(gloc0)[s] = make_float2(gx, gy);
          }
        }
      }
      __syncthreads();          // this tile's records are complete (and everyone finished the tile before last)
      // ---- hand-over: warp w adds the records of the pixels it owns; chunk c holds warp c's 32 records
      {
        const float* gw = rec_w + buf * kSlabRecords;
        const unsigned short* gp = rec_p + buf * kSlabRecords;
        const float* gg = go_s + buf * kSlabRecords;
#pragma unroll 4
        for (int c = 0; c < kSlabWarps; ++c) {
          const float wv = gw[c * 32 + lane];
          const unsigned pv = gp[c * 32 + lane];
          unsigned m = __ballot_sync(0xffffffffu, wv != 0.f && (pv & (kSlabWarps - 1)) == (unsigned)warp);
          if (m == 0) continue;
          const float gval = gg[c * 32 + lane];           // lane = channel of the source query's grad_out row
          while (m) {
            const int srcl = __ffs(m) - 1;
            m &= m - 1;
            const float wb = __shfl_sync(0xffffffffu, wv, srcl);
            const unsigned pb = __shfl_sync(0xffffffffu, pv, srcl);
            float* sp = slab + pb * 32 + lane;
            *sp = fmaf(wb, gval, *sp);
          }
        }
      }
    }
    __syncthreads();
    // ---- flush the unit's slab into grad_value[n, start .. start+rows, h, :]
    const int row0 = n * p.K + lv.start;
    if (lv.box_rows > 0) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the TMA
      __syncthreads();
      if (tid == 0) {
        for (int r = 0; r < lv.rows; r += lv.box_rows) tma_reduce_add_2d(&gmap, h * 32, row0 + r, slab + r * 32);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the slab may be overwritten afterwards
      }
    } else {
      float* gs = grad_value + (size_t)row0 * pix + (size_t)h * 32;
      for (int i = tid; i < lv.rows * 8; i += kSlabWarps * 32) {
        const float4 v = reinterpret_cast<const float4*>(slab)[i];
        if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) red_add_v4(gs + (size_t)(i >> 3) * pix + (i & 7) * 4, v);
      }
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------------------------
// forward
// ----------------------------------------------------------------------------------------------
template <bool EPI, bool IDX>
__global__ void __launch_bounds__(kSlabWarps * 32, 2)
msda_forward_slab_kernel(const MsdaParams p, const SlabGeo sg, const __grid_constant__ CUtensorMap vmap,
                         float* __restrict__ out) {
  constexpr int CV = 8, NG = 4, ITERS = 8;
  extern __shared__ __align__(128) unsigned char slab_smem[];
  float* slab = reinterpret_cast<float*>(slab_smem);                       // [kSlabMaxRows + box slack][32]
  __shared__ __align__(8) unsigned long long bar;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane / CV, cl = lane % CV;
  const unsigned pix = (unsigned)p.pix_stride;
  const int units = p.B * p.H * sg.parts;
  const SlabLevel lv = slab_level(p, sg);
  if (lv.box_rows > 0 && tid == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  unsigned phase = 0;

  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int nh = u / sg.parts, part = u % sg.parts;
    const int n = nh / p.H, h = nh % p.H;
    const int row0 = n * p.K + lv.start;
    // ---- stage the head's slab of the coarsest level: [rows][32 floats]
    if (lv.box_rows > 0) {
      if (tid == 0) {
        const int nbox = (lv.rows + lv.box_rows - 1) / lv.box_rows;
        mbar_expect_tx(&bar, (unsigned)(nbox * lv.box_rows * 128));
        for (int b = 0; b < nbox; ++b) tma_load_2d(slab + b * lv.box_rows * 32, &vmap, h * 32, row0 + b * lv.box_rows, &bar);
      }
      mbar_wait(&bar, phase);
      phase ^= 1;
    } else {
      const float* vsrc = p.value + (size_t)row0 * pix + (size_t)h * 32;
      for (int i = tid; i < lv.rows * 8; i += kSlabWarps * 32)
        reinterpret_cast<float4*>(slab)[i] = ldg4(vsrc + (size_t)(i >> 3) * pix + (i & 7) * 4);
      __syncthreads();
    }

    for (int qt = part; qt < sg.tiles; qt += sg.parts) {
      const int q = qt * kSlabWarps + warp;
      const long long item0 = ((long long)n * p.Q + q) * p.H + h;
      Row row;
      if (!(q < p.Q && resolve_row<IDX>(p, item0, row))) continue;
      const long long prow = (EPI && IDX) ? row.dense : item0;
      const float* loc0 = p.loc + (size_t)prow * 64;
      const float* att0 = p.attn + (size_t)prow * 32;
      const float* vb = p.value + slab_offset(p, item0) + cl * 4;
      const float* sb = slab + cl * 4;
      const int s = lane;
      int base = 0, meta = 0;
      float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
      {
        const int l = s / p.P;
        const int Hl = (int)__ldg(p.shapes + 2 * l), Wl = (int)__ldg(p.shapes + 2 * l + 1);
        float2 xy;
        float aw;
        if (EPI) {
          epi_decode(p, row.refrow, s, (float)Wl, (float)Hl, loc0, att0, xy, aw);
        } else {
          xy = __ldg(reinterpret_cast<const float2*>(loc0) + s);
          aw = __ldg(att0 + s);
        }
        float lh, lw;
        decode_sample(xy.x, xy.y, Hl, Wl, (int)__ldg(p.lsi + l), base, meta, lh, lw, p.pix_stride);
        if (meta && (unsigned)(Hl * Wl) * 128u > p.na_bytes) meta |= kHintBit;
        const float hh = 1.f - lh, hw = 1.f - lw;
        w1 = (meta & 1) ? aw * (hh * hw) : 0.f;
        w2 = (meta & 2) ? aw * (hh * lw) : 0.f;
        w3 = (meta & 4) ? aw * (lh * hw) : 0.f;
        w4 = (meta & 8) ? aw * (lh * lw) : 0.f;
      }
      float4 acc = f4_zero();
#pragma unroll
      for (int it = 0; it < ITERS; ++it) {
        const int src = it * NG + g;
        const int sbase = __shfl_sync(0xffffffffu, base, src);
        const int smeta = __shfl_sync(0xffffffffu, meta, src);
        const float a1 = __shfl_sync(0xffffffffu, w1, src);
        const float a2 = __shfl_sync(0xffffffffu, w2, src);
        const float a3 = __shfl_sync(0xffffffffu, w3, src);
        const float a4 = __shfl_sync(0xffffffffu, w4, src);
        if (smeta & 15) {
          const unsigned o1 = (unsigned)sbase;
          const unsigned o2 = o1 + ((smeta & 16) ? pix : 0u);
          const unsigned o3 = o1 + (unsigned)((smeta & ~kHintBit) >> 5);
          const unsigned o4 = o3 + (o2 - o1);
          float4 v1, v2, v3, v4;
          if (it >= lv.first_it) {          // coarsest level: from the staged slab (pixel -> 128-byte row)
            const unsigned sh = (unsigned)sg.pix_shift, st0 = (unsigned)lv.start;
            v1 = *reinterpret_cast<const float4*>(sb + (((o1 >> sh) - st0) << 5));
            v2 = *reinterpret_cast<const float4*>(sb + (((o2 >> sh) - st0) << 5));
            v3 = *reinterpret_cast<const float4*>(sb + (((o3 >> sh) - st0) << 5));
            v4 = *reinterpret_cast<const float4*>(sb + (((o4 >> sh) - st0) << 5));
          } else {
            const bool na = (smeta & kHintBit) != 0;
            v1 = ldg4_h(vb + o1, na);
            v2 = ldg4_h(vb + o2, na);
            v3 = ldg4_h(vb + o3, na);
            v4 = ldg4_h(vb + o4, na);
          }
          f4_fma(acc, a1, v1);
          f4_fma(acc, a2, v2);
          f4_fma(acc, a3, v3);
          f4_fma(acc, a4, v4);
        }
      }
#pragma unroll
      for (int off = CV; off < 32; off <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, off);
        acc.w += __shfl_xor_sync(0xffffffffu, acc.w, off);
      }
      if (g == 0) {
        if (IDX) red_add_v4(out + (size_t)row.dense * 32 + cl * 4, f4_scale(row.inv, acc));
        else *reinterpret_cast<float4*>(out + (size_t)item0 * 32 + cl * 4) = acc;
      }
    }
    __syncthreads();            // every warp is done with this unit's slab before the next one is staged
  }
}
