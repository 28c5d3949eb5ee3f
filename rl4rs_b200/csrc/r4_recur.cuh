// r4_recur.cuh -- the two gated recurrences of the DIEN simulator on the Hopper tensor cores (wgmma):
//   GRU-1, the interest extractor (TF1 GRUCell via deepctr DynamicGRU, nets/utils.py:120), hidden 128, every step's output
//   kept; with hard = 1 the Keras-v1 GRU of the `lstm` simulator (hard sigmoid, last state only);
//   AUGRU, the interest evolution (deepctr VecAttGRUCell, nets/utils.py:123-124), hidden 256, final state only.
//
//   r = sigmoid(Xr_t + h Wr)   u = sigmoid(Xu_t + h Wu)   c = tanh(Xc_t + (r*h) Wc)
//   GRU: h <- u h + (1-u) c          AUGRU: u' = (1 - score_t) u ;  h <- u' h + (1-u') c
//
// One CTA = 64 rows = one consumer warpgroup (the wgmma M) + one producer warp that streams the recurrent weights
// through a 4-stage ring by bulk copy.  The fp32 state h lives in the consumer threads' registers in the wgmma
// accumulator layout, so every gate is element-wise on registers; its bf16 hi/lo copies are the A operands in shared
// memory: h (double buffered: step t reads one while it writes the next) and r*h.  Per step: phase R walks the gate
// columns in chunks of 64 (r -> r*h), phase UC walks them again (u and c -> h').  Products: hi*hi + lo*hi + hi*lo
// (3 bf16 wgmmas per fp32 product, fp32 accumulation): relative error ~2^-16 per term.
#pragma once
#include "r4_augru_tc.cuh"

namespace r4tc {

constexpr int GH = 128;                          // GRU-1 hidden
constexpr int G1_XT_COLS = 3 * GH;               // GRU-1 input halves [r | u | c]
constexpr int RC_ROWS = 64, RC_NC = 64;          // rows per CTA, gate columns per chunk
constexpr int RC_SPLIT = RC_NC * KB * 2;         // 4 KB: one split of a 64-column x 32-K weight block
constexpr int RC_STAGE = 2 * RC_SPLIT;           // ring stage = [hi | lo]
constexpr int RC_NST = 4;
constexpr int RC_THREADS = 160;                  // consumer warpgroup + producer warp

template <int HD> struct Rc {
  static constexpr int NCH = HD / RC_NC, NKB = HD / KB;
  static constexpr int A_SPLIT = RC_ROWS * HD * 2;          // one split of a 64-row operand
  static constexpr int A_SBO = (HD / 8) * 128;              // 8-row groups of an A operand
  static constexpr int STAGES_PER_STEP = 3 * NCH * NKB;
  static constexpr int IMAGE_BYTES = STAGES_PER_STEP * RC_STAGE;
  static constexpr int SMEM_BYTES = 6 * A_SPLIT + RC_NST * RC_STAGE;
  static constexpr int XT_COLS = 3 * HD;
};
constexpr int G1_IMAGE_BYTES = Rc<GH>::IMAGE_BYTES;         // 196608
constexpr int G1_SMEM_BYTES = Rc<GH>::SMEM_BYTES;
constexpr int AU_IMAGE_BYTES = Rc<HID>::IMAGE_BYTES;        // 786432 per sequence
constexpr int AU_SMEM_BYTES = Rc<HID>::SMEM_BYTES;          // 224 KB

// host: Wg [HD k][2 HD = r | u], Wc [HD k][HD] (the h halves of the cell kernels) -> the weight stream of one step, in the
// order the kernel consumes it: phase R (r: chunk, K block), phase UC (per chunk: u K blocks, then c K blocks).
inline void build_recur_image(int HD, const float* Wg, const float* Wc, uint8_t* img) {
  const int nch = HD / RC_NC, nkb = HD / KB;
  size_t off = 0;
  auto stage = [&](int mat, int c, int kb) {
    for (int sp = 0; sp < 2; ++sp)
      for (int nl = 0; nl < RC_NC; ++nl)
        for (int kk = 0; kk < KB; ++kk) {
          const int k = kb * KB + kk, n = c * RC_NC + nl;
          const float w = mat == 0 ? Wg[(size_t)k * 2 * HD + n] : (mat == 1 ? Wg[(size_t)k * 2 * HD + HD + n] : Wc[(size_t)k * HD + n]);
          const uint16_t hi = host_bf16_bits(w);
          const uint16_t v = sp == 0 ? hi : host_bf16_bits(w - host_bf16_val(hi));
          memcpy(img + off + sp * RC_SPLIT + (nl / 8) * B_SBO + (kk / 8) * LBO + (nl % 8) * 16 + (kk % 8) * 2, &v, 2);
        }
    off += RC_STAGE;
  };
  for (int c = 0; c < nch; ++c)
    for (int kb = 0; kb < nkb; ++kb) stage(0, c, kb);
  for (int c = 0; c < nch; ++c) {
    for (int kb = 0; kb < nkb; ++kb) stage(1, c, kb);
    for (int kb = 0; kb < nkb; ++kb) stage(2, c, kb);
  }
}

struct GruTcParams {
  const float* XT;        // [ceil(n/128), steps, 384 / 4, 128, 4]  input halves (+bias), lane-major tiles, quad layout
  const uint8_t* Wimg;    // G1_IMAGE_BYTES (build_recur_image)
  float* H;               // [n, steps, 128] outputs of every step, or nullptr
  int n;
  int steps = STEPS;      // recurrence length (<= 64): 64 for the behaviour sequences, 21 for the `lstm` simulator's category GRU
  int hard = 0;           // 1: Keras v1 GRU gates, hard sigmoid clip(0.2 x + 0.5, 0, 1) (nets/utils.py:34,92); 0: TF1 GRUCell
  float* Hlast = nullptr; // [n, ld_last] the LAST state only (the `lstm` simulator), or nullptr
  int ld_last = GH;
};

__device__ __forceinline__ float gru_gate(float x, int hard) {
  return hard ? fminf(fmaxf(fmaf(0.2f, x, 0.5f), 0.0f), 1.0f) : fast_sigmoid(x);
}

template <int HD, bool AUG>
__device__ __forceinline__ void recur_body(const GruTcParams* gp, const AugruTcParams* ap) {
  using C = Rc<HD>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sH = smem;                          // h operand: 2 buffers x (hi, lo)
  uint8_t* sR = smem + 4 * C::A_SPLIT;         // r*h operand: hi, lo
  uint8_t* sB = smem + 6 * C::A_SPLIT;         // weight ring
  __shared__ uint64_t bar_full[RC_NST], bar_empty[RC_NST];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int steps = AUG ? STEPS : gp->steps;
  const uint8_t* img = AUG ? ap->s[blockIdx.y].Wimg : gp->Wimg;

  if (tid == 0) {
    for (int i = 0; i < RC_NST; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 4) {
    // ===== producer: the step's weight image, stage by stage, once per step =====
    if (lane == 0) {
      int stage = 0; uint32_t ph = 0;
      for (int t = 0; t < steps; ++t)
        for (int i = 0; i < C::STAGES_PER_STEP; ++i) {
          mbar_wait(&bar_empty[stage], ph ^ 1);
          mbar_expect_tx(&bar_full[stage], RC_STAGE);
          bulk_g2s(sB + stage * RC_STAGE, img + (size_t)i * RC_STAGE, RC_STAGE, &bar_full[stage]);
          if (++stage == RC_NST) { stage = 0; ph ^= 1; }
        }
    }
    return;
  }

  // ===== consumer warpgroup: thread (warp w, lane l) owns rows 16 w + l / 4 (+ 8) and column pairs 8 j + 2 (l % 4) =====
  const int g = lane >> 2, tq = lane & 3;
  const int m0 = blockIdx.x * RC_ROWS;
  const float* xrow[2];                        // the row's lane in its input tile, step 0
  const float* srow[2] = {nullptr, nullptr};   // AUGRU: the row's attention scores, step 0
  int rows[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = m0 + warp * 16 + g + 8 * h;
    rows[h] = r;
    if constexpr (AUG) {
      const AugruTcSeq& S = ap->s[blockIdx.y];
      valid[h] = r < ap->R;
      const int rc = min(r, ap->R - 1);
      const int ci = S.shared ? 0 : (ap->row0 + rc) / ap->div;
      xrow[h] = S.XT + (size_t)(ci / TM) * STEPS * C::XT_COLS * TM + (ci % TM) * 4;
      srow[h] = S.scoresT + (size_t)(rc / TM) * STEPS * TM + rc % TM;
    } else {
      valid[h] = r < gp->n;
      const int rc = min(r, gp->n - 1);
      rows[h] = rc;
      xrow[h] = gp->XT + (size_t)(rc / TM) * steps * C::XT_COLS * TM + (rc % TM) * 4;
    }
  }
  // byte offset of (row pair h, column pair of chunk c, j) inside an A operand split
  auto aoff = [&](int h, int c, int jj) -> uint32_t {
    return (uint32_t)(warp * 2 + h) * C::A_SBO + (uint32_t)(c * 8 + jj) * LBO + (uint32_t)g * 16 + (uint32_t)tq * 4;
  };
  auto ldx = [&](const float* base, int col) -> float2 {
    return __ldg(reinterpret_cast<const float2*>(base + (size_t)(col & ~3) * TM + (col & 3)));
  };

  for (int i = tid; i < 2 * C::A_SPLIT / 16; i += 128) reinterpret_cast<uint4*>(sH)[i] = make_uint4(0, 0, 0, 0);   // h0 = 0
  proxy_fence();
  named_bar_sync(1, 128);

  float hreg[C::NCH][32];
#pragma unroll
  for (int c = 0; c < C::NCH; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) hreg[c][i] = 0.f;

  int stage = 0; uint32_t ph = 0;
  // acc (+)= A[64 x HD] . W-chunk[HD x 64] over the next NKB ring stages; a stage is released once its wgmmas are done
  auto gemm = [&](float (&acc)[32], uint32_t aHi, uint32_t aLo) {
    int prev = -1;
    for (int kb = 0; kb < C::NKB; ++kb) {
      mbar_wait(&bar_full[stage], ph);
      wgmma_fence();
      const uint32_t b = smem_u32(sB + stage * RC_STAGE);
#pragma unroll
      for (int j = 0; j < KB / 16; ++j) {
        const uint32_t ko = (uint32_t)(kb * (KB / 16) + j) * 2 * LBO;
        const uint64_t dah = make_desc(aHi + ko, LBO, C::A_SBO), dal = make_desc(aLo + ko, LBO, C::A_SBO);
        const uint64_t dbh = make_desc(b + j * 2 * LBO, LBO, B_SBO), dbl = make_desc(b + RC_SPLIT + j * 2 * LBO, LBO, B_SBO);
        wgmma_m64n64k16(acc, dah, dbh);
        wgmma_m64n64k16(acc, dal, dbh);
        wgmma_m64n64k16(acc, dah, dbl);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&bar_empty[prev]);
      prev = stage;
      if (++stage == RC_NST) { stage = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&bar_empty[prev]);
  };

  const int hard = AUG ? 0 : gp->hard;
  const uint32_t rHi = smem_u32(sR), rLo = rHi + C::A_SPLIT;
  for (int t = 0; t < steps; ++t) {
    const uint32_t hHi = smem_u32(sH + (t & 1) * 2 * C::A_SPLIT), hLo = hHi + C::A_SPLIT;
    uint8_t* nHi = sH + ((t + 1) & 1) * 2 * C::A_SPLIT;
    uint8_t* nLo = nHi + C::A_SPLIT;
    const size_t tso = (size_t)t * C::XT_COLS * TM;
    float oms[2] = {1.f, 1.f};
    if constexpr (AUG) {
#pragma unroll
      for (int h = 0; h < 2; ++h) oms[h] = 1.0f - __ldg(srow[h] + (size_t)t * TM);
    }
    // ---- phase R: r*h -> its operand buffer ----
#pragma unroll
    for (int c = 0; c < C::NCH; ++c) {
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      gemm(acc, hHi, hLo);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = jj * 4 + 2 * h, col = c * RC_NC + jj * 8 + 2 * tq;
          const float2 x = ldx(xrow[h] + tso, col);
          const float v0 = gru_gate(acc[i] + x.x, hard) * hreg[c][i];
          const float v1 = gru_gate(acc[i + 1] + x.y, hard) * hreg[c][i + 1];
          uint32_t hi, lo;
          split2(v0, v1, hi, lo);
          *reinterpret_cast<uint32_t*>(sR + aoff(h, c, jj)) = hi;
          *reinterpret_cast<uint32_t*>(sR + C::A_SPLIT + aoff(h, c, jj)) = lo;
        }
    }
    proxy_fence();
    named_bar_sync(1, 128);
    // ---- phase UC: u, c -> h' (registers, the other h operand buffer, H[t]) ----
#pragma unroll
    for (int c = 0; c < C::NCH; ++c) {
      float au[32], ac[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) { au[i] = 0.f; ac[i] = 0.f; }
      gemm(au, hHi, hLo);
      gemm(ac, rHi, rLo);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = jj * 4 + 2 * h, col = c * RC_NC + jj * 8 + 2 * tq;
          const float2 xu = ldx(xrow[h] + tso, HD + col), xc = ldx(xrow[h] + tso, 2 * HD + col);
          float hn[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float u = gru_gate(au[i + e] + (e ? xu.y : xu.x), hard) * oms[h];
            const float cc = fast_tanh(ac[i + e] + (e ? xc.y : xc.x));
            hn[e] = fmaf(u, hreg[c][i + e] - cc, cc);
            hreg[c][i + e] = hn[e];
          }
          uint32_t hi, lo;
          split2(hn[0], hn[1], hi, lo);
          *reinterpret_cast<uint32_t*>(nHi + aoff(h, c, jj)) = hi;
          *reinterpret_cast<uint32_t*>(nLo + aoff(h, c, jj)) = lo;
          if constexpr (!AUG) {
            if (gp->H && valid[h])
              *reinterpret_cast<float2*>(gp->H + ((size_t)rows[h] * steps + t) * GH + col) = make_float2(hn[0], hn[1]);
          }
        }
    }
    proxy_fence();
    named_bar_sync(1, 128);
  }
  // ---- final state ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!valid[h]) continue;
    float* o;
    if constexpr (AUG) o = ap->s[blockIdx.y].out + (size_t)rows[h] * ap->out_ld;
    else { if (!gp->Hlast) continue; o = gp->Hlast + (size_t)rows[h] * gp->ld_last; }
#pragma unroll
    for (int c = 0; c < C::NCH; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int i = jj * 4 + 2 * h;
        *reinterpret_cast<float2*>(o + c * RC_NC + jj * 8 + 2 * tq) = make_float2(hreg[c][i], hreg[c][i + 1]);
      }
  }
}

// grid: ceil(n / 64) CTAs
__global__ void __launch_bounds__(RC_THREADS, 1) k_gru_tc(const __grid_constant__ GruTcParams p) { recur_body<GH, false>(&p, nullptr); }
// grid: (ceil(R / 64), 2 sequences)
__global__ void __launch_bounds__(RC_THREADS, 1) k_augru_tc(const __grid_constant__ AugruTcParams p) { recur_body<HID, true>(nullptr, &p); }

}  // namespace r4tc
