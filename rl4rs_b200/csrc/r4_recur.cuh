// r4_recur.cuh -- the two gated recurrences of the DIEN simulator on the Hopper tensor cores (wgmma):
//   GRU-1, the interest extractor (TF1 GRUCell via deepctr DynamicGRU, nets/utils.py:120), hidden 128, every step's output
//   kept; with hard = 1 the Keras-v1 GRU of the `lstm` simulator (hard sigmoid, last state only);
//   AUGRU, the interest evolution (deepctr VecAttGRUCell, nets/utils.py:123-124), hidden 256, final state only.
//
//   r = sigmoid(Xr_t + h Wr)   u = sigmoid(Xu_t + h Wu)   c = tanh(Xc_t + (r*h) Wc)
//   GRU: h <- u h + (1-u) c          AUGRU: u' = (1 - score_t) u ;  h <- u' h + (1-u') c
//
// One CTA = 64 rows = two consumer warpgroups + a producer warpgroup, one thread of which streams the weights (setmaxnreg
// moves the producer's registers to the consumers).  Both consumers hold the same 64 rows (the wgmma M);
// warpgroup w owns gate columns [HD/2 w, HD/2 (w+1)) of r, u, c and h, in chunks of 64 (the wgmma N).  The producer
// streams the recurrent weights through a 6-stage ring by bulk copy; a 16 KB stage holds one 32-deep K block of one
// 64-column chunk for each warpgroup, so both consume the ring in lockstep.  The fp32 state h lives in the consumer
// threads' registers in the wgmma accumulator layout, so every gate is element-wise on registers; its bf16 hi/lo copies
// are the full-K A operands in shared memory that both warpgroups read: h (single buffered) and r*h.
//
// Per step and warpgroup (chunks 0, 1 of HD 256; GRU-1 has one chunk): r0, r1, u0 | c0, u1, c1 | h'.  Each GEMM is
// committed one ring stage at a time and a stage is released as soon as its group retires (RC_LAG groups stay in
// flight), and the gate epilogue of the previous chunk runs in the slots between the stages of the next GEMM, so the
// MUFU / split / store work overlaps the tensor pipe (the first slot waits until only the group just committed is in
// flight, so the previous GEMM's accumulators have retired); the gate inputs are loaded RC_XPF slots ahead.  The
// u GEMMs read only h, so u0 is issued before the r*h barrier.  h' is kept in registers until every h-reading wgmma of
// both warpgroups has retired (a barrier), then written over h.  Products: hi*hi + lo*hi + hi*lo (3 bf16 wgmmas per fp32
// product, fp32 accumulation, K ascending): relative error ~2^-16 per term.
#pragma once
#include <type_traits>
#include "r4_augru_tc.cuh"

namespace r4tc {

constexpr int GH = 128;                          // GRU-1 hidden
constexpr int G1_XT_COLS = 3 * GH;               // GRU-1 input halves [r | u | c]
constexpr int RC_ROWS = 64, RC_NC = 64;          // rows per CTA, gate columns per chunk
constexpr int RC_WGS = 2;                        // consumer warpgroups, each owning half of the gate columns
constexpr int RC_SPLIT = RC_NC * KB * 2;         // 4 KB: one split of a 64-column x 32-K weight block
constexpr int RC_STAGE = RC_WGS * 2 * RC_SPLIT;  // 16 KB ring stage = [warpgroup 0: hi | lo][warpgroup 1: hi | lo]
constexpr int RC_NST = 6;
constexpr int RC_LAG = 2;                        // wgmma groups a warpgroup leaves in flight before it releases a stage
constexpr int RC_XPF = 1;                        // gate inputs are loaded this many ring slots before their epilogue
constexpr int RC_THREADS = (RC_WGS + 1) * 128;   // consumer warpgroups + producer warpgroup (one thread of it streams)
constexpr int RC_REG_CONSUMER = 240, RC_REG_PRODUCER = 24;   // setmaxnreg: 2 x 128 x 240 + 128 x 24 <= 64 K registers
static_assert(RC_LAG < RC_NST, "a warpgroup must release a stage before it waits for the stage's refill");

template <int HD> struct Rc {
  static constexpr int NCH = HD / RC_NC, NCW = NCH / RC_WGS, NKB = HD / KB;
  static constexpr int JPS = 8 / NKB;                       // epilogue column groups (of 8) per ring slot
  static constexpr int A_SPLIT = RC_ROWS * HD * 2;          // one split of a 64-row operand
  static constexpr int A_SBO = (HD / 8) * 128;              // 8-row groups of an A operand
  static constexpr int STAGES_PER_STEP = 3 * NCW * NKB;
  static constexpr int IMAGE_BYTES = STAGES_PER_STEP * RC_STAGE;
  static constexpr int SMEM_BYTES = 4 * A_SPLIT + RC_NST * RC_STAGE;
  static constexpr int XT_COLS = 3 * HD;
  static_assert(NCW == 1 || NCW == 2, "one or two chunks per warpgroup");
};
constexpr int G1_IMAGE_BYTES = Rc<GH>::IMAGE_BYTES;         // 196608
constexpr int G1_SMEM_BYTES = Rc<GH>::SMEM_BYTES;           // 160 KB
constexpr int AU_IMAGE_BYTES = Rc<HID>::IMAGE_BYTES;        // 786432 per sequence
constexpr int AU_SMEM_BYTES = Rc<HID>::SMEM_BYTES;          // 224 KB

// host: Wg [HD k][2 HD = r | u], Wc [HD k][HD] (the h halves of the cell kernels) -> the weight stream of one step, in the
// order the kernel consumes it: GEMMs r0 .. r(NCW-1), u0, then c0, u1, c1 (chunk numbers local to a warpgroup), each as
// its K blocks; a stage holds that K block of warpgroup 0's chunk, then of warpgroup 1's.
inline void build_recur_image(int HD, const float* Wg, const float* Wc, uint8_t* img) {
  const int nkb = HD / KB, ncw = HD / RC_NC / RC_WGS;
  size_t off = 0;
  auto gemm = [&](int mat, int lc) {
    for (int kb = 0; kb < nkb; ++kb) {
      for (int w = 0; w < RC_WGS; ++w) {
        uint8_t* dst = img + off + (size_t)w * 2 * RC_SPLIT;
        const int c = w * ncw + lc;
        for (int sp = 0; sp < 2; ++sp)
          for (int nl = 0; nl < RC_NC; ++nl)
            for (int kk = 0; kk < KB; ++kk) {
              const int k = kb * KB + kk, n = c * RC_NC + nl;
              const float wv = mat == 0 ? Wg[(size_t)k * 2 * HD + n] : (mat == 1 ? Wg[(size_t)k * 2 * HD + HD + n] : Wc[(size_t)k * HD + n]);
              const uint16_t hi = host_bf16_bits(wv);
              const uint16_t v = sp == 0 ? hi : host_bf16_bits(wv - host_bf16_val(hi));
              memcpy(dst + sp * RC_SPLIT + (nl / 8) * B_SBO + (kk / 8) * LBO + (nl % 8) * 16 + (kk % 8) * 2, &v, 2);
            }
      }
      off += RC_STAGE;
    }
  };
  for (int lc = 0; lc < ncw; ++lc) gemm(0, lc);
  gemm(1, 0);
  for (int lc = 0; lc < ncw; ++lc) {
    gemm(2, lc);
    if (lc + 1 < ncw) gemm(1, lc + 1);
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

// Wait until at most N of the warpgroup's wgmma groups are pending, then release the ring stages of the retired ones
// (one arrive per warp).  Every group reads exactly one stage, in ring order.
template <int N>
__device__ __forceinline__ void rc_retire(int& pend, int& rel, uint64_t* bar_empty, int lane) {
  wgmma_wait<N>();
  while (pend > N) {
    if (lane == 0) mbar_arrive(&bar_empty[rel]);
    if (++rel == RC_NST) rel = 0;
    --pend;
  }
}

template <int HD, bool AUG>
__device__ __forceinline__ void recur_body(const GruTcParams* gp, const AugruTcParams* ap) {
  using C = Rc<HD>;
  constexpr int NCW = C::NCW, JPS = C::JPS, NPRE = RC_XPF * JPS < 8 ? RC_XPF * JPS : 8;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sH = smem;                          // h operand: hi, lo
  uint8_t* sR = smem + 2 * C::A_SPLIT;         // r*h operand: hi, lo
  uint8_t* sB = smem + 4 * C::A_SPLIT;         // weight ring
  __shared__ uint64_t bar_full[RC_NST], bar_empty[RC_NST];
  __shared__ uint32_t zero_word;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int steps = AUG ? STEPS : gp->steps;
  const uint8_t* img = AUG ? ap->s[blockIdx.y].Wimg : gp->Wimg;

  if (tid == 0) {
    zero_word = 0;
    for (int i = 0; i < RC_NST; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 4 * RC_WGS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= 4 * RC_WGS) {
    // ===== producer: the step's weight image, stage by stage, once per step =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(RC_REG_PRODUCER));
    if (warp == 4 * RC_WGS && lane == 0) {
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

  // ===== consumer warpgroup wg, warp wq of it: thread (wq, lane l) owns rows 16 wq + l / 4 (+ 8) and, in each of the
  // warpgroup's chunks, column pairs 8 j + 2 (l % 4) =====
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(RC_REG_CONSUMER));
  const int wg = warp >> 2, wq = warp & 3;
  const int g = lane >> 2, tq = lane & 3;
  const int m0 = blockIdx.x * RC_ROWS;
  const float* xrow[2];                        // the row's lane in its input tile, step 0, at the thread's first column
  uint32_t srow[2] = {0, 0};                   // AUGRU: the row's attention scores, step 0 (offset in scoresT)
  int rows[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = m0 + wq * 16 + g + 8 * h;
    rows[h] = r;
    if constexpr (AUG) {
      const AugruTcSeq& S = ap->s[blockIdx.y];
      valid[h] = r < ap->R;
      const int rc = min(r, ap->R - 1);
      const int ci = S.shared ? 0 : (ap->row0 + rc) / ap->div;
      xrow[h] = S.XT + (size_t)(ci / TM) * STEPS * C::XT_COLS * TM + (ci % TM) * 4;
      srow[h] = (uint32_t)(rc / TM) * STEPS * TM + rc % TM;
    } else {
      valid[h] = r < gp->n;
      const int rc = min(r, gp->n - 1);
      rows[h] = rc;
      xrow[h] = gp->XT + (size_t)(rc / TM) * steps * C::XT_COLS * TM + (rc % TM) * 4;
    }
  }
  const int xcol = wg * NCW * RC_NC + 2 * tq;   // a multiple of 4 plus 0 or 2
#pragma unroll
  for (int h = 0; h < 2; ++h) xrow[h] += (size_t)(xcol & ~3) * TM + (xcol & 3);
  // byte offset of (row pair h, column pair j of global chunk c) inside an A operand split
  const uint32_t tofs = (uint32_t)(wq * 2) * C::A_SBO + (uint32_t)g * 16 + (uint32_t)tq * 4;
  auto aoff = [&](int h, int c, int jj) -> uint32_t { return tofs + (uint32_t)h * C::A_SBO + (uint32_t)(c * 8 + jj) * LBO; };
  // the thread's column pair of input column group `col8` (a multiple of 8, relative to the thread's first column)
  // (volatile: the loads stay in the ring slot they are written in; hoisted, they would run the registers out)
  auto ldx = [&](const float* base, int col8) -> float2 {
    float2 v;
    asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(base + (size_t)col8 * TM));
    return v;
  };
  auto colof = [&](int lc, int jj) { return (wg * NCW + lc) * RC_NC + jj * 8 + 2 * tq; };

  for (int i = tid; i < 2 * C::A_SPLIT / 16; i += RC_WGS * 128) reinterpret_cast<uint4*>(sH)[i] = make_uint4(0, 0, 0, 0);   // h0 = 0
  proxy_fence();
  named_bar_sync(1, RC_WGS * 128);

  float hreg[NCW][32];
#pragma unroll
  for (int c = 0; c < NCW; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) hreg[c][i] = 0.f;

  int stage = 0, rel = 0, pend; uint32_t ph = 0;     // pend: groups not yet released, 0 at every step boundary
  // acc = A[64 x HD] . W-chunk[HD x 64] over the next NKB ring stages, one wgmma group per stage; after each group
  // (and the release of what has retired) slot(kb) runs a share of the epilogue of the previous GEMM's chunk.  With
  // `epi` (std::true_type) slot 0 reads that GEMM's accumulators, so its last group must have retired first: only the
  // group just committed stays in flight there.
  auto gemm = [&](float (&acc)[32], uint32_t aHi, uint32_t aLo, auto&& slot, auto epi) {
#pragma unroll
    for (int kb = 0; kb < C::NKB; ++kb) {
      mbar_wait(&bar_full[stage], ph);
      // the slot's A address goes through an opaque 0: otherwise the compiler computes the A descriptors of every K
      // step once and keeps them (64-bit each) live across all GEMMs of the step, which runs the registers out
      const uint32_t a = aHi + (uint32_t)kb * (KB / 16) * 2 * LBO + lds_opaque(&zero_word);
      wgmma_fence();
      const uint32_t b = smem_u32(sB + stage * RC_STAGE + wg * 2 * RC_SPLIT);
#pragma unroll
      for (int j = 0; j < KB / 16; ++j) {
        const uint32_t ko = (uint32_t)j * 2 * LBO;
        const uint64_t dah = make_desc(a + ko, LBO, C::A_SBO), dal = make_desc(a + (aLo - aHi) + ko, LBO, C::A_SBO);
        const uint64_t dbh = make_desc(b + j * 2 * LBO, LBO, B_SBO), dbl = make_desc(b + RC_SPLIT + j * 2 * LBO, LBO, B_SBO);
        wgmma_m64n64k16(acc, dah, dbh, kb + j > 0);   // the first product overwrites acc: +0 + x = x (up to the sign of 0)
        wgmma_m64n64k16(acc, dal, dbh);
        wgmma_m64n64k16(acc, dah, dbl);
      }
      wgmma_commit();
      if (++stage == RC_NST) { stage = 0; ph ^= 1; }
      ++pend;
      if (decltype(epi)::value && kb == 0) rc_retire<1>(pend, rel, bar_empty, lane);
      else rc_retire<RC_LAG>(pend, rel, bar_empty, lane);
      slot(kb);
    }
  };
  auto no_slot = [](int) {};

  const int hard = AUG ? 0 : gp->hard;
  const uint32_t hHi = smem_u32(sH), hLo = hHi + C::A_SPLIT;
  const uint32_t rHi = smem_u32(sR), rLo = rHi + C::A_SPLIT;
  for (int t = 0; t < steps; ++t) {
    pend = 0;
    const size_t tso = (size_t)t * C::XT_COLS * TM;
    float oms[2] = {1.f, 1.f};
    if constexpr (AUG) {
#pragma unroll
      for (int h = 0; h < 2; ++h) oms[h] = 1.0f - __ldg(ap->s[blockIdx.y].scoresT + srow[h] + (uint32_t)t * TM);
    }
    float ar[NCW][32], au[NCW][32], ac[NCW][32];
    float2 xr[NCW][8][2], xu[NCW][8][2], xc[NCW][8][2];

    // ---- phase R: r*h -> its operand buffer ----
    auto ldR = [&](int lc, int jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) xr[lc][jj][h] = ldx(xrow[h] + tso, lc * RC_NC + jj * 8);
    };
    auto epR = [&](int lc, int jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = jj * 4 + 2 * h;
        const float v0 = gru_gate(ar[lc][i] + xr[lc][jj][h].x, hard) * hreg[lc][i];
        const float v1 = gru_gate(ar[lc][i + 1] + xr[lc][jj][h].y, hard) * hreg[lc][i + 1];
        uint32_t hi, lo;
        split2(v0, v1, hi, lo);
        sts32(rHi + aoff(h, wg * NCW + lc, jj), hi);
        sts32(rLo + aoff(h, wg * NCW + lc, jj), lo);
      }
    };
    // ---- phase UC: u, c -> h' (registers; the h operand and H[t] when `store`) ----
    auto ldUC = [&](int lc, int jj) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        xu[lc][jj][h] = ldx(xrow[h] + tso, HD + lc * RC_NC + jj * 8);
        xc[lc][jj][h] = ldx(xrow[h] + tso, 2 * HD + lc * RC_NC + jj * 8);
      }
    };
    auto epUC = [&](int lc, int jj, bool store) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = jj * 4 + 2 * h;
        float hn[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float u = gru_gate(au[lc][i + e] + (e ? xu[lc][jj][h].y : xu[lc][jj][h].x), hard) * oms[h];
          const float cc = fast_tanh(ac[lc][i + e] + (e ? xc[lc][jj][h].y : xc[lc][jj][h].x));
          hn[e] = fmaf(u, hreg[lc][i + e] - cc, cc);
          hreg[lc][i + e] = hn[e];
        }
        if (store) {
          uint32_t hi, lo;
          split2(hn[0], hn[1], hi, lo);
          sts32(hHi + aoff(h, wg * NCW + lc, jj), hi);
          sts32(hLo + aoff(h, wg * NCW + lc, jj), lo);
        }
        if constexpr (!AUG) {
          if (gp->H && valid[h])
            *reinterpret_cast<float2*>(gp->H + ((size_t)rows[h] * steps + t) * GH + colof(lc, jj)) = make_float2(hn[0], hn[1]);
        }
      }
    };
    // loads of the first NPRE column groups of an epilogue (issued one GEMM ahead), then per slot: the loads RC_XPF slots
    // ahead and the slot's own column groups
    auto preR = [&](int lc) {
#pragma unroll
      for (int jj = 0; jj < NPRE; ++jj) ldR(lc, jj);
    };
    auto preUC = [&](int lc) {
#pragma unroll
      for (int jj = 0; jj < NPRE; ++jj) ldUC(lc, jj);
    };
    auto slotR = [&](int lc) {
      return [&, lc](int kb) {
#pragma unroll
        for (int q = 0; q < JPS; ++q) {
          if ((kb + RC_XPF) * JPS + q < 8) ldR(lc, (kb + RC_XPF) * JPS + q);
          epR(lc, kb * JPS + q);
        }
      };
    };
    auto slotUC = [&](int lc) {
      return [&, lc](int kb) {
#pragma unroll
        for (int q = 0; q < JPS; ++q) {
          if ((kb + RC_XPF) * JPS + q < 8) ldUC(lc, (kb + RC_XPF) * JPS + q);
          epUC(lc, kb * JPS + q, false);
        }
      };
    };
    // the last chunk's inputs, loaded under its c GEMM
    auto lastUC = [&](int kb) {
      if (kb == 0) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) ldUC(NCW - 1, jj);
      }
    };

    preR(0);
    gemm(ar[0], hHi, hLo, no_slot, std::false_type{});
    if constexpr (NCW == 2) {
      preR(1);
      gemm(ar[1], hHi, hLo, slotR(0), std::true_type{});
    }
    gemm(au[0], hHi, hLo, slotR(NCW - 1), std::true_type{});
    proxy_fence();
    named_bar_sync(1, RC_WGS * 128);           // r*h complete in both warpgroups
    if constexpr (NCW == 2) {
      preUC(0);
      gemm(ac[0], rHi, rLo, no_slot, std::false_type{});
      gemm(au[1], hHi, hLo, slotUC(0), std::true_type{});
    }
    gemm(ac[NCW - 1], rHi, rLo, lastUC, std::false_type{});       // lastUC only loads inputs
    rc_retire<0>(pend, rel, bar_empty, lane);
    named_bar_sync(1, RC_WGS * 128);           // every h-reading wgmma of the step has retired: h' may overwrite h
    if constexpr (NCW == 2) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = jj * 4 + 2 * h;
          uint32_t hi, lo;
          split2(hreg[0][i], hreg[0][i + 1], hi, lo);
          sts32(hHi + aoff(h, wg * NCW, jj), hi);
          sts32(hLo + aoff(h, wg * NCW, jj), lo);
        }
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      if (jj < 4) ldUC(NCW - 1, jj + 4);
      epUC(NCW - 1, jj, true);
    }
    proxy_fence();
    named_bar_sync(1, RC_WGS * 128);
  }
  // ---- final state ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!valid[h]) continue;
    float* o;
    if constexpr (AUG) o = ap->s[blockIdx.y].out + (size_t)rows[h] * ap->out_ld;
    else { if (!gp->Hlast) continue; o = gp->Hlast + (size_t)rows[h] * gp->ld_last; }
#pragma unroll
    for (int c = 0; c < NCW; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int i = jj * 4 + 2 * h;
        *reinterpret_cast<float2*>(o + colof(c, jj)) = make_float2(hreg[c][i], hreg[c][i + 1]);
      }
  }
}

// grid: ceil(n / 64) CTAs
__global__ void __launch_bounds__(RC_THREADS, 1) k_gru_tc(const __grid_constant__ GruTcParams p) { recur_body<GH, false>(&p, nullptr); }
// grid: (ceil(R / 64), 2 sequences)
__global__ void __launch_bounds__(RC_THREADS, 1) k_augru_tc(const __grid_constant__ AugruTcParams p) { recur_body<HID, true>(nullptr, &p); }

}  // namespace r4tc
