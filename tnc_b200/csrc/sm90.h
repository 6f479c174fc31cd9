// Hopper (sm_90a) building blocks of the int8 tensor-core engines (crt.cu, ozaki.cu): mbarrier, TMA, wgmma.
//
// Both engines run the same warp-specialised int8 GEMM main loop:
//   warpgroup 0     TMA producer (one thread; cp.async.bulk.tensor 2D, mbarrier complete_tx)
//   warpgroups 1-2  consumers: each owns 64 of the CTA's 128 Bt rows and issues wgmma.m64n256k32.s32.s8.s8 from shared
//                   memory into 128 int32 registers per thread (a 64 x 256 accumulator).
// A stage holds BK K bytes of every operand tile: BK = 128 (one 128-byte swizzle row, SWIZZLE_128B) or BK = 64 (SWIZZLE_64B),
// so that a shallower stage buys a deeper ring in the same shared memory.  The operand planes stay padded to 128 K bytes
// (WG_BKB); a 128-byte block is 128 / BK stages.  Four-product complex form (Br, Bi | -Ai, Ar, Ai):
//   stage = Br (128 rows) | Bi (128 rows) | [-Ai ; Ar ; Ai] (384 rows); per 32-byte K step two wgmmas,
//   Br x [Ar ; Ai]^T and Bi x [-Ai ; Ar]^T, into one accumulator (columns 0-127 real, 128-255 imaginary).
// Three-product form (one plane per operand): stage = B_p (128 rows) | A_p (256 rows); one wgmma per K step.
#pragma once
#include <cstdint>
#include <cuda.h>

namespace tncb {

constexpr int WG_ROWS = 128;                 // Bt rows per CTA tile; TMA box rows
constexpr int WG_BKB = 128;                  // K padding of the operand planes (one 128-byte swizzle row)
constexpr int WG_THREADS = 384;              // producer warpgroup + two consumer warpgroups

// stage layout (bytes): B0 | B1 (four products only) | A; TILE is one 128-row operand tile of BK K bytes (16 or 8 KB)
template <bool KARA, int BK> struct WgStage {
  static_assert(BK == 128 || BK == 64, "a stage is 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B) K bytes deep");
  static constexpr int TILE = WG_ROWS * BK;
  static constexpr int B1 = TILE;
  static constexpr int A = KARA ? TILE : 2 * TILE;
  static constexpr int BYTES = KARA ? 3 * TILE : 5 * TILE;
};

__device__ __forceinline__ uint32_t wg_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wg_mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(wg_smem(bar)), "r"(count));
}
__device__ __forceinline__ void wg_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(wg_smem(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void wg_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(wg_smem(bar)) : "memory");
}
__device__ __forceinline__ void wg_mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t}"
        : "=r"(done) : "r"(wg_smem(bar)), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ void wg_tma_2d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(wg_smem(smem)), "l"(map), "r"(wg_smem(bar)), "r"(c0), "r"(c1) : "memory");
}

// wgmma shared-memory descriptor of a K-major tile with BK-byte rows as TMA writes it with SWIZZLE_<BK>B (8-row groups
// of 8 BK bytes, aligned to that size): LBO unused (1), SBO = 8 BK bytes, layout type 1 (128-byte swizzle) or 2 (64-byte
// swizzle).  A K offset inside the swizzle row is added to the start address.
template <int BK>
__device__ __forceinline__ uint64_t wg_desc(const void* smem) {
  static_assert(BK == 128 || BK == 64, "SWIZZLE_128B or SWIZZLE_64B");
  uint64_t d = 0;
  d |= (uint64_t)((wg_smem(smem) & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((8 * BK) >> 4) << 32;
  d |= (uint64_t)(BK == 128 ? 1 : 2) << 62;
  return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 256] (+)= A[64 x 32] . B[256 x 32]^T, signed int8 operands, int32 accumulators.  Fragment of thread (warp w of the
// warpgroup, lane l): d[4j + 2h + e] is row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e.
__device__ __forceinline__ void wg_mma_s8_m64n256k32(uint32_t (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
      "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
      "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
      "}, %128, %129, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
        "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]),
        "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]),
        "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]),
        "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]),
        "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]),
        "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]),
        "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]),
        "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
      : "l"(da), "l"(db), "r"(accumulate));
}

// Consumer side of the stage ring.  `it` counts stages over the kernel's lifetime (slot it % STAGES, phase (it / STAGES) & 1),
// so an item whose stage count is not a multiple of STAGES simply leaves the next item starting mid-ring.
// The stage just issued is released one stage later (wgmma.wait_group 1), so the tensor core never drains between stages;
// drain() releases the last one before the accumulator is read.
template <int STAGES, bool KARA, int BK>
struct WgRing {
  using Stage = WgStage<KARA, BK>;
  uint8_t* smem; uint64_t* full; uint64_t* empty;
  int it = 0, pending = -1;

  // one stage of this warpgroup's 64 Bt rows (`wg` = 0, 1) against the stage's A operand
  __device__ __forceinline__ void mma_stage(uint32_t (&acc)[128], int wg, bool& first, bool signal) {
    const int s = it % STAGES;
    wg_mbar_wait(&full[s], (it / STAGES) & 1);
    const uint8_t* st = smem + s * Stage::BYTES;
    const uint8_t* b0 = st + wg * 64 * BK;
    const uint8_t* a = st + Stage::A;
    wg_fence();
    if (KARA) {
      const uint64_t d_b = wg_desc<BK>(b0), d_a = wg_desc<BK>(a);
#pragma unroll
      for (int k = 0; k < BK / 32; k++) {
        wg_mma_s8_m64n256k32(acc, d_b + (uint64_t)(k * 2), d_a + (uint64_t)(k * 2), first ? 0u : 1u);   // B_p x A_p
        first = false;
      }
    } else {
      const uint64_t d_br = wg_desc<BK>(b0), d_bi = wg_desc<BK>(b0 + Stage::B1);
      const uint64_t d_x = wg_desc<BK>(a + Stage::TILE), d_y = wg_desc<BK>(a);     // X = [Ar ; Ai], Y = [-Ai ; Ar]
#pragma unroll
      for (int k = 0; k < BK / 32; k++) {
        const uint64_t ko = (uint64_t)(k * 2);    // 32 bytes in 16-byte units
        wg_mma_s8_m64n256k32(acc, d_br + ko, d_x + ko, first ? 0u : 1u);
        first = false;
        wg_mma_s8_m64n256k32(acc, d_bi + ko, d_y + ko, 1u);
      }
    }
    wg_commit();
    wg_wait<1>();
    if (pending >= 0 && signal) wg_mbar_arrive(&empty[pending]);
    pending = s;
    it++;
  }
  __device__ __forceinline__ void drain(bool signal) {
    wg_wait<0>();
    if (pending >= 0 && signal) wg_mbar_arrive(&empty[pending]);
    pending = -1;
  }
};

// Producer side: wait until slot it % STAGES is free, arm its barrier with the stage's bytes.  Returns the stage base.
template <int STAGES, bool KARA, int BK>
__device__ __forceinline__ uint8_t* wg_produce_begin(uint8_t* smem, uint64_t* full, uint64_t* empty, int it) {
  const int s = it % STAGES;
  if (it >= STAGES) wg_mbar_wait(&empty[s], ((it / STAGES) - 1) & 1);
  wg_mbar_expect_tx(&full[s], WgStage<KARA, BK>::BYTES);
  return smem + s * WgStage<KARA, BK>::BYTES;
}

__device__ __forceinline__ void wg_setmaxnreg_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void wg_setmaxnreg_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

// 2D tensor map over K-major int8 planes [rows][kbytes], box 128 rows x BK bytes, BK-byte swizzle (BK = 128 or 64)
template <int BK> int wg_make_map(CUtensorMap* m, void* ptr, uint64_t rows, uint64_t kbytes);

}  // namespace tncb
