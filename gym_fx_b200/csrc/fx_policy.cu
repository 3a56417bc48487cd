// fx_policy.cu -- the policy of the closed loop `decide_action -> env.step` (reference caller loop: app/main.py:57-65,
// with a learned actor-critic in place of strategy.decide_action) as ONE fused sm_90a kernel per step:
//
//     h1 = tanh(obs . W1^T + b1)      obs bf16 [N, KP]   (KP = obs_dim padded to a multiple of 64; written by the env
//     h2 = tanh(h1  . W2^T + b2)                           step kernel next to the float32 row)
//     logits = h2 . Wa^T + ba  (3),  value = h2 . Wv + bv
//     action = argmax(logits + gumbel)          Gumbel-max sample (noise supplied, or counter-based in-kernel)
//     logp   = logits[action] - logsumexp(logits)
//
// Continuous action mode (FX_ACTION_CONTINUOUS, the template parameter CONT): head row 0 is the mean, rows 1 and 2 are
// unused, and the fp32 head bias holds {b_mu, log sigma, 0, b_v} -- the state-independent Gaussian of PPO:
//     mu = h2 . wmu + bmu,  action = mu + sigma * eps   eps ~ N(0, 1) (noise supplied, or Box-Muller in-kernel)
//     logp = -eps^2 / 2 - log sigma - log(2 pi) / 2
// The sample is neither clipped nor squashed: the env step thresholds it (fx_coerce_continuous).  Greedy evaluation
// (launch argument, both modes): the argmax of the logits / the mean, no noise read or generated.
//
// Layer 1 ([N x 900] . [900 x HID]) and layer 2 are real contractions: Hopper warpgroup tensor-core MMAs (wgmma).  The
// hidden width HID (both layers) is a template parameter, 64, 128, 256 (the default policy) or 512.  A 128-env row tile
// is owned by a CLUSTER OF TWO CTAs, each computing HID / 2 of the hidden units of both layers: a CTA alone would stream
// the whole obs tile and all of W1 and W2 from L2 per tile, and only N / 128 SMs would have a tile; the pair halves the
// weight bytes, the MMA and the epilogue work per SM.  Per CTA (shown for HID = 256):
//   warp 8      TMA producer: 128 x 64 obs tiles + 128 x 64 W1 tiles (its half of the hidden units), then for layer 2
//               the 128 x 64 h1 tiles + 128 x 64 W2 tiles, through one 4-stage shared-memory ring (cp.async.bulk.tensor,
//               128-byte swizzle, mbarrier complete_tx);
//   warps 0-7   two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: wgmma.mma_async m64n128k16 (bf16 x bf16
//               -> fp32, both operands K-major from the swizzled ring), accumulators in registers (64 per thread); each
//               warp hands a ring slot back to the producer once its warpgroup's MMAs on it have completed; then the
//               epilogue in the same registers: bias + tanh.
// The two halves of h1 meet in global memory (bf16 [N][256], L2-resident: 32 KB written per CTA, then read back by both
// CTAs of the pair as the K-major A operand of layer 2 through TMA) across a cluster barrier; after layer 2 each CTA
// reduces its 128 columns of h2 against the four head rows, rank 1 hands its partial sums to rank 0 (global scratch,
// second cluster barrier), and rank 0 samples and stores.  No cuBLAS / torch on this path.  Launched with the
// programmatic-dependent-launch attribute: the W1 tiles of the first ring slots are requested before griddepcontrol.wait.
// Other widths change only the N of the MMAs (HID / 2), the accumulators per thread (HID / 4), the W1 / W2 tile rows,
// the layer-2 k-blocks (HID / 64), the h1 row stride and the head loops; at 512 the eight layer-2 k-blocks outrun the
// 4-stage ring, so the later ones are streamed after the cluster barrier (kRefill2), and the kernel runs one CTA per SM.
//
// Separate actor and critic networks (the template parameter SEP): two CTA pairs per tile, blockIdx.x = 4 tile + 2 net
// + rank, net 0 = the actor, 1 = the critic.  Each pair is the kernel above at width HID over its own network's rows
// of the stacked parameters (W1 [2 HID][KP], W2 [2 HID][HID], b1 / b2 [2 HID], actor first; h1 [rows][2 HID], the
// network's HID columns at net HID).  The pairs never talk to each other: the actor pair samples from head rows 0-2
// and stores action / log-prob, the critic pair stores the value of row 3; head_part holds one float4 per row and
// network.  No per-tile hand-over: the actor pair's act_flag would not cover the critic pair's reads of the
// observation slot.
//
// Policy population (launch argument tiles_per_member): M members, each a whole actor-critic of the layout above,
// stacked member-major in every parameter (W1 [M][nets][HID][KP], W2 [M][nets][HID][HID], b1 / b2 [M][nets][HID],
// head_w [M][4][HID], head_b [M][4]).  Member m owns the 128-env tiles [m tiles_per_member, (m + 1) tiles_per_member);
// a CTA takes its member from its tile and reads that member's rows and parameters.  h1, head_part, sampling, noise
// and the tile hand-over are per env row and do not see members.  One member (tiles_per_member >= the tile count) is
// member 0 everywhere: the kernel above.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "fx_policy.cuh"

namespace {

constexpr int kTileM = FX_POLICY_TILE_M;   // env rows per cluster (both CTAs work on the same rows)
constexpr int kWgM = 64;                   // rows per consumer warpgroup (= wgmma M)
constexpr int kBlockK = 64;                // bf16 elements per 128-byte swizzled row
constexpr int kStages = 4;
constexpr int kMmaK = 16;
constexpr uint32_t kABytes = kTileM * kBlockK * 2;    // 16 KB
constexpr int kConsumerThreads = 256;                 // two warpgroups
constexpr int kConsumerWarps = kConsumerThreads / 32;
constexpr int kThreads = kConsumerThreads + 32;       // + the TMA producer warp

struct __align__(8) Barriers {
  unsigned long long full[kStages], empty[kStages];
};

// Everything that depends on the hidden width HID.  Stage sizes 20, 24, 32, 48 KB: every stage stays 1024-byte aligned,
// which the swizzled descriptors assume.
template <int HID>
struct Width {
  static_assert(HID == 64 || HID == 128 || HID == 256 || HID == 512, "policy width");
  static constexpr int kHalfN = HID / 2;                         // hidden units per CTA (= wgmma N)
  static constexpr int kAcc = kHalfN / 2;                        // fp32 accumulators per thread of an m64nN wgmma
  static constexpr uint32_t kBBytes = kHalfN * kBlockK * 2;      // 4, 8, 16, 32 KB
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  // shared memory map (1024-byte aligned base): [stages: A | B] x kStages | head weights | biases | barriers
  static constexpr uint32_t kOffHeadW = kStages * kStageBytes;   // float [4][HID]: Wa[0..2], Wv
  static constexpr uint32_t kOffBias = kOffHeadW + 4 * HID * 4;  // float b1[HID], b2[HID], head bias[4]
  static constexpr uint32_t kOffBar = kOffBias + (2 * HID + 4) * 4;
  static constexpr uint32_t kSmemBytes = kOffBar + sizeof(Barriers) + 1024;  // + slack for the 1024-byte alignment
  // 512: 128 accumulators per thread do not fit the 112 registers of 2 CTAs per SM
  static constexpr int kMinBlocks = HID <= 256 ? 2 : 1;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, unsigned long long* bar, void* dst, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// K-major, 128-byte swizzle wgmma shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor): start address >> 4 in
// bits [0,14), leading byte offset (unused for swizzled K-major) in [16,30), stride byte offset = 1024 B (8 rows x 128 B)
// >> 4 in [32,46), base offset 0 (the ring stages are 1024-byte aligned), layout type SWIZZLE_128B = 1 in [62,64).
// A step of 16 elements along K inside the 128-byte swizzle atom is a 32-byte advance of the start address.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int NACC>
__device__ __forceinline__ void acc_fence(float (&d)[NACC]) {
#pragma unroll
  for (int i = 0; i < NACC; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, bf16 operands from shared memory, fp32 accumulators in registers (N / 2 per
// thread).  Fragment layout of d[i] for thread t of the warpgroup: row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),
// column 8 * (i / 4) + 2 * (t % 4) + i % 2.
template <int N>
__device__ __forceinline__ void wgmma_m64k16(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate);

// The accumulator operands of the asm statement are generated from one list: FX_SEQ<n>(X) expands X(i) for i = 1 .. n - 1
// (operand 0 is written out, so neither list ends in a comma).
#define FX_SEQ16(X) X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15)
#define FX_SEQ32(X) FX_SEQ16(X) X(16) X(17) X(18) X(19) X(20) X(21) X(22) X(23) X(24) X(25) X(26) X(27) X(28) X(29) \
  X(30) X(31)
#define FX_SEQ64(X) FX_SEQ32(X) X(32) X(33) X(34) X(35) X(36) X(37) X(38) X(39) X(40) X(41) X(42) X(43) X(44) X(45) \
  X(46) X(47) X(48) X(49) X(50) X(51) X(52) X(53) X(54) X(55) X(56) X(57) X(58) X(59) X(60) X(61) X(62) X(63)
#define FX_SEQ128(X) FX_SEQ64(X) X(64) X(65) X(66) X(67) X(68) X(69) X(70) X(71) X(72) X(73) X(74) X(75) X(76) X(77)   \
  X(78) X(79) X(80) X(81) X(82) X(83) X(84) X(85) X(86) X(87) X(88) X(89) X(90) X(91) X(92) X(93) X(94) X(95) X(96) \
  X(97) X(98) X(99) X(100) X(101) X(102) X(103) X(104) X(105) X(106) X(107) X(108) X(109) X(110) X(111) X(112)      \
  X(113) X(114) X(115) X(116) X(117) X(118) X(119) X(120) X(121) X(122) X(123) X(124) X(125) X(126) X(127)
#define FX_ACC_REG(i) ", %" #i
#define FX_ACC_OPERAND(i) , "+f"(d[i])
// m64nNk16 with NACC = N / 2 accumulators (%0 .. %NACC-1); desc_a, desc_b and accumulate follow as %IA, %IA+1, %IA+2
#define FX_DEFINE_WGMMA(N, NACC, IA, IB, IP)                                                                            \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_m64k16<N>(float (&d)[NACC], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) { \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IP ", 0;\n\t"                                                \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 "                                            \
                 "{%0" FX_SEQ##NACC(FX_ACC_REG) "}, %" #IA ", %" #IB ", p, 1, 1, 0, 0;\n\t}\n"                          \
                 : "+f"(d[0]) FX_SEQ##NACC(FX_ACC_OPERAND)                                                              \
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate)                                                            \
                 : "memory");                                                                                           \
  }
FX_DEFINE_WGMMA(32, 16, 16, 17, 18)
FX_DEFINE_WGMMA(64, 32, 32, 33, 34)
FX_DEFINE_WGMMA(128, 64, 64, 65, 66)
FX_DEFINE_WGMMA(256, 128, 128, 129, 130)
#undef FX_DEFINE_WGMMA
#undef FX_ACC_OPERAND
#undef FX_ACC_REG
#undef FX_SEQ128
#undef FX_SEQ64
#undef FX_SEQ32
#undef FX_SEQ16

// one ring stage (64 elements of K) of this warpgroup's 64 rows against the CTA's HID / 2 hidden units
template <int HID>
__device__ __forceinline__ void mma_stage(float (&d)[Width<HID>::kAcc], uint32_t stage_addr, int wg, bool first) {
  const uint32_t a = stage_addr + (uint32_t)wg * (kWgM * 128), b = stage_addr + kABytes;  // 64 rows x 128 B per warpgroup
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kBlockK / kMmaK; k++)
    wgmma_m64k16<HID / 2>(d, wgmma_desc(a + k * kMmaK * 2), wgmma_desc(b + k * kMmaK * 2), (first && k == 0) ? 0u : 1u);
  wgmma_commit();
  wgmma_wait_all();
  acc_fence(d);
}

__device__ __forceinline__ float fast_tanh(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// counter-based uniform in (0, 1): a 64-bit mix of (seed, step, env, action index) -- used when no noise tensor is given
__device__ __forceinline__ float hash_uniform(unsigned long long seed, unsigned step, unsigned env, unsigned a) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * ((unsigned long long)step * 0x100000001B3ull + ((unsigned long long)env << 2) + a + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return ((float)(unsigned)(z >> 40) + 0.5f) * (1.0f / 16777216.0f);
}

// cluster barrier with release / acquire semantics: every thread of both CTAs executes it (the same number of times)
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire;" ::: "memory");
}

// log(2 pi) / 2
constexpr float kHalfLog2Pi = 0.918938533204672742f;

// (min 2 CTAs per SM only to cap the registers at 112: a policy CTA then fits next to the one-warp CTAs of an env step
// that is still draining, so its prologue -- barrier init, parameter loads, the first weight tiles -- overlaps the
// step's tail instead of waiting for whole SMs to empty.  HID = 512 needs more registers: one CTA per SM.)
// HID: hidden units of both layers (64, 128, 256 or 512).
// CONT = false: discrete actions (int32, Gumbel-max over 3 logits; noise: float32 [num_envs][3] Gumbel(0,1)).
// CONT = true:  continuous actions (float32, Gaussian; noise: float32 [num_envs] N(0,1)).
// SEP = true:   separate actor and critic networks, two CTA pairs per tile (see the top of the file).
// tiles_per_member: 128-env tiles per population member (see the top of the file).
template <int HID, bool CONT, bool SEP>
__global__ void __launch_bounds__(kThreads, Width<HID>::kMinBlocks)
fx_policy_kernel(const __grid_constant__ CUtensorMap map_obs, const __grid_constant__ CUtensorMap map_w1,
                 const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_h1, const FxPolicyDev pol,
                 const int num_envs, const int k_blocks1, const float* __restrict__ noise, const unsigned long long seed,
                 const unsigned step, void* __restrict__ action_, float* __restrict__ logp, float* __restrict__ value,
                 const int env_begin, const int tile_sync, const int greedy, const int tiles_per_member) {
  using S = Width<HID>;
  constexpr int kHalfN = S::kHalfN, kAcc = S::kAcc;
  constexpr uint32_t kStageBytes = S::kStageBytes, kOffBar = S::kOffBar, kOffHeadW = S::kOffHeadW, kOffBias = S::kOffBias;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  Barriers* bar = reinterpret_cast<Barriers*>(smem + kOffBar);
  float* head_w = reinterpret_cast<float*>(smem + kOffHeadW);
  float* bias = reinterpret_cast<float*>(smem + kOffBias);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = blockIdx.x & 1;                         // which half of the hidden units (cluster = CTA pair)
  const int m0 = env_begin + (blockIdx.x >> (SEP ? 2 : 1)) * kTileM;  // a launch covers the envs [env_begin, num_envs)
  const int n0 = rank * kHalfN;
  // SEP: which network this pair computes; its columns of h1 start at net * HID
  const int net = SEP ? (int)(blockIdx.x >> 1) & 1 : 0;
  constexpr int kNets = SEP ? 2 : 1;
  const int member = (m0 / kTileM) / tiles_per_member;    // population member of this tile
  const int trunk = (member * kNets + net) * HID;          // the network's first row of W1 / W2, first entry of b1 / b2
  const int wrow = trunk + n0;                             // this CTA's first row of W1 / W2
  const int hcol = net * HID + n0;                         // this CTA's first column of h1
  constexpr int kH1Cols = SEP ? 2 * HID : HID;             // h1 row stride
  constexpr int kParts = SEP ? 2 : 1;                      // head_part float4s per row
  const bool actor = !SEP || net == 0, critic = !SEP || net == 1;
  const bool tsync = !SEP && tile_sync;
  const bool producer = warp == kConsumerWarps;
#ifdef FXENV_ENABLE_TIMING  // kernel-chain probe (tools/chain_probe.py): CTA 0 logs {kind, entry, after the wait, exit}
  long long* klog = nullptr;
  if (pol.dbg && blockIdx.x == 0 && threadIdx.x == 0) {
    long long g0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));
    const unsigned long long seqno = atomicAdd(reinterpret_cast<unsigned long long*>(pol.dbg), 1ull);
    klog = pol.dbg + 8 + (seqno % 1024ull) * 4;
    klog[0] = 0; klog[1] = g0;
  }
#endif

  if (producer && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_obs) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w2) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_h1) : "memory");
    for (int s = 0; s < kStages; s++) { mbar_init(&bar->full[s], 1); mbar_init(&bar->empty[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // small fp32 parameters (weights of this launch, not produced by the previous kernel): plain loads
  for (int i = threadIdx.x; i < 4 * HID; i += kThreads) head_w[i] = pol.head_w[member * 4 * HID + i];
  for (int i = threadIdx.x; i < 2 * HID + 4; i += kThreads)
    bias[i] = (i < HID) ? pol.b1[trunk + i] : (i < 2 * HID ? pol.b2[trunk + i - HID] : pol.head_b[member * 4 + i - 2 * HID]);
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;");  // the env step that consumes our actions may get scheduled early
  const int kb2 = HID / kBlockK;             // k-blocks of layer 2 (1, 2, 4, 8)
  const int total = k_blocks1 + kb2;
  // HID = 512: layer 2 has more k-blocks than the ring has stages.  Its W2 tiles are requested in phase 1 only for the
  // stages the ring can hold (the slots of later ones are released by layer-2 MMAs, after the cluster barrier); the rest
  // are streamed in phase 2, each slot handed back by the consumers like in layer 1.
  constexpr bool kRefill2 = HID / kBlockK > kStages;
  const int total1 = k_blocks1 + (kb2 < kStages ? kb2 : kStages);
  // consumer thread -> accumulator rows: warpgroup wg owns tile rows [64 wg, 64 wg + 64), d[i] covers rows r and r + 8
  const int wg = warp >> 2;
  const int r_lo = wg * kWgM + (warp & 3) * 16 + (lane >> 2);
  const int c_lane = 2 * (lane & 3);
  const uint32_t ring = smem_u32(smem);
  float d[kAcc];

  // ================= phase 1: layer 1 (this CTA's HID / 2 hidden units), h1 half -> global =================
  if (producer) {
    if (lane == 0) {  // ===== TMA producer =====
      const int pre = total < kStages ? total : kStages;
      // weight tiles of the first slots do not depend on the previous kernel: request them before the dependency wait
      for (int it = 0; it < pre; it++) {
        unsigned char* st = smem + it * kStageBytes;
        const bool l1 = it < k_blocks1;
        mbar_expect_tx(&bar->full[it], kStageBytes);
        tma_load_2d(l1 ? &map_w1 : &map_w2, &bar->full[it], st + kABytes, (l1 ? it : it - k_blocks1) * kBlockK, wrow);
      }
      if (tsync && step > 0u) {
        // closed loop: this tile's rows are complete once its envs have finished step - 1 (counted by the step kernel,
        // which is resident with us: see FxTileSync) -- no need to wait for the whole step grid to drain
        const int valid = (num_envs - m0 < kTileM) ? num_envs - m0 : kTileM;
        const int need = valid * (int)step;
        const int32_t* cnt = pol.done_cnt + m0 / kTileM;
        int polls = 0, have;
        do {
          asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(have) : "l"(cnt) : "memory");
          if (have >= need) break;
          __nanosleep(64);
        } while (++polls <= (1 << 22) || (atomicAdd(pol.timeouts, 1), false));
        asm volatile("fence.proxy.async;" ::: "memory");  // the rows were written through the generic proxy
      } else {
        asm volatile("griddepcontrol.wait;" ::: "memory");  // the observation rows come from the kernel before us
      }
#ifdef FXENV_ENABLE_TIMING
      if (klog) { long long g1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1)); klog[2] = g1; }
#endif
      for (int it = 0; it < total1; it++) {
        const int s = it % kStages;
        unsigned char* st = smem + s * kStageBytes;
        const bool l1 = it < k_blocks1;
        if (it >= kStages) {
          mbar_wait(&bar->empty[s], ((it / kStages) - 1) & 1);
          mbar_expect_tx(&bar->full[s], kStageBytes);
          tma_load_2d(l1 ? &map_w1 : &map_w2, &bar->full[s], st + kABytes, (l1 ? it : it - k_blocks1) * kBlockK, wrow);
        }
        if (l1) tma_load_2d(&map_obs, &bar->full[s], st, it * kBlockK, m0);
        // (layer 2: the W2 tile is in flight; the h1 tile of the same stage follows in phase 2)
      }
    }
  } else {
    // ===== consumers: layer-1 MMAs, then h1[:, n0 .. n0 + HID / 2) = tanh(D1 + b1) -> bf16, row-major [row][HID] in
    // global memory (the other half comes from the peer CTA); rows beyond the env count are written too (the scratch is
    // padded to whole tiles) and never used
    for (int it = 0; it < k_blocks1; it++) {
      const int s = it % kStages;
      mbar_wait(&bar->full[s], (it / kStages) & 1);
      mma_stage<HID>(d, ring + s * kStageBytes, wg, it == 0);
      if (lane == 0) mbar_arrive(&bar->empty[s]);
    }
    const float* b1 = bias + n0;
    uint32_t* h_lo = reinterpret_cast<uint32_t*>(pol.h1 + (size_t)(m0 + r_lo) * kH1Cols + hcol + c_lane);
    uint32_t* h_hi = h_lo + 8 * kH1Cols / 2;
#pragma unroll
    for (int j = 0; j < kAcc / 4; j++) {
      const float bb0 = b1[8 * j + c_lane], bb1 = b1[8 * j + c_lane + 1];
      __nv_bfloat162 lo = __floats2bfloat162_rn(fast_tanh(d[4 * j] + bb0), fast_tanh(d[4 * j + 1] + bb1));
      __nv_bfloat162 hi = __floats2bfloat162_rn(fast_tanh(d[4 * j + 2] + bb0), fast_tanh(d[4 * j + 3] + bb1));
      h_lo[4 * j] = *reinterpret_cast<uint32_t*>(&lo);
      h_hi[4 * j] = *reinterpret_cast<uint32_t*>(&hi);
    }
    asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy global stores -> the peer's (and our) TMA reads
  }
  cluster_sync();  // both halves of h1 are in global memory (release / acquire at cluster scope)

  // ================= phase 2: layer 2 (this CTA's HID / 2 units of h2), head partial sums =================
  float acc_lo[4] = {0.f, 0.f, 0.f, 0.f}, acc_hi[4] = {0.f, 0.f, 0.f, 0.f};  // rows r_lo and r_lo + 8
  if (producer) {
    if (lane == 0) {
      asm volatile("fence.proxy.async;" ::: "memory");
      for (int j = 0; j < kb2; j++) {  // the A operand of the stages whose W2 tile was requested in phase 1
        const int it = k_blocks1 + j, s = it % kStages;
        if (kRefill2 && j >= kStages) {  // (HID = 512: the W2 tile of a stage past the ring, once its slot is free)
          mbar_wait(&bar->empty[s], ((it / kStages) - 1) & 1);
          mbar_expect_tx(&bar->full[s], kStageBytes);
          tma_load_2d(&map_w2, &bar->full[s], smem + s * kStageBytes + kABytes, j * kBlockK, wrow);
        }
        tma_load_2d(&map_h1, &bar->full[s], smem + s * kStageBytes, net * HID + j * kBlockK, m0);
      }
    }
  } else {
    for (int j = 0; j < kb2; j++) {
      const int it = k_blocks1 + j, s = it % kStages;
      mbar_wait(&bar->full[s], (it / kStages) & 1);
      mma_stage<HID>(d, ring + s * kStageBytes, wg, j == 0);
      if (kRefill2 && j + kStages < kb2 && lane == 0) mbar_arrive(&bar->empty[s]);  // the slot takes k-block j + 4
    }
    const float* b2 = bias + HID + n0;
    // (SEP: both pairs reduce all four rows and each stores only its own; skipping the other network's rows takes a
    // copy of this unrolled loop per network, which at HID = 256 and 512 spills past the register cap)
#pragma unroll
    for (int i = 0; i < kAcc; i++) {
      const int k = n0 + 8 * (i / 4) + c_lane + (i & 1);
      const float h = fast_tanh(d[i] + b2[k - n0]);
      float* a = ((i / 2) & 1) ? acc_hi : acc_lo;
      a[0] = fmaf(h, head_w[k], a[0]);
      if (!CONT) {  // (continuous: rows 1 and 2 are zero and unused)
        a[1] = fmaf(h, head_w[HID + k], a[1]);
        a[2] = fmaf(h, head_w[2 * HID + k], a[2]);
      }
      a[3] = fmaf(h, head_w[3 * HID + k], a[3]);
    }
    // the four lanes of a row hold interleaved columns: a fixed butterfly, so the sum does not depend on timing
#pragma unroll
    for (int q = 0; q < 4; q++) {
      acc_lo[q] += __shfl_xor_sync(0xffffffffu, acc_lo[q], 1);
      acc_hi[q] += __shfl_xor_sync(0xffffffffu, acc_hi[q], 1);
      acc_lo[q] += __shfl_xor_sync(0xffffffffu, acc_lo[q], 2);
      acc_hi[q] += __shfl_xor_sync(0xffffffffu, acc_hi[q], 2);
    }
    if (rank == 1 && (lane & 3) == 0) {
      pol.head_part[(m0 + r_lo) * kParts + net] = make_float4(acc_lo[0], acc_lo[1], acc_lo[2], acc_lo[3]);
      pol.head_part[(m0 + r_lo + 8) * kParts + net] = make_float4(acc_hi[0], acc_hi[1], acc_hi[2], acc_hi[3]);
    }
  }
  cluster_sync();  // rank 1's partial head sums are visible to rank 0
  if (!producer && rank == 0) {
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const int env = m0 + r_lo + 8 * half;
      const float* acc = half ? acc_hi : acc_lo;
      if ((lane & 3) == 0 && env < num_envs) {
        const float4 o = pol.head_part[env * kParts + net];
        const float* hb = bias + 2 * HID;
        // (rank 0's columns first, then rank 1's: a fixed order, so the result does not depend on timing)
        // (SEP: the actor pair samples and stores action / log-prob, the critic pair stores the value)
        if (actor && CONT) {
          const float mu = (acc[0] + o.x) + hb[0], log_std = hb[1];
          float eps = 0.f;  // greedy: the mean
          if (!greedy) {
            if (noise) eps = noise[env];
            else {  // Box-Muller over two counter-based uniforms in (0, 1)
              float sn, cs;
              sincospif(2.f * hash_uniform(seed, step, env, 1), &sn, &cs);
              eps = sqrtf(-2.f * logf(hash_uniform(seed, step, env, 0))) * cs;
            }
          }
          reinterpret_cast<float*>(action_)[env] = fmaf(expf(log_std), eps, mu);
          logp[env] = (-0.5f * eps * eps - log_std) - kHalfLog2Pi;
        } else if (actor) {
          const float l0 = (acc[0] + o.x) + hb[0], l1 = (acc[1] + o.y) + hb[1], l2 = (acc[2] + o.z) + hb[2];
          float g0 = 0.f, g1 = 0.f, g2 = 0.f;  // greedy: the argmax of the logits
          if (!greedy) {
            if (noise) { g0 = noise[(size_t)env * 3]; g1 = noise[(size_t)env * 3 + 1]; g2 = noise[(size_t)env * 3 + 2]; }
            else {
              g0 = -__logf(-__logf(hash_uniform(seed, step, env, 0)));
              g1 = -__logf(-__logf(hash_uniform(seed, step, env, 1)));
              g2 = -__logf(-__logf(hash_uniform(seed, step, env, 2)));
            }
          }
          const float s0 = l0 + g0, s1 = l1 + g1, s2 = l2 + g2;
          int a = 0; float best = s0;  // first maximum wins, like torch.argmax
          if (s1 > best) { best = s1; a = 1; }
          if (s2 > best) { best = s2; a = 2; }
          const float mx = fmaxf(l0, fmaxf(l1, l2));
          const float lse = mx + logf(expf(l0 - mx) + expf(l1 - mx) + expf(l2 - mx));
          reinterpret_cast<int32_t*>(action_)[env] = a;
          logp[env] = (a == 0 ? l0 : (a == 1 ? l1 : l2)) - lse;
        }
        if (critic) value[env] = (acc[3] + o.w) + hb[3];
      }
    }
    if (tsync) {  // the tile's actions are stored: the step kernel's warps of these envs may go
      asm volatile("bar.sync 1, %0;" :: "n"(kConsumerThreads) : "memory");  // the two consumer warpgroups
      if (threadIdx.x == 0) {
        __threadfence();
        asm volatile("st.release.gpu.global.s32 [%0], %1;" :: "l"(pol.act_flag + m0 / kTileM), "r"((int)step + 1) : "memory");
      }
    }
  }
#ifdef FXENV_ENABLE_TIMING
  __syncthreads();
  if (klog) { long long g2; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g2)); klog[3] = g2; }
#endif
}

// fp32 nn.Linear weights [rows][cols] -> bf16 [rows][cols_pad] (zero padded), round-to-nearest-even
__global__ void fx_policy_pack_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, int rows, int cols, int cols_pad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * cols_pad) return;
  const int r = (int)(i / cols_pad), c = (int)(i - (int64_t)r * cols_pad);
  dst[i] = c < cols ? __bfloat16_as_ushort(__float2bfloat16_rn(src[(int64_t)r * cols + c])) : (uint16_t)0;
}

using PolicyKernel = decltype(&fx_policy_kernel<256, false, false>);

// the instantiation of one width, action mode and network layout, with its dynamic shared memory; nullptr for an
// unsupported width
template <bool CONT, bool SEP>
PolicyKernel policy_kernel(int hidden, uint32_t* smem) {
  switch (hidden) {
    case 64: *smem = Width<64>::kSmemBytes; return fx_policy_kernel<64, CONT, SEP>;
    case 128: *smem = Width<128>::kSmemBytes; return fx_policy_kernel<128, CONT, SEP>;
    case 256: *smem = Width<256>::kSmemBytes; return fx_policy_kernel<256, CONT, SEP>;
    case 512: *smem = Width<512>::kSmemBytes; return fx_policy_kernel<512, CONT, SEP>;
    default: *smem = 0; return nullptr;
  }
}

PolicyKernel policy_kernel(int hidden, bool continuous, bool separate, uint32_t* smem) {
  if (separate) return continuous ? policy_kernel<true, true>(hidden, smem) : policy_kernel<false, true>(hidden, smem);
  return continuous ? policy_kernel<true, false>(hidden, smem) : policy_kernel<false, false>(hidden, smem);
}

}  // namespace

cudaError_t fx_policy_pack(const float* src, uint16_t* dst, int rows, int cols, int cols_pad, cudaStream_t stream) {
  const int64_t n = (int64_t)rows * cols_pad;
  fx_policy_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, rows, cols, cols_pad);
  return cudaGetLastError();
}

bool fx_policy_width_ok(int hidden) { return hidden == 64 || hidden == 128 || hidden == 256 || hidden == 512; }

size_t fx_policy_smem_bytes(int hidden) {
  uint32_t smem = 0;
  policy_kernel<false, false>(hidden, &smem);
  return smem;
}

cudaError_t fx_policy_configure() {
  for (int hidden : {64, 128, 256, 512})
    for (bool cont : {false, true})
      for (bool sep : {false, true}) {
        uint32_t smem = 0;
        PolicyKernel k = policy_kernel(hidden, cont, sep, &smem);
        cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
      }
  return cudaSuccess;
}

cudaError_t fx_launch_policy(const CUtensorMap& map_obs, const CUtensorMap& map_w1, const CUtensorMap& map_w2,
                             const CUtensorMap& map_h1, const FxPolicyDev& pol, int hidden, int num_envs, int k_pad,
                             const float* noise, unsigned long long seed, unsigned step, void* action, float* logp,
                             float* value, cudaStream_t stream, int env_begin, int env_end, bool tile_sync, bool continuous,
                             bool greedy, bool separate, int tiles_per_member) {
  uint32_t smem = 0;
  PolicyKernel kernel = policy_kernel(hidden, continuous, separate, &smem);
  if (!kernel || tiles_per_member < 1) return cudaErrorInvalidValue;
  if (env_end < 0) env_end = num_envs;
  if (separate) tile_sync = false;  // the actor pair's act_flag does not cover the critic pair's observation reads
  cudaLaunchConfig_t lc = {};
  // one CTA pair per 128-env tile and network
  lc.gridDim = dim3((separate ? 4 : 2) * ((env_end - env_begin + kTileM - 1) / kTileM));
  lc.blockDim = dim3(kThreads);
  lc.dynamicSmemBytes = smem;
  lc.stream = stream;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  at[1].id = cudaLaunchAttributeClusterDimension;
  at[1].val.clusterDim.x = 2; at[1].val.clusterDim.y = 1; at[1].val.clusterDim.z = 1;
  lc.attrs = at;
  lc.numAttrs = 2;
  return cudaLaunchKernelEx(&lc, kernel, map_obs, map_w1, map_w2, map_h1,
                            pol, env_end, k_pad / kBlockK, noise, seed, step, action, logp, value, env_begin,
                            (tile_sync && pol.act_flag) ? 1 : 0, greedy ? 1 : 0, tiles_per_member);
}
