// Scene-cut detection of a streamed step: the mean absolute frame difference (mafd) of the step's two LR frames,
// quantised to 8-bit codes, and the per-slot decision of oracle/scene_cut.py.  One launch scores every slot; the
// last CTA of each slot takes the decision in float64 and clears the slot's workspace.
// Contract: include/tecogan_b200.h (tg_scene_cut).
#include <math.h>

#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxC = 4;                  // tg_stream_frame_in's channel limit
constexpr int kFloatsPerCta = 4096;       // kThreads x 4 float4: one pass of loads per thread
constexpr int kMaxCtasPerSlot = 256;

// the workspace of one slot (TG_SCENE_CUT_WORK_BYTES): zero between launches
struct SlotWork {
  unsigned long long sad;                 // integer sum of |q(a) - q(b)| over the slot's frame
  unsigned int arrived;                   // CTAs of the slot that have added their partial
  unsigned int pad;
};
static_assert(sizeof(SlotWork) == TG_SCENE_CUT_WORK_BYTES, "workspace size of the header");

// q(x) = clip(rint(x * 255), 0, 255): an fp32 product, round half to even; NaN counts as 0
__device__ __forceinline__ int q8(float x) { return (int)fminf(fmaxf(rintf(__fmul_rn(x, 255.f)), 0.f), 255.f); }
__device__ __forceinline__ unsigned int ad(float a, float b) { return (unsigned int)abs(q8(a) - q8(b)); }

__global__ void __launch_bounds__(kThreads)
scene_cut_kernel(const float* __restrict__ lr_curr, const float* __restrict__ lr_prev, size_t count, int cps,
                 const int32_t* __restrict__ reset, double threshold, double* __restrict__ prev_mafd,
                 SlotWork* __restrict__ work, double* __restrict__ score, int32_t* __restrict__ cut) {
  // lr_curr / lr_prev are written by the frame input just before; work, prev_mafd, score and cut belong to the
  // previous launch until it has finished
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int slot = blockIdx.x / cps, part = blockIdx.x - slot * cps;
  const float* a = lr_curr + (size_t)slot * count;
  const float* b = lr_prev + (size_t)slot * count;
  const size_t worker = (size_t)part * kThreads + t, workers = (size_t)cps * kThreads;
  unsigned long long acc = 0;
  if ((((uintptr_t)a ^ (uintptr_t)b) & 15u) == 0) {
    // both frames at the same offset within 16 bytes: scalar head, 16-byte loads, scalar tail
    size_t head = ((16u - ((uintptr_t)a & 15u)) & 15u) / 4u;
    if (head > count) head = count;
    const size_t n4 = (count - head) / 4, tail0 = head + n4 * 4;
    const float4* a4 = reinterpret_cast<const float4*>(a + head);
    const float4* b4 = reinterpret_cast<const float4*>(b + head);
    size_t i = worker;
    for (; i + workers < n4; i += 2 * workers) {          // two pairs of loads in flight
      const float4 x0 = __ldg(a4 + i), y0 = __ldg(b4 + i);
      const float4 x1 = __ldg(a4 + i + workers), y1 = __ldg(b4 + i + workers);
      acc += ad(x0.x, y0.x) + ad(x0.y, y0.y) + ad(x0.z, y0.z) + ad(x0.w, y0.w) +
             ad(x1.x, y1.x) + ad(x1.y, y1.y) + ad(x1.z, y1.z) + ad(x1.w, y1.w);
    }
    if (i < n4) {
      const float4 x0 = __ldg(a4 + i), y0 = __ldg(b4 + i);
      acc += ad(x0.x, y0.x) + ad(x0.y, y0.y) + ad(x0.z, y0.z) + ad(x0.w, y0.w);
    }
    if (worker < head) acc += ad(__ldg(a + worker), __ldg(b + worker));
    if (worker < count - tail0) acc += ad(__ldg(a + tail0 + worker), __ldg(b + tail0 + worker));
  } else {
    for (size_t i = worker; i < count; i += workers) acc += ad(__ldg(a + i), __ldg(b + i));
  }
  // CTA sum: warp shuffles, then the 8 warp sums; one 64-bit atomic per CTA
  __shared__ unsigned long long warp_sum[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((t & 31) == 0) warp_sum[t >> 5] = acc;
  __syncthreads();
  if (t != 0) return;
  unsigned long long sum = 0;
#pragma unroll
  for (int k = 0; k < kThreads / 32; ++k) sum += warp_sum[k];
  SlotWork* ws = work + slot;
  atomicAdd(&ws->sad, sum);
  __threadfence();
  if (atomicAdd(&ws->arrived, 1u) != (unsigned int)cps - 1) return;
  // the slot's last CTA: every partial has landed
  __threadfence();
  const unsigned long long sad = atomicAdd(&ws->sad, 0ull);
  double pm = prev_mafd[slot], sc = 0.0;
  int ct = 0;
  if (reset != nullptr && __ldg(reset + slot) != 0) {
    pm = -1.0;
  } else {
    // float64(SAD) * 100 / count / 255, in that order, each operation rounded to nearest
    const double mafd = __ddiv_rn(__ddiv_rn(__dmul_rn((double)sad, 100.0), (double)count), 255.0);
    if (pm < 0.0) {
      pm = mafd;
    } else {
      sc = fmin(fmax(fmin(mafd, fabs(__dsub_rn(mafd, pm))), 0.0), 100.0);
      ct = sc >= threshold;
      pm = ct ? -1.0 : mafd;
    }
  }
  prev_mafd[slot] = pm;
  score[slot] = sc;
  cut[slot] = ct;
  ws->sad = 0;                            // zero again for the next launch (graph replays need no memset)
  ws->arrived = 0;
}

}  // namespace

extern "C" int tg_scene_cut(const float* lr_curr, const float* lr_prev, int n, int c, int h, int w,
                            const int32_t* reset, double threshold, double* prev_mafd, void* work, double* score,
                            int32_t* cut, void* stream) {
  const char* name = "scene_cut";
  TG_REQUIRE(lr_curr && lr_prev && prev_mafd && work && score && cut, TG_E_INVALID,
             "%s: null pointer (lr_curr / lr_prev / prev_mafd / work / score / cut)", name);
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size n=%d c=%d h=%d w=%d", name, n, c, h, w);
  TG_REQUIRE(((((uintptr_t)lr_curr | (uintptr_t)lr_prev | (uintptr_t)cut | (uintptr_t)reset) & 3u) == 0) &&
                 ((((uintptr_t)prev_mafd | (uintptr_t)work | (uintptr_t)score) & 7u) == 0),
             TG_E_INVALID, "%s: lr_curr / lr_prev / reset / cut must be 4-byte aligned, prev_mafd / work / score "
             "8-byte aligned", name);
  TG_REQUIRE(isfinite(threshold) && threshold > 0.0 && threshold <= 100.0, TG_E_INVALID,
             "%s: threshold %g outside (0, 100]", name, threshold);
  TG_REQUIRE(c <= kMaxC, TG_E_UNSUPPORTED, "%s: %d channels (at most %d)", name, c, kMaxC);
  const size_t count = (size_t)c * h * w;
  const size_t per_slot = (count + kFloatsPerCta - 1) / kFloatsPerCta;
  const int cps = (int)(per_slot < kMaxCtasPerSlot ? per_slot : kMaxCtasPerSlot);
  const size_t ctas = (size_t)cps * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large (n=%d)", name, n);
  tg_launch(scene_cut_kernel, dim3((unsigned)ctas), dim3(kThreads), 0, (cudaStream_t)stream, lr_curr, lr_prev,
            count, cps, reset, threshold, prev_mafd, static_cast<SlotWork*>(work), score, cut);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}
