// Device-resident proposal selection, sorting and NMS.
//
// The reference does these steps with ~10 tiny ATen kernels plus a device->host copy of the NMS mask
// and a serial host loop per call (upstream csrc/cuda/nms.cu), seven times per frame.  Here every step
// stays on the device (fixed capacities, device-side counts), so the whole detection stage is
// capturable in a CUDA graph.  Every job is latency bound, so each is split so that the quadratic / linear
// work spreads over many SMs, all repeated passes run out of shared memory, and only O(n) bookkeeping is
// serial:
//
//   sort + NMS   : nms_sort_kernel   (1 CTA / problem)  64-bit keys (score key << 32 | ~index), bitonic sort
//                                    (or a stable compaction when the rows already arrive in order)
//                  nms_mask_kernel   (one 64-thread CTA per 64x64 tile of the upper triangle) IoU(+1) bitmask
//                  nms_reduce_kernel (1 CTA / problem)  bitmask staged in shared memory; 64 sorted rows per round:
//                                    branch-free serial resolve by one thread + CTA-wide OR of the survivors' rows
//   RPN top-k    : rpn_local_topk_kernel (1 CTA / ~10k anchors) keys staged once in shared memory, exact local
//                                        top-k by radix select (11-bit digits, parallel threshold search)
//                  rpn_merge_kernel      (1 CTA / level) top-k of the local winners, sort, anchor synthesis +
//                                        BoxCoder decode + clip  (rpn_patch.py:15-52)
//                  rpn_final_kernel      cross-level top-n by rank (each level is already sorted)
//   box_decode_kernel: softmax + per-class decode + clip + track-row rule (inference.py:58-110).
#include "common.cuh"

namespace smot {

constexpr int SN_THREADS = 1024;
constexpr int SN_MAX = 4096;
constexpr int SN_CACHE_BYTES = 176 * 1024;  // largest bitmask nms_reduce_kernel stages in shared memory
constexpr float BBOX_XFORM_CLIP = 4.135166556742356f;  // log(1000/16)

struct SortNmsArgs {
  const float* boxes;
  int box_stride;
  const float* scores;
  int score_stride;
  const int* count;
  int n_max, np;  // np = power of two >= n_max
  float min_score, thresh;
  int max_keep, tag, append, fill_tail;
  int presorted;    // rows arrive in (score desc, index asc) order: nms_sort_kernel only drops rows <= min_score
  int cache_pitch;  // > 0: nms_reduce_kernel stages the bitmask in shared memory with this row pitch (words)
  int* out_index;
  float* out_boxes;
  float* out_scores;
  int* out_tag;
  int* out_count;
  // workspace (per problem p): sorted boxes / original indices / number of candidates / bitmask
  float4* s_boxes;             // [P][n_max]
  int* s_index;                // [P][n_max]
  int* s_m;                    // [P]
  unsigned long long* mask;    // [P][n_max][words_max], words_max = ceil(n_max / 64)
  unsigned long long* diag_t;  // [P][n_max] transposed diagonal blocks: bit b of row i <=> row 64*(i/64)+b < i suppresses i
  int words_max;
  // batching (blockIdx = problem): element offsets added per problem
  int in_step, out_step;
  // segments (smot_sort_nms_segmented): seg > 0 classes per image; problem p is class p % seg of image p / seg, whose rows
  // start at image * in_step rows + class * cls_*_step elements, bounded by count[image].  0: problem p is rows p * in_step...
  int seg = 0, cls_box_step = 0, cls_score_step = 0;
};

// first box / score of problem `prob` and the index of its count.  SEG (compile time) = the segmented addressing; the other
// instantiations are the unsegmented kernels as they were before segments existed.
template <bool SEG> __device__ __forceinline__ int sn_image(const SortNmsArgs& a, int prob) { return SEG ? prob / a.seg : prob; }
template <bool SEG> __device__ __forceinline__ const float* sn_boxes(const SortNmsArgs& a, int prob) {
  if (!SEG) return a.boxes + (size_t)prob * a.in_step * a.box_stride;
  const int img = prob / a.seg, cls = prob - img * a.seg;
  return a.boxes + (size_t)img * a.in_step * a.box_stride + (size_t)cls * a.cls_box_step;
}
template <bool SEG> __device__ __forceinline__ const float* sn_scores(const SortNmsArgs& a, int prob) {
  if (!SEG) return a.scores + (size_t)prob * a.in_step * a.score_stride;
  const int img = prob / a.seg, cls = prob - img * a.seg;
  return a.scores + (size_t)img * a.in_step * a.score_stride + (size_t)cls * a.cls_score_step;
}

// one compare-exchange pair per thread and stage
__device__ __forceinline__ void bitonic_sort_desc(unsigned long long* keys, int np) {
  for (int k = 2; k <= np; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (np >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), p = i | j;
        const unsigned long long a = keys[i], b = keys[p];
        const bool desc = (i & k) == 0;
        if (desc ? (a < b) : (a > b)) {
          keys[i] = b;
          keys[p] = a;
        }
      }
      __syncthreads();
    }
  }
}

// ---- K1: order the candidates -----------------------------------------------------------------
template <bool SEG>
__global__ void __launch_bounds__(SN_THREADS) nms_sort_kernel(SortNmsArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
  __shared__ int s_cnt;
  __shared__ int wcnt[SN_THREADS / 32];
  const int prob = blockIdx.x;
  const float* boxes = sn_boxes<SEG>(a, prob);
  const float* scores = sn_scores<SEG>(a, prob);
  const int n = a.count ? min(a.count[sn_image<SEG>(a, prob)], a.n_max) : a.n_max;
  float4* sb = a.s_boxes + (size_t)prob * a.n_max;
  int* si = a.s_index + (size_t)prob * a.n_max;
  if (a.presorted) {
    // stable compaction of the rows with score > min_score
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = 0;
    for (int i0 = 0; i0 < n; i0 += SN_THREADS) {  // block-uniform trip count
      const int i = i0 + threadIdx.x;
      const bool valid = i < n && scores[(size_t)i * a.score_stride] > a.min_score;
      const unsigned bal = __ballot_sync(0xffffffffu, valid);
      if (lane == 0) wcnt[warp] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < SN_THREADS / 32; ++w) {
        const int c = wcnt[w];
        total += c;
        before += w < warp ? c : 0;
      }
      if (valid) {
        const int pos = base + before + __popc(bal & ((1u << lane) - 1u));
        const float* b = boxes + (size_t)i * a.box_stride;
        sb[pos] = make_float4(b[0], b[1], b[2], b[3]);
        si[pos] = i;
      }
      base += total;
      __syncthreads();
    }
    if (threadIdx.x == 0) a.s_m[prob] = base;
    return;
  }
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  int local = 0;
  for (int i = threadIdx.x; i < a.np; i += blockDim.x) {
    unsigned long long key = 0ull;
    if (i < n) {
      float s = scores[(size_t)i * a.score_stride];
      if (s > a.min_score) {
        key = ((unsigned long long)float_key(s) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
        ++local;
      }
    }
    keys[i] = key;
  }
  if (local) atomicAdd(&s_cnt, local);
  __syncthreads();
  bitonic_sort_desc(keys, a.np);
  const int m = s_cnt;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const unsigned idx = 0xFFFFFFFFu - (unsigned)(keys[i] & 0xFFFFFFFFull);
    const float* b = boxes + (size_t)idx * a.box_stride;
    sb[i] = make_float4(b[0], b[1], b[2], b[3]);
    si[i] = (int)idx;
  }
  if (threadIdx.x == 0) a.s_m[prob] = m;
}

// ---- K2: suppression bitmask, mask[i][w] bit b set <=> j = 64w+b > i and IoU(i,j) > thresh -------
//      grid (column block w, row block, problem), upper triangle only; thread = row i of the tile, the 64
//      column boxes are broadcast from shared memory.  Words left of the diagonal are never written or read.
//      Diagonal tiles also emit the transposed word diag_t[i] (bit b <=> row 64*(i/64)+b < i suppresses i; the
//      IoU test is symmetric bit for bit), which lets nms_reduce_kernel resolve a 64-row block in parallel.
__global__ void __launch_bounds__(64) nms_mask_kernel(SortNmsArgs a) {
  __shared__ float4 cbox[64];
  const int cb = blockIdx.x, rb = blockIdx.y, prob = blockIdx.z;
  if (cb < rb) return;
  const int m = a.s_m[prob];
  if ((cb << 6) >= m) return;
  const float4* __restrict__ sb = a.s_boxes + (size_t)prob * a.n_max;
  const int j0 = cb << 6, i = (rb << 6) + threadIdx.x;
  cbox[threadIdx.x] = j0 + threadIdx.x < m ? sb[j0 + threadIdx.x] : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  if (i >= m) return;
  const float4 bi = sb[i];
  const int jn = min(64, m - j0);
  const bool diag = cb == rb;
  unsigned long long word = 0ull, tword = 0ull;
  for (int b = 0; b < jn; ++b) {
    if (diag && b == (int)threadIdx.x) continue;
    const float4 bj = cbox[b];
    // disjoint boxes have IoU 0: skip the division (same result, most pairs are disjoint)
    if (fminf(bi.z, bj.z) - fmaxf(bi.x, bj.x) + 1.f > 0.f && fminf(bi.w, bj.w) - fmaxf(bi.y, bj.y) + 1.f > 0.f)
      if (iou_plus1(bi, bj) > a.thresh) {
        if (!diag || b > (int)threadIdx.x) word |= 1ull << b; else tword |= 1ull << b;
      }
  }
  a.mask[((size_t)prob * a.n_max + i) * a.words_max + cb] = word;
  if (diag) a.diag_t[(size_t)prob * a.n_max + i] = tword;
}

// ---- K3: greedy reduction + outputs ------------------------------------------------------------
template <bool SEG>
__global__ void __launch_bounds__(SN_THREADS) nms_reduce_kernel(SortNmsArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* kept_all = reinterpret_cast<int*>(smem_raw);                                        // sorted row of the k-th survivor, [np]
  unsigned long long* dT = reinterpret_cast<unsigned long long*>(smem_raw + (size_t)a.np * 4);  // transposed diagonal words, [np]
  unsigned long long* cache = dT + a.np;                                                   // staged bitmask (cache_pitch > 0)
  __shared__ unsigned long long removed[SN_MAX / 64];
  __shared__ unsigned long long s_km;
  __shared__ int s_kept, s_base, s_done;
  const int prob = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* scores = sn_scores<SEG>(a, prob);
  const float4* __restrict__ sb = a.s_boxes + (size_t)prob * a.n_max;
  const int* __restrict__ si = a.s_index + (size_t)prob * a.n_max;
  const unsigned long long* gmask = a.mask + (size_t)prob * a.n_max * a.words_max;
  int* out_count = a.out_count + prob;
  const int m = a.s_m[prob];
  const int words = (m + 63) >> 6;
  if (threadIdx.x == 0) s_kept = 0, s_done = 0;
  for (int i = threadIdx.x; i < SN_MAX / 64; i += blockDim.x) removed[i] = 0ull;
  int kept_total;
  if (a.thresh <= 0.f || a.max_keep <= 0) {
    __syncthreads();
    kept_total = max(min(m, a.max_keep), 0);
    for (int i = threadIdx.x; i < kept_total; i += blockDim.x) kept_all[i] = i;
  } else {
    // everything the rounds below touch goes to shared memory first (the bitmask when it fits): the rounds are a
    // dependent chain and must not wait for global loads
    for (int i = threadIdx.x; i < m; i += blockDim.x) dT[i] = a.diag_t[(size_t)prob * a.n_max + i];
    const unsigned long long* M = gmask;
    int pitch = a.words_max;
    if (a.cache_pitch > 0) {
      for (int idx = threadIdx.x; idx < m * words; idx += blockDim.x) {
        const int row = idx / words, w = idx - row * words;
        if (w > (row >> 6)) cache[row * a.cache_pitch + w] = gmask[(size_t)row * a.words_max + w];
      }
      M = cache;
      pitch = a.cache_pitch;
    }
    __syncthreads();
    // 64 sorted rows per round.  (A) warp 0 resolves the block by fixed-point iteration: a row whose in-block
    // suppressors are all removed is kept, a row with a kept suppressor is removed; the lowest undecided row always
    // decides, so this is the greedy result, in (dependency depth) steps instead of 64.  (B) warp w ORs the
    // survivors' rows of bitmask word c+1+w into `removed` (no atomics: one warp per word).
    for (int c = 0; c < words; ++c) {
      if (warp == 0) {
        const int rows_here = min(64, m - (c << 6));
        const unsigned long long vm = rows_here == 64 ? ~0ull : ((1ull << rows_here) - 1ull);
        unsigned long long rem = removed[c] & vm, kept = 0ull, und = vm & ~rem;
        const unsigned long long sup0 = lane < rows_here ? dT[(c << 6) + lane] : 0ull;
        const unsigned long long sup1 = lane + 32 < rows_here ? dT[(c << 6) + 32 + lane] : 0ull;
        while (und) {
          const bool u0 = (und >> lane) & 1ull, u1 = (und >> (lane + 32)) & 1ull;
          const bool r0 = u0 && (sup0 & kept), r1 = u1 && (sup1 & kept);
          const bool k0 = u0 && !r0 && (sup0 & ~rem) == 0ull, k1 = u1 && !r1 && (sup1 & ~rem) == 0ull;
          const unsigned long long nk = (unsigned long long)__ballot_sync(0xffffffffu, k0) |
                                        ((unsigned long long)__ballot_sync(0xffffffffu, k1) << 32);
          const unsigned long long nr = (unsigned long long)__ballot_sync(0xffffffffu, r0) |
                                        ((unsigned long long)__ballot_sync(0xffffffffu, r1) << 32);
          kept |= nk, rem |= nr, und &= ~(nk | nr);
        }
        if (lane == 0) {
          const int base = s_kept, room = a.max_keep - base;
          int nk = __popcll(kept);
          if (nk >= room) {
            for (; nk > room; --nk) kept &= ~(1ull << (63 - __clzll((long long)kept)));
            s_done = 1;
          }
          s_km = kept;
          s_base = base;
          s_kept = base + nk;
        }
      }
      __syncthreads();
      const unsigned long long km = s_km;
      if (threadIdx.x < 64 && ((km >> threadIdx.x) & 1ull))
        kept_all[s_base + __popcll(km & ((1ull << threadIdx.x) - 1ull))] = (c << 6) + threadIdx.x;
      if (s_done) break;
      for (int w = c + 1 + warp; w < words; w += SN_THREADS / 32) {
        unsigned long long v = 0ull;
        if ((km >> lane) & 1ull) v = M[(size_t)((c << 6) + lane) * pitch + w];
        if ((km >> (lane + 32)) & 1ull) v |= M[(size_t)((c << 6) + 32 + lane) * pitch + w];
        const unsigned lo = __reduce_or_sync(0xffffffffu, (unsigned)v), hi = __reduce_or_sync(0xffffffffu, (unsigned)(v >> 32));
        if (lane == 0) removed[w] |= ((unsigned long long)hi << 32) | lo;
      }
      __syncthreads();
    }
    __syncthreads();
    kept_total = s_kept;
  }
  __syncthreads();
  const int base = a.append ? *out_count : 0;
  const int out_off = prob * a.out_step + base;
  for (int k = threadIdx.x; k < kept_total; k += blockDim.x) {
    const int row = kept_all[k];
    const int idx = si[row];
    if (a.out_index) a.out_index[out_off + k] = idx;
    if (a.out_boxes) reinterpret_cast<float4*>(a.out_boxes)[out_off + k] = sb[row];
    if (a.out_scores) a.out_scores[out_off + k] = scores[(size_t)idx * a.score_stride];
    if (a.out_tag) a.out_tag[out_off + k] = a.tag;
  }
  // rows [kept, fill_tail) of this problem's output slot are marked invalid (score -1)
  if (a.fill_tail > 0 && a.out_scores)
    for (int i = kept_total + threadIdx.x; i < a.fill_tail - base; i += blockDim.x) a.out_scores[out_off + i] = -1.f;
  __syncthreads();
  if (threadIdx.x == 0) *out_count = base + kept_total;
}

static int next_pow2(int n) {
  int p = 64;
  while (p < n) p <<= 1;
  return p;
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static size_t sort_nms_ws_bytes(int problems, int n_max) {
  const size_t P = (size_t)problems, n = (size_t)n_max, words = (n + 63) / 64;
  return align256(P * n * 16) + align256(P * n * 4) + align256(P * 4) + align256(P * n * 8) + align256(P * n * words * 8);
}

static void carve_sort_nms_ws(SortNmsArgs& a, void* ws, int problems) {
  const size_t P = (size_t)problems, n = (size_t)a.n_max;
  unsigned char* w = (unsigned char*)ws;
  a.s_boxes = (float4*)w;            w += align256(P * n * 16);
  a.s_index = (int*)w;               w += align256(P * n * 4);
  a.s_m = (int*)w;                   w += align256(P * 4);
  a.diag_t = (unsigned long long*)w; w += align256(P * n * 8);
  a.mask = (unsigned long long*)w;
  a.words_max = (a.n_max + 63) / 64;
}

static int launch_sort_nms(SortNmsArgs& a, int problems, cudaStream_t st) {
  a.np = next_pow2(a.n_max);
  SMOT_ENSURE_SMEM(nms_sort_kernel<false>, SN_MAX * 8, "sort_nms(sort)");
  SMOT_ENSURE_SMEM(nms_reduce_kernel<false>, SN_MAX * 12 + SN_CACHE_BYTES, "sort_nms(reduce)");
  SMOT_ENSURE_SMEM(nms_sort_kernel<true>, SN_MAX * 8, "sort_nms(sort)");
  SMOT_ENSURE_SMEM(nms_reduce_kernel<true>, SN_MAX * 12 + SN_CACHE_BYTES, "sort_nms(reduce)");
  const bool seg = a.seg > 0;
  // the bitonic network has np/2 compare-exchanges per stage: a smaller CTA makes its ~50 barriers cheaper
  const int sort_threads = a.presorted ? SN_THREADS : (a.np / 2 < 128 ? 128 : (a.np / 2 > SN_THREADS ? SN_THREADS : a.np / 2));
  if (seg)
    nms_sort_kernel<true><<<problems, sort_threads, a.presorted ? 0 : (size_t)a.np * 8, st>>>(a);
  else
    nms_sort_kernel<false><<<problems, sort_threads, a.presorted ? 0 : (size_t)a.np * 8, st>>>(a);
  SMOT_CHECK_LAUNCH("sort_nms(sort)");
  const bool suppress = a.thresh > 0.f && a.max_keep > 0;
  a.cache_pitch = 0;
  size_t cache_bytes = 0;
  if (suppress) {
    const int blocks = (a.n_max + 63) / 64;
    nms_mask_kernel<<<dim3(blocks, blocks, problems), 64, 0, st>>>(a);
    SMOT_CHECK_LAUNCH("sort_nms(mask)");
    const int pitch = a.words_max | 1;  // odd pitch: a column of 64-bit words spreads over all banks
    if ((size_t)a.n_max * pitch * 8 <= (size_t)SN_CACHE_BYTES) a.cache_pitch = pitch, cache_bytes = (size_t)a.n_max * pitch * 8;
  }
  if (seg)
    nms_reduce_kernel<true><<<problems, SN_THREADS, (size_t)a.np * 12 + cache_bytes, st>>>(a);
  else
    nms_reduce_kernel<false><<<problems, SN_THREADS, (size_t)a.np * 12 + cache_bytes, st>>>(a);
  SMOT_CHECK_LAUNCH("sort_nms(reduce)");
  return SMOT_OK;
}

// ---------------------------------------------------------------------------------------------
// RPN: per-level top-k by objectness logit + decode
// ---------------------------------------------------------------------------------------------
constexpr int RPN_CHUNK = 10752;   // anchors per local-top-k CTA (level 0 of a 704x1280 frame = 16 chunks)
constexpr int RPN_MAX_CHUNKS = 256;
constexpr int RPN_IDX_BITS = 22;   // anchors per level < 4M
constexpr int RPN_KEY_BITS = 32 + RPN_IDX_BITS;
constexpr unsigned long long RPN_IDX_MASK = (1ull << RPN_IDX_BITS) - 1ull;
constexpr int RPN_MERGE_SMEM_KEYS = 20 * 1024;  // local winners rpn_merge_kernel stages in shared memory (160 KB)

struct RpnArgs {
  smot_rpn_level lv[SMOT_MAX_LEVELS];
  int num_levels;
  int pre_nms_top_n;  // <= 1024
  int post_nms_top_n, final_top_n;
  float min_size;
  int img_w, img_h, amodal;
  int nchunks;
  int chunk_first[SMOT_MAX_LEVELS + 1];  // chunks of level l are [chunk_first[l], chunk_first[l+1])
  int merge_in_smem;                     // every level's local winners fit RPN_MERGE_SMEM_KEYS
  unsigned long long* local;             // [nchunks][1024] composite keys of the local winners (0 = empty)
  float* cand_boxes;                     // [levels][pre_nms_top_n][4]
  float* cand_scores;                    // [levels][pre_nms_top_n]
  int* cand_count;                       // [levels]
  const float* kept_boxes;               // [levels][post_nms_top_n][4]  per-level NMS survivors, score order
  const float* kept_scores;              // [levels][post_nms_top_n]
  const int* kept_count;                 // [levels]
  float* out_boxes;
  float* out_scores;
  int* out_count;
  // smot_rpn_select_batched (the kernels' BATCHED instantiations): image blockIdx.y reads its heads at lv[l].head + y *
  // head_img_stride[l] and owns image slices of every array above ([image][...]).  Unread by smot_rpn_select's instantiations.
  long long head_img_stride[SMOT_MAX_LEVELS];
};

// composite key: (objectness logit as monotone u32) << 22 | (2^22 - 1 - anchor index in the level): unique, and
// descending key order = (logit desc, anchor index asc)
__device__ __forceinline__ unsigned long long rpn_key(float logit, int g) {
  return ((unsigned long long)float_key(logit) << RPN_IDX_BITS) | (RPN_IDX_MASK - (unsigned long long)g);
}

// Exact top-k of n UNIQUE keys of RPN_KEY_BITS bits by radix select (11-bit digits, MSB first); keys[] (shared or
// global memory) holds 0 for "absent".  The k winners go to out[0..k) in arbitrary order, out[k..1024) = 0.
// All threads of the CTA (1024) must call this; n, k uniform; k <= 1024.
__device__ void select_topk_u64(const unsigned long long* keys, int n, int k, unsigned long long* out) {
  constexpr int DIGIT = 11, BINS = 1 << DIGIT;
  __shared__ unsigned hist[BINS];
  __shared__ unsigned wsum[32];
  __shared__ unsigned long long s_prefix;
  __shared__ unsigned s_need, s_cnt, s_active;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) out[i] = 0ull;
  if (threadIdx.x == 0) s_prefix = 0ull, s_need = (unsigned)k, s_cnt = 0u, s_active = (unsigned)n;
  __syncthreads();
  if (k > 0 && n > 0) {
    for (int hi = RPN_KEY_BITS; hi > 0;) {
      const int width = hi < DIGIT ? hi : DIGIT, shift = hi - width;
      for (int i = threadIdx.x; i < BINS; i += blockDim.x) hist[i] = 0u;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const unsigned long long pmask = hi >= 64 ? 0ull : (~0ull << hi);
      const unsigned dmask = (1u << width) - 1u;
      // many candidates in few bins (first pass, or heavy ties): one atomic per distinct bin per warp
      const bool aggregate = s_active > 4096u;
      for (int b0 = 0; b0 < n; b0 += blockDim.x) {  // block-uniform trip count
        const int i = b0 + threadIdx.x;
        const unsigned long long key = i < n ? keys[i] : 0ull;
        const bool act = key != 0ull && (key & pmask) == prefix;
        const unsigned bin = (unsigned)(key >> shift) & dmask;
        if (aggregate) {
          const unsigned peers = __match_any_sync(0xffffffffu, act ? bin : 0xFFFFFFFFu);
          if (act && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (unsigned)__popc(peers));
        } else if (act) {
          atomicAdd(&hist[bin], 1u);
        }
      }
      __syncthreads();
      // parallel threshold search: thread t owns bins 2t, 2t+1; E = number of keys in bins above 2t+1
      {
        const unsigned h0 = hist[2 * threadIdx.x], h1 = hist[2 * threadIdx.x + 1], s = h0 + h1;
        unsigned v = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned u = __shfl_down_sync(0xffffffffu, v, o);
          if (lane + o < 32) v += u;
        }
        if (lane == 0) wsum[warp] = v;
        __syncthreads();
        unsigned E = v - s;
        for (int w = warp + 1; w < 32; ++w) E += wsum[w];
        const unsigned need = s_need;
        __syncthreads();  // everyone has read s_need before the owner of the threshold bin rewrites it
        if (E < need && need <= E + h1) {
          s_need = need - E, s_active = h1;
          s_prefix = prefix | ((unsigned long long)(2 * threadIdx.x + 1) << shift);
        } else if (E + h1 < need && need <= E + s) {
          s_need = need - E - h1, s_active = h0;
          s_prefix = prefix | ((unsigned long long)(2 * threadIdx.x) << shift);
        }
        // fewer than `need` keys present: no bin qualifies, the digit stays 0 and everything present is taken
      }
      __syncthreads();
      hi = shift;
      // every key left in the threshold bin is needed: the prefix (lower digits 0) already is the threshold.  Typical after
      // the logit digits -- the index digits only matter when equal logits straddle the cut.
      if (s_need == s_active) break;
    }
    const unsigned long long T = s_prefix;  // the k-th largest key (0 if fewer than k keys exist)
    for (int b0 = 0; b0 < n; b0 += blockDim.x) {
      const int i = b0 + threadIdx.x;
      const unsigned long long key = i < n ? keys[i] : 0ull;
      if (key != 0ull && key >= T) {
        const unsigned pos = atomicAdd(&s_cnt, 1u);
        if (pos < 1024u) out[pos] = key;
      }
    }
  }
  __syncthreads();
}

template <bool BATCHED>
__global__ void __launch_bounds__(1024) rpn_local_topk_kernel(const RpnArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);  // [RPN_CHUNK]
  __shared__ unsigned long long win[1024];
  int lvl = 0;
  while (lvl + 1 < SMOT_MAX_LEVELS && (int)blockIdx.x >= a.chunk_first[lvl + 1]) ++lvl;
  const smot_rpn_level& L = a.lv[lvl];
  const int img = BATCHED ? (int)blockIdx.y : 0;
  const int start = ((int)blockIdx.x - a.chunk_first[lvl]) * RPN_CHUNK;
  const int count = min(RPN_CHUNK, L.H * L.W * L.A - start);
  const int k = min(a.pre_nms_top_n, count);
  const float* __restrict__ head = L.head + (BATCHED ? img * a.head_img_stride[lvl] : 0);
  const int A = L.A, ld = L.head_ld;
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    const int g = start + i;  // anchor index within the level: (cell * A + a)
    keys[i] = rpn_key(head[(size_t)(g / A) * ld + (g % A)], g);
  }
  __syncthreads();
  select_topk_u64(keys, count, k, win);
  unsigned long long* dst = a.local + ((size_t)img * a.nchunks + blockIdx.x) * 1024;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) dst[i] = win[i];
}

template <bool BATCHED>
__global__ void __launch_bounds__(1024) rpn_merge_kernel(const RpnArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ unsigned long long cand[1024];
  const int lvl = blockIdx.x, img = BATCHED ? (int)blockIdx.y : 0;
  const smot_rpn_level& L = a.lv[lvl];
  const int c0 = a.chunk_first[lvl], c1 = a.chunk_first[lvl + 1];
  const int n = (c1 - c0) * 1024;
  const int total = L.H * L.W * L.A;
  const int k = min(a.pre_nms_top_n, total);
  const unsigned long long* __restrict__ src = a.local + ((size_t)img * a.nchunks + c0) * 1024;
  if (c1 - c0 == 1) {
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) cand[i] = src[i];
    __syncthreads();
  } else if (a.merge_in_smem) {
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
    for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = src[i];
    __syncthreads();
    select_topk_u64(keys, n, k, cand);
  } else {
    select_topk_u64(src, n, k, cand);
  }
  bitonic_sort_desc(cand, 1024);
  // ---- decode the k candidates in sorted order
  const float* __restrict__ head = L.head + (BATCHED ? img * a.head_img_stride[lvl] : 0);
  const int slot = img * a.num_levels + lvl;   // the (image, level) candidate slot
  float* cb = a.cand_boxes + (size_t)slot * a.pre_nms_top_n * 4;
  float* cs = a.cand_scores + (size_t)slot * a.pre_nms_top_n;
  for (int j = threadIdx.x; j < a.pre_nms_top_n; j += blockDim.x) {
    if (j >= k) {
      cs[j] = -1.f;
      continue;
    }
    const int i = (int)(RPN_IDX_MASK - (cand[j] & RPN_IDX_MASK));
    const int cell = i / L.A, an = i - cell * L.A;
    const int y = cell / L.W, x = cell - y * L.W;
    const float* row = head + (size_t)cell * L.head_ld;
    const float logit = row[an];
    const float score = __fdiv_rn(1.f, 1.f + expf(-logit));
    const float sx = (float)(x * L.stride), sy = (float)(y * L.stride);
    const float ax1 = L.cell_anchors[an * 4 + 0] + sx, ay1 = L.cell_anchors[an * 4 + 1] + sy;
    const float ax2 = L.cell_anchors[an * 4 + 2] + sx, ay2 = L.cell_anchors[an * 4 + 3] + sy;
    const float* d = row + L.A + 4 * an;
    // BoxCoder(1,1,1,1).decode (TO_REMOVE = 1)
    const float w = ax2 - ax1 + 1.f, h = ay2 - ay1 + 1.f;
    const float cx = ax1 + 0.5f * w, cy = ay1 + 0.5f * h;
    const float dw = fminf(d[2], BBOX_XFORM_CLIP), dh = fminf(d[3], BBOX_XFORM_CLIP);
    const float pcx = d[0] * w + cx, pcy = d[1] * h + cy;
    const float pw = expf(dw) * w, phh = expf(dh) * h;
    float x1 = pcx - 0.5f * pw, y1 = pcy - 0.5f * phh;
    float x2 = pcx + 0.5f * pw - 1.f, y2 = pcy + 0.5f * phh - 1.f;
    if (!a.amodal) {
      x1 = fminf(fmaxf(x1, 0.f), (float)a.img_w - 1.f), y1 = fminf(fmaxf(y1, 0.f), (float)a.img_h - 1.f);
      x2 = fminf(fmaxf(x2, 0.f), (float)a.img_w - 1.f), y2 = fminf(fmaxf(y2, 0.f), (float)a.img_h - 1.f);
    }
    const bool big = (x2 - x1 + 1.f) >= a.min_size && (y2 - y1 + 1.f) >= a.min_size;
    reinterpret_cast<float4*>(cb)[j] = make_float4(x1, y1, x2, y2);
    cs[j] = big ? score : -1.f;
  }
  if (threadIdx.x == 0) a.cand_count[slot] = k;
}

// Cross-level top-n (upstream select_over_all_levels at test time: topk of the concatenated objectness).  Every
// level's survivors are already in (score desc, position asc) order, so the global rank of a row is its own
// position plus, per other level, the number of rows that precede it: rows of lower levels win ties (the order
// topk sees in the level-major concatenation).  No sort, no CTA-wide synchronisation.
template <bool BATCHED>
__global__ void __launch_bounds__(256) rpn_final_kernel(const RpnArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int P = a.post_nms_top_n;
  const int img = BATCHED ? (int)blockIdx.y : 0;   // this image's slices of the kept arrays and of the outputs
  const int* kept_count = a.kept_count + (size_t)img * a.num_levels;
  const float* kept_scores = a.kept_scores + (size_t)img * a.num_levels * P;
  const float* kept_boxes = a.kept_boxes + (size_t)img * a.num_levels * P * 4;
  float* out_boxes = a.out_boxes + (size_t)img * a.final_top_n * 4;
  float* out_scores = a.out_scores + (size_t)img * a.final_top_n;
  if (e == 0) {
    int total = 0;
    for (int l = 0; l < a.num_levels; ++l) total += min(kept_count[l], P);
    a.out_count[img] = min(total, a.final_top_n);
  }
  if (e >= a.num_levels * P) return;
  const int l = e / P, p = e - l * P;
  if (p >= min(kept_count[l], P)) return;
  const float s = kept_scores[e];
  int rank = p;
  for (int o = 0; o < a.num_levels; ++o) {
    if (o == l) continue;
    const float* so = kept_scores + (size_t)o * P;
    int lo = 0, hi = min(kept_count[o], P);  // first position in level o that does NOT precede (l, p)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      const float v = so[mid];
      if (o < l ? v >= s : v > s) lo = mid + 1; else hi = mid;
    }
    rank += lo;
  }
  if (rank < a.final_top_n) {
    reinterpret_cast<float4*>(out_boxes)[rank] = reinterpret_cast<const float4*>(kept_boxes)[e];
    out_scores[rank] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// box head: softmax + per-class decode
// ---------------------------------------------------------------------------------------------
// BATCHED (smot_box_decode_batched): rows are `batch` segments of n_max, row r is row r % n_max of image r / n_max and is decoded
// only below count[image]; the rest of a segment gets score -1 and an empty box, so no later step can read a stale row.
template <bool BATCHED>
__global__ void box_decode_kernel(const float* __restrict__ head, int head_ld, const float* __restrict__ rois,
                                  const int* count, int n_max, int batch, int ncls, float wx, float wy, float ww, float wh,
                                  int img_w, int img_h, int amodal, const int* track_labels,
                                  float* __restrict__ out_boxes, float* __restrict__ out_scores) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (BATCHED ? batch * n_max : n_max)) return;
  const int img = BATCHED ? r / n_max : 0;
  const int n = count ? min(count[img], n_max) : n_max;
  if (r - img * n_max >= n) {
    for (int j = 0; j < ncls; ++j) {
      out_scores[(size_t)r * ncls + j] = -1.f;
      reinterpret_cast<float4*>(out_boxes)[(size_t)r * ncls + j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    return;
  }
  const float* row = head + (size_t)r * head_ld;
  float mx = row[0];
  for (int j = 1; j < ncls; ++j) mx = fmaxf(mx, row[j]);
  float den = 0.f;
  for (int j = 0; j < ncls; ++j) den += expf(row[j] - mx);
  const float4 b = reinterpret_cast<const float4*>(rois)[r];
  const float w = b.z - b.x + 1.f, h = b.w - b.y + 1.f;
  const float cx = b.x + 0.5f * w, cy = b.y + 0.5f * h;
  const int label = track_labels ? track_labels[r] : -1;
  for (int j = 0; j < ncls; ++j) {
    float prob = __fdiv_rn(expf(row[j] - mx), den);
    if (track_labels) prob = (j == label) ? prob + 1.f : 0.f;
    const float* d = row + ncls + 4 * j;
    const float dx = __fdiv_rn(d[0], wx), dy = __fdiv_rn(d[1], wy);
    const float dw = fminf(__fdiv_rn(d[2], ww), BBOX_XFORM_CLIP), dh = fminf(__fdiv_rn(d[3], wh), BBOX_XFORM_CLIP);
    const float pcx = dx * w + cx, pcy = dy * h + cy;
    const float pw = expf(dw) * w, phh = expf(dh) * h;
    float x1 = pcx - 0.5f * pw, y1 = pcy - 0.5f * phh;
    float x2 = pcx + 0.5f * pw - 1.f, y2 = pcy + 0.5f * phh - 1.f;
    if (!amodal) {
      x1 = fminf(fmaxf(x1, 0.f), (float)img_w - 1.f), y1 = fminf(fmaxf(y1, 0.f), (float)img_h - 1.f);
      x2 = fminf(fmaxf(x2, 0.f), (float)img_w - 1.f), y2 = fminf(fmaxf(y2, 0.f), (float)img_h - 1.f);
    }
    out_scores[(size_t)r * ncls + j] = prob;
    reinterpret_cast<float4*>(out_boxes)[(size_t)r * ncls + j] = make_float4(x1, y1, x2, y2);
  }
}

// ---------------------------------------------------------------------------------------------
// per-image detection blocks of the segmented per-class NMS (smot_sort_nms_segmented)
// ---------------------------------------------------------------------------------------------
// One CTA per (image, class) segment.  The NMS kernels left segment p's survivors as original row indices, in kept order, in
// kept_index[p][0 .. kept_n[p]).  The per-class loop of the single-image path appends class j's survivors behind those of
// classes 1 .. j-1, so a segment's first output row is the prefix sum of the keep counts of the image's lower classes: every
// CTA recomputes that prefix (ncls - 1 loads) and scatters its rows; the image's class-1 CTA writes the count and marks the
// rest of the block invalid (score -1), which is what the loop's fill + appends leave behind.
__global__ void __launch_bounds__(256) nms_scatter_segments_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                                   int n_max, int ncls, const int* __restrict__ kept_index,
                                                                   const int* __restrict__ kept_n, int cap, float* __restrict__ out_boxes,
                                                                   float* __restrict__ out_scores, int* __restrict__ out_block) {
  const int K = ncls - 1;
  const int prob = blockIdx.x, img = prob / K, cls = prob - img * K;
  int base = 0, total = 0;
  for (int q = 0; q < K; ++q) {
    const int c = kept_n ? kept_n[img * K + q] : 0;
    total += c;
    base += q < cls ? c : 0;
  }
  const int m = kept_n ? kept_n[prob] : 0;   // (null: no candidates at all)
  const int* idx = kept_index + (size_t)prob * n_max;
  float* ob = out_boxes + (size_t)img * cap * 4;
  float* os = out_scores + (size_t)img * cap;
  int* blk = out_block + (size_t)img * (1 + cap);
  for (int k = threadIdx.x; k < m; k += blockDim.x) {
    const size_t row = ((size_t)img * n_max + idx[k]) * ncls + cls + 1;
    reinterpret_cast<float4*>(ob)[base + k] = reinterpret_cast<const float4*>(boxes)[row];
    os[base + k] = scores[row];
    blk[1 + base + k] = cls + 1;
  }
  if (cls == 0) {
    for (int k = total + threadIdx.x; k < cap; k += blockDim.x) os[k] = -1.f;
    if (threadIdx.x == 0) blk[0] = total;
  }
}

// ---------------------------------------------------------------------------------------------
// candidate assembly for the solver: detections ++ refined tracks (roi_heads.py:60-84,44; track_solver.py:69)
// ---------------------------------------------------------------------------------------------
__global__ void track_combine_kernel(const float* __restrict__ det_boxes, const float* __restrict__ det_scores, int ncap,
                                     const float* __restrict__ dec_boxes, const float* __restrict__ dec_scores, int ncls,
                                     const int* __restrict__ labels, const float* __restrict__ conf,
                                     const int* __restrict__ valid, const float* __restrict__ active, int n, int tracktor,
                                     float* __restrict__ cat_boxes, float* __restrict__ cat_scores, int* zero_me) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && zero_me) *zero_me = 0;
  if (i < ncap) {
    reinterpret_cast<float4*>(cat_boxes)[i] = reinterpret_cast<const float4*>(det_boxes)[i];
    cat_scores[i] = det_scores[i];
  } else if (i < ncap + n) {
    const int r = i - ncap;
    const int lab = labels[r];
    const float det_part = dec_scores[(size_t)r * ncls + lab];  // p + 1 (inference.py:103)
    float s = det_part;
    if (!tracktor) s = __fdiv_rn(det_part + (conf[r] + 1.f), 2.f);  // roi_heads.py:67,76
    s = s + active[r];                                              // track_solver.py:69 (active rows +1)
    reinterpret_cast<float4*>(cat_boxes)[i] = reinterpret_cast<const float4*>(dec_boxes)[(size_t)r * ncls + lab];
    cat_scores[i] = valid[r] ? s : -1.f;
  }
}

// Multi-class form (NUM_CLASSES > 2).  The reference's box head returns the refined tracks GROUPED BY CLASS (filter_results
// loops over the classes, inference.py:145-191), while _refine_tracks took the EMM scores before the box head ran
// (roi_heads.py:67) and adds them position by position (:76).  With one foreground class both orders coincide; with more,
// position g of the class-grouped list carries box / id / label / detection score of track G[g] but the EMM score of V[g],
// where V = the valid tracks in memory order and G = V stably sorted by label.  Replicated here exactly (it decides scores,
// hence ids): the thread of valid track r finds g = its rank in G and the row src = V[g], writes candidate ncap + g and
// perm[g] = r (the host maps solver survivors back to memory rows through perm); positions >= |V| get score -1, perm -1.
// O(n) work per thread, n = tracks in memory (tens).
__global__ void track_combine_grouped_kernel(const float* __restrict__ det_boxes, const float* __restrict__ det_scores, int ncap,
                                             const float* __restrict__ dec_boxes, const float* __restrict__ dec_scores, int ncls,
                                             const int* __restrict__ labels, const float* __restrict__ conf,
                                             const int* __restrict__ valid, const float* __restrict__ active, int n, int tracktor,
                                             float* __restrict__ cat_boxes, float* __restrict__ cat_scores, int* zero_me,
                                             int* __restrict__ perm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && zero_me) *zero_me = 0;
  if (i < ncap) {
    reinterpret_cast<float4*>(cat_boxes)[i] = reinterpret_cast<const float4*>(det_boxes)[i];
    cat_scores[i] = det_scores[i];
    return;
  }
  if (i >= ncap + n) return;
  const int r = i - ncap;
  int m = 0;  // |V|
  for (int q = 0; q < n; ++q) m += valid[q] ? 1 : 0;
  if (r >= m) {  // unused tail position r
    reinterpret_cast<float4*>(cat_boxes)[ncap + r] = make_float4(0.f, 0.f, 0.f, 0.f);
    cat_scores[ncap + r] = -1.f;
    perm[r] = -1;
  }
  if (!valid[r]) return;
  const int lab = labels[r];
  int g = 0;
  for (int q = 0; q < n; ++q)
    if (valid[q] && (labels[q] < lab || (labels[q] == lab && q < r))) ++g;
  int src = -1, cnt = 0;
  for (int q = 0; q < n; ++q)
    if (valid[q]) {
      if (cnt == g) { src = q; break; }
      ++cnt;
    }
  const float det_part = dec_scores[(size_t)r * ncls + lab];          // p + 1 (inference.py:103)
  float s = det_part;
  if (!tracktor) s = __fdiv_rn(det_part + (conf[src] + 1.f), 2.f);    // roi_heads.py:67,76: the score of V[g], not of G[g]
  s = s + active[r];                                                  // track_solver.py:69
  reinterpret_cast<float4*>(cat_boxes)[ncap + g] = reinterpret_cast<const float4*>(dec_boxes)[(size_t)r * ncls + lab];
  cat_scores[ncap + g] = s;
  perm[g] = r;
}

}  // namespace smot

using namespace smot;

extern "C" int smot_track_combine_grouped(const float* det_boxes, const float* det_scores, int ncap, const float* dec_boxes,
                                          const float* dec_scores, int ncls, const int* labels, const float* conf,
                                          const int* valid, const float* active, int n, int tracktor, float* cat_boxes,
                                          float* cat_scores, int* zero_count, int* perm, void* stream) {
  SMOT_CHECK_ARG(ncap >= 0 && n >= 0 && cat_boxes && cat_scores, "smot_track_combine_grouped: bad arguments");
  SMOT_CHECK_ARG(ncap == 0 || (det_boxes && det_scores), "smot_track_combine_grouped: null detections");
  SMOT_CHECK_ARG(n == 0 || (dec_boxes && dec_scores && labels && conf && valid && active && perm && ncls >= 2),
                 "smot_track_combine_grouped: null track arrays");
  const int total = ncap + n;
  track_combine_grouped_kernel<<<(total + 1 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      det_boxes, det_scores, ncap, dec_boxes, dec_scores, ncls, labels, conf, valid, active, n, tracktor, cat_boxes,
      cat_scores, zero_count, perm);
  SMOT_CHECK_LAUNCH("smot_track_combine_grouped");
  return SMOT_OK;
}

extern "C" int smot_track_combine(const float* det_boxes, const float* det_scores, int ncap, const float* dec_boxes,
                                  const float* dec_scores, int ncls, const int* labels, const float* conf, const int* valid,
                                  const float* active, int n, int tracktor, float* cat_boxes, float* cat_scores,
                                  int* zero_count, void* stream) {
  SMOT_CHECK_ARG(ncap >= 0 && n >= 0 && cat_boxes && cat_scores, "smot_track_combine: bad arguments");
  SMOT_CHECK_ARG(ncap == 0 || (det_boxes && det_scores), "smot_track_combine: null detections");
  SMOT_CHECK_ARG(n == 0 || (dec_boxes && dec_scores && labels && conf && valid && active && ncls >= 2),
                 "smot_track_combine: null track arrays");
  const int total = ncap + n;
  track_combine_kernel<<<(total + 1 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      det_boxes, det_scores, ncap, dec_boxes, dec_scores, ncls, labels, conf, valid, active, n, tracktor, cat_boxes,
      cat_scores, zero_count);
  SMOT_CHECK_LAUNCH("smot_track_combine");
  return SMOT_OK;
}

extern "C" size_t smot_sort_nms_workspace(int n_max) {
  if (n_max <= 0) return 0;
  return sort_nms_ws_bytes(1, n_max);
}

extern "C" int smot_sort_nms(const float* boxes, int box_stride, const float* scores, int score_stride, const int* count,
                             int n_max, float min_score, float thresh, int max_keep, int tag, int* out_index,
                             float* out_boxes, float* out_scores, int* out_tag, int* out_count, void* workspace,
                             size_t workspace_bytes, void* stream) {
  SMOT_CHECK_ARG(out_count, "smot_sort_nms: out_count is required");
  SMOT_CHECK_ARG(n_max >= 0 && n_max <= SN_MAX, "smot_sort_nms: n_max %d out of range [0,%d]", n_max, SN_MAX);
  if (n_max == 0) return SMOT_OK;
  SMOT_CHECK_ARG(boxes && scores && box_stride >= 4 && score_stride >= 1 && max_keep >= 0, "smot_sort_nms: bad arguments");
  SMOT_CHECK_ARG(workspace && workspace_bytes >= smot_sort_nms_workspace(n_max), "smot_sort_nms: workspace too small (%zu < %zu)",
                 workspace_bytes, smot_sort_nms_workspace(n_max));
  SortNmsArgs a;
  a.boxes = boxes, a.box_stride = box_stride, a.scores = scores, a.score_stride = score_stride, a.count = count;
  a.n_max = n_max, a.min_score = min_score, a.thresh = thresh, a.max_keep = max_keep, a.tag = tag;
  a.append = 1, a.fill_tail = 0, a.presorted = 0;
  a.out_index = out_index, a.out_boxes = out_boxes, a.out_scores = out_scores, a.out_tag = out_tag, a.out_count = out_count;
  a.in_step = 0, a.out_step = 0;
  carve_sort_nms_ws(a, workspace, 1);
  return launch_sort_nms(a, 1, (cudaStream_t)stream);
}

static int rpn_chunk_count(const smot_rpn_level* levels, int num_levels) {
  int n = 0;
  for (int l = 0; l < num_levels; ++l) n += (levels[l].H * levels[l].W * levels[l].A + RPN_CHUNK - 1) / RPN_CHUNK;
  return n;
}

static size_t rpn_ws_bytes(int num_levels, int pre_nms_top_n, int batch) {
  const size_t L = (size_t)num_levels * batch, P = (size_t)pre_nms_top_n;   // L = (image, level) slots
  size_t b = 0;
  b += align256(L * P * 16);                                 // cand_boxes
  b += align256(L * P * 4);                                  // cand_scores
  b += align256(L * 4);                                      // cand_count
  b += align256(L * P * 16);                                 // kept boxes per level
  b += align256(L * P * 4);                                  // kept scores per level
  b += align256(L * 4);                                      // kept count per level
  b += align256((size_t)batch * RPN_MAX_CHUNKS * 1024 * 8);  // local winners
  b += sort_nms_ws_bytes((int)L, pre_nms_top_n);             // per-level NMS
  return b;
}

extern "C" size_t smot_rpn_select_workspace(int num_levels, int pre_nms_top_n) {
  if (num_levels <= 0 || pre_nms_top_n <= 0) return 0;
  return rpn_ws_bytes(num_levels, pre_nms_top_n, 1);
}

extern "C" size_t smot_rpn_select_batched_workspace(int num_levels, int pre_nms_top_n, int batch) {
  if (num_levels <= 0 || pre_nms_top_n <= 0 || batch <= 0) return 0;
  return rpn_ws_bytes(num_levels, pre_nms_top_n, batch);
}

// smot_rpn_select over `batch` images: every kernel's grid has the image in y (the per-level NMS: problem = image * levels +
// level), so the launch sequence is the single-image one and each image's arithmetic is the single-image arithmetic.
static int rpn_select(const char* who, const smot_rpn_level* levels, const long long* head_img_stride, int batch, int num_levels,
                      int pre_nms_top_n, int post_nms_top_n, float nms_thresh, float min_size, int fpn_post_nms_top_n, int img_w,
                      int img_h, int amodal, float* out_boxes, float* out_scores, int* out_count, void* workspace,
                      size_t workspace_bytes, cudaStream_t st) {
  SMOT_CHECK_ARG(levels && out_boxes && out_scores && out_count && workspace, "%s: null argument", who);
  SMOT_CHECK_ARG(batch >= 1 && batch <= 1024, "%s: batch %d", who, batch);
  SMOT_CHECK_ARG(num_levels >= 1 && num_levels <= SMOT_MAX_LEVELS, "%s: num_levels %d", who, num_levels);
  SMOT_CHECK_ARG(pre_nms_top_n >= 1 && pre_nms_top_n <= 1024, "%s: pre_nms_top_n %d not in [1,1024]", who, pre_nms_top_n);
  SMOT_CHECK_ARG(post_nms_top_n >= 1 && post_nms_top_n <= pre_nms_top_n, "%s: post_nms_top_n %d", who, post_nms_top_n);
  SMOT_CHECK_ARG(num_levels * post_nms_top_n <= SN_MAX, "%s: levels*post_nms_top_n > %d", who, SN_MAX);
  SMOT_CHECK_ARG(workspace_bytes >= rpn_ws_bytes(num_levels, pre_nms_top_n, batch), "%s: workspace too small", who);
  for (int l = 0; l < num_levels; ++l)
    SMOT_CHECK_ARG(levels[l].head && levels[l].A >= 1 && levels[l].A <= SMOT_MAX_ANCHORS && levels[l].H > 0 && levels[l].W > 0 &&
                       levels[l].head_ld >= 5 * levels[l].A &&
                       (long long)levels[l].H * levels[l].W * levels[l].A <= (long long)RPN_IDX_MASK,
                   "%s: bad level %d", who, l);
  const int nchunks = rpn_chunk_count(levels, num_levels);
  SMOT_CHECK_ARG(nchunks <= RPN_MAX_CHUNKS, "%s: feature maps too large (%d chunks > %d)", who, nchunks, RPN_MAX_CHUNKS);
  const size_t L = (size_t)num_levels * batch, P = (size_t)pre_nms_top_n;
  unsigned char* w = (unsigned char*)workspace;
  float* cand_boxes = (float*)w;   w += align256(L * P * 16);
  float* cand_scores = (float*)w;  w += align256(L * P * 4);
  int* cand_count = (int*)w;       w += align256(L * 4);
  float* kept_boxes = (float*)w;   w += align256(L * P * 16);
  float* kept_scores = (float*)w;  w += align256(L * P * 4);
  int* kept_count = (int*)w;       w += align256(L * 4);
  unsigned long long* local = (unsigned long long*)w; w += align256((size_t)batch * RPN_MAX_CHUNKS * 1024 * 8);
  void* ws_level = w;

  RpnArgs ra;
  int nc = 0, widest = 0;
  for (int l = 0; l < SMOT_MAX_LEVELS; ++l) {
    ra.chunk_first[l] = nc;
    ra.head_img_stride[l] = head_img_stride && l < num_levels ? head_img_stride[l] : 0;
    if (l < num_levels) {
      ra.lv[l] = levels[l];
      const int c = (levels[l].H * levels[l].W * levels[l].A + RPN_CHUNK - 1) / RPN_CHUNK;
      nc += c;
      widest = c > widest ? c : widest;
    }
  }
  ra.chunk_first[SMOT_MAX_LEVELS] = nc;
  ra.num_levels = num_levels;
  ra.nchunks = nc, ra.local = local;
  ra.merge_in_smem = widest * 1024 <= RPN_MERGE_SMEM_KEYS;
  ra.pre_nms_top_n = pre_nms_top_n, ra.post_nms_top_n = post_nms_top_n, ra.final_top_n = fpn_post_nms_top_n;
  ra.min_size = min_size, ra.img_w = img_w, ra.img_h = img_h, ra.amodal = amodal;
  ra.cand_boxes = cand_boxes, ra.cand_scores = cand_scores, ra.cand_count = cand_count;
  ra.kept_boxes = kept_boxes, ra.kept_scores = kept_scores, ra.kept_count = kept_count;
  ra.out_boxes = out_boxes, ra.out_scores = out_scores, ra.out_count = out_count;
  // the batched entry point takes the BATCHED instantiations; smot_rpn_select the ones without image offsets
  const bool batched = head_img_stride != nullptr;
  const size_t merge_smem = ra.merge_in_smem && widest > 1 ? (size_t)widest * 1024 * 8 : 0;
  if (batched) {
    SMOT_ENSURE_SMEM(rpn_local_topk_kernel<true>, RPN_CHUNK * 8, "smot_rpn_select(local top-k)");
    SMOT_ENSURE_SMEM(rpn_merge_kernel<true>, RPN_MERGE_SMEM_KEYS * 8, "smot_rpn_select(merge)");
    rpn_local_topk_kernel<true><<<dim3(nc, batch), 1024, RPN_CHUNK * 8, st>>>(ra);
  } else {
    SMOT_ENSURE_SMEM(rpn_local_topk_kernel<false>, RPN_CHUNK * 8, "smot_rpn_select(local top-k)");
    SMOT_ENSURE_SMEM(rpn_merge_kernel<false>, RPN_MERGE_SMEM_KEYS * 8, "smot_rpn_select(merge)");
    rpn_local_topk_kernel<false><<<nc, 1024, RPN_CHUNK * 8, st>>>(ra);
  }
  SMOT_CHECK_LAUNCH("smot_rpn_select(local top-k)");
  if (batched)
    rpn_merge_kernel<true><<<dim3(num_levels, batch), 1024, merge_smem, st>>>(ra);
  else
    rpn_merge_kernel<false><<<num_levels, 1024, merge_smem, st>>>(ra);
  SMOT_CHECK_LAUNCH("smot_rpn_select(merge)");

  // per-level NMS (the candidates are already in score order), survivors into slots of post_nms_top_n rows
  SortNmsArgs a;
  a.boxes = cand_boxes, a.box_stride = 4, a.scores = cand_scores, a.score_stride = 1, a.count = cand_count;
  a.n_max = pre_nms_top_n, a.min_score = -0.5f, a.thresh = nms_thresh, a.max_keep = post_nms_top_n, a.tag = 0;
  a.append = 0, a.fill_tail = post_nms_top_n, a.presorted = 1;
  a.out_index = nullptr, a.out_boxes = kept_boxes, a.out_scores = kept_scores, a.out_tag = nullptr, a.out_count = kept_count;
  a.in_step = pre_nms_top_n, a.out_step = post_nms_top_n;
  carve_sort_nms_ws(a, ws_level, (int)L);
  int rc = launch_sort_nms(a, (int)L, st);
  if (rc) return rc;

  // cross-level top-n
  if (batched)
    rpn_final_kernel<true><<<dim3((num_levels * post_nms_top_n + 255) / 256, batch), 256, 0, st>>>(ra);
  else
    rpn_final_kernel<false><<<(num_levels * post_nms_top_n + 255) / 256, 256, 0, st>>>(ra);
  SMOT_CHECK_LAUNCH("smot_rpn_select(final)");
  return SMOT_OK;
}

extern "C" int smot_rpn_select(const smot_rpn_level* levels, int num_levels, int pre_nms_top_n, int post_nms_top_n,
                               float nms_thresh, float min_size, int fpn_post_nms_top_n, int img_w, int img_h,
                               int amodal, float* out_boxes, float* out_scores, int* out_count, void* workspace,
                               size_t workspace_bytes, void* stream) {
  return rpn_select("smot_rpn_select", levels, nullptr, 1, num_levels, pre_nms_top_n, post_nms_top_n, nms_thresh, min_size,
                    fpn_post_nms_top_n, img_w, img_h, amodal, out_boxes, out_scores, out_count, workspace, workspace_bytes,
                    (cudaStream_t)stream);
}

extern "C" int smot_rpn_select_batched(const smot_rpn_level* levels, const long long* head_image_stride, int batch, int num_levels,
                                       int pre_nms_top_n, int post_nms_top_n, float nms_thresh, float min_size,
                                       int fpn_post_nms_top_n, int img_w, int img_h, int amodal, float* out_boxes,
                                       float* out_scores, int* out_count, void* workspace, size_t workspace_bytes, void* stream) {
  SMOT_CHECK_ARG(head_image_stride, "smot_rpn_select_batched: null head_image_stride");
  return rpn_select("smot_rpn_select_batched", levels, head_image_stride, batch, num_levels, pre_nms_top_n, post_nms_top_n,
                    nms_thresh, min_size, fpn_post_nms_top_n, img_w, img_h, amodal, out_boxes, out_scores, out_count, workspace,
                    workspace_bytes, (cudaStream_t)stream);
}

extern "C" int smot_box_decode(const float* head, int head_ld, const float* rois, const int* count, int n_max, int ncls,
                               const float* weights4, int img_w, int img_h, int amodal, const int* track_labels,
                               float* out_boxes, float* out_scores, void* stream) {
  SMOT_CHECK_ARG(n_max >= 0 && ncls >= 2 && head_ld >= 5 * ncls && weights4, "smot_box_decode: bad arguments");
  if (n_max == 0) return SMOT_OK;
  SMOT_CHECK_ARG(head && rois && out_boxes && out_scores, "smot_box_decode: null argument");
  box_decode_kernel<false><<<(n_max + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      head, head_ld, rois, count, n_max, 1, ncls, weights4[0], weights4[1], weights4[2], weights4[3], img_w, img_h, amodal,
      track_labels, out_boxes, out_scores);
  SMOT_CHECK_LAUNCH("smot_box_decode");
  return SMOT_OK;
}

extern "C" int smot_box_decode_batched(const float* head, int head_ld, const float* rois, const int* count, int batch, int n_max,
                                       int ncls, const float* weights4, int img_w, int img_h, int amodal, float* out_boxes,
                                       float* out_scores, void* stream) {
  SMOT_CHECK_ARG(batch >= 0 && n_max >= 0 && ncls >= 2 && head_ld >= 5 * ncls && weights4 && count,
                 "smot_box_decode_batched: bad arguments");
  const long long rows = (long long)batch * n_max;
  if (rows == 0) return SMOT_OK;
  SMOT_CHECK_ARG(rows <= (1ll << 30), "smot_box_decode_batched: %lld rows", rows);
  SMOT_CHECK_ARG(head && rois && out_boxes && out_scores, "smot_box_decode_batched: null argument");
  box_decode_kernel<true><<<(unsigned)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      head, head_ld, rois, count, n_max, batch, ncls, weights4[0], weights4[1], weights4[2], weights4[3], img_w, img_h, amodal,
      nullptr, out_boxes, out_scores);
  SMOT_CHECK_LAUNCH("smot_box_decode_batched");
  return SMOT_OK;
}

static size_t segmented_ws_bytes(int problems, int n_max) {
  return sort_nms_ws_bytes(problems, n_max) + align256((size_t)problems * n_max * 4) + align256((size_t)problems * 4);
}

extern "C" size_t smot_sort_nms_segmented_workspace(int batch, int ncls, int n_max) {
  if (batch <= 0 || ncls < 2 || n_max <= 0) return 0;
  return segmented_ws_bytes(batch * (ncls - 1), n_max);
}

extern "C" int smot_sort_nms_segmented(const float* boxes, const float* scores, const int* count, int batch, int n_max, int ncls,
                                       float min_score, float thresh, int max_keep, int cap, float* out_boxes, float* out_scores,
                                       int* out_block, void* workspace, size_t workspace_bytes, void* stream) {
  SMOT_CHECK_ARG(batch >= 0 && ncls >= 2 && n_max >= 0 && n_max <= SN_MAX && max_keep >= 0,
                 "smot_sort_nms_segmented: bad arguments (batch %d, ncls %d, n_max %d)", batch, ncls, n_max);
  if (batch == 0) return SMOT_OK;
  const int K = ncls - 1, problems = batch * K;
  SMOT_CHECK_ARG(problems <= 65535, "smot_sort_nms_segmented: %d segments", problems);
  SMOT_CHECK_ARG(boxes && scores && count && out_boxes && out_scores && out_block, "smot_sort_nms_segmented: null argument");
  SMOT_CHECK_ARG((long long)cap >= (long long)K * (max_keep < n_max ? max_keep : n_max),
                 "smot_sort_nms_segmented: cap %d < %d classes x %d survivors", cap, K, max_keep < n_max ? max_keep : n_max);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_max == 0) {   // no candidates: every image's block is empty
    nms_scatter_segments_kernel<<<problems, 256, 0, st>>>(boxes, scores, 0, ncls, nullptr, nullptr, cap, out_boxes, out_scores,
                                                          out_block);
    SMOT_CHECK_LAUNCH("smot_sort_nms_segmented(scatter)");
    return SMOT_OK;
  }
  SMOT_CHECK_ARG(workspace && workspace_bytes >= segmented_ws_bytes(problems, n_max),
                 "smot_sort_nms_segmented: workspace too small (%zu < %zu)", workspace_bytes, segmented_ws_bytes(problems, n_max));
  unsigned char* w = (unsigned char*)workspace + sort_nms_ws_bytes(problems, n_max);
  int* kept_index = (int*)w;
  int* kept_n = (int*)(w + align256((size_t)problems * n_max * 4));
  // the single-image NMS kernels over all (image, class) segments; survivors stay in the workspace as row indices
  SortNmsArgs a;
  a.boxes = boxes + 4, a.box_stride = 4 * ncls, a.scores = scores + 1, a.score_stride = ncls, a.count = count;   // class 1 on
  a.n_max = n_max, a.min_score = min_score, a.thresh = thresh, a.max_keep = max_keep, a.tag = 0;
  a.append = 0, a.fill_tail = 0, a.presorted = 0;
  a.out_index = kept_index, a.out_boxes = nullptr, a.out_scores = nullptr, a.out_tag = nullptr, a.out_count = kept_n;
  a.in_step = n_max, a.out_step = n_max;
  a.seg = K, a.cls_box_step = 4, a.cls_score_step = 1;
  carve_sort_nms_ws(a, workspace, problems);
  int rc = launch_sort_nms(a, problems, st);
  if (rc) return rc;
  nms_scatter_segments_kernel<<<problems, 256, 0, st>>>(boxes, scores, n_max, ncls, kept_index, kept_n, cap, out_boxes, out_scores,
                                                        out_block);
  SMOT_CHECK_LAUNCH("smot_sort_nms_segmented(scatter)");
  return SMOT_OK;
}
