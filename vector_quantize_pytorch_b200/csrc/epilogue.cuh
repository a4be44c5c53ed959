// Row-wise arg-max with a certificate, as run by the consumer warpgroups of the search kernel (vq_assign.cu) on the
// fp32 score tiles the tensor cores leave in their registers (one thread = one row slice).  Replaces the reference's
// `dist.argmax(dim=-1)` over the materialised (N x K) matrix (vector_quantize_pytorch.py:130-145).
//
// Two layers:
//   ScanState  the HOT loop.  Per group of G columns: a max tree and one compare against the row's
//              running threshold thr = (best so far) - W.  Only a group whose maximum beats thr can hold a candidate; it
//              is copied, raw, to a tiny per-thread queue of LIVE groups.  A group that beats the running maximum by
//              more than W kills every older group (queue reset), so the queue almost always holds ONE group.
//   RowState   the exact tagged top-3 (scores carry their column in 4 low mantissa bits), rebuilt once per row sweep
//              from the live groups only.
//
// A group is the 16 accumulator values one thread holds for one row across eight consecutive 8-column blocks of a
// wgmma tile: element e sits at column  base + group_col(e) = base + 8 (e / 2) + (e % 2).  Columns grow with e, so the
// tag order (first column wins among equal truncated values) is the column order.
#pragma once
#include <stdint.h>

namespace vqb {

__host__ __device__ __forceinline__ int group_col(int e) { return ((e >> 1) << 3) | (e & 1); }

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
template <int G>
__device__ __forceinline__ float max_group(const uint32_t* r) {
  static_assert(G == 4 || G == 8 || G == 16, "group size");
  if (G == 4) return fmaxf(fmax3(__uint_as_float(r[0]), __uint_as_float(r[1]), __uint_as_float(r[2])), __uint_as_float(r[3]));
  if (G == 8)
    return fmax3(fmax3(__uint_as_float(r[0]), __uint_as_float(r[1]), __uint_as_float(r[2])),
                 fmax3(__uint_as_float(r[3]), __uint_as_float(r[4]), __uint_as_float(r[5])),
                 fmaxf(__uint_as_float(r[6]), __uint_as_float(r[7])));
  const float a = fmax3(__uint_as_float(r[0]), __uint_as_float(r[1]), __uint_as_float(r[2]));
  const float b = fmax3(__uint_as_float(r[3]), __uint_as_float(r[4]), __uint_as_float(r[5]));
  const float c = fmax3(__uint_as_float(r[6]), __uint_as_float(r[7]), __uint_as_float(r[8]));
  const float d = fmax3(__uint_as_float(r[9]), __uint_as_float(r[10]), __uint_as_float(r[11]));
  const float e = fmax3(__uint_as_float(r[12]), __uint_as_float(r[13]), __uint_as_float(r[14]));
  return fmaxf(fmax3(a, b, c), fmax3(d, e, __uint_as_float(r[15])));
}
__device__ __forceinline__ float max16(const uint32_t (&r)[16]) { return max_group<16>(r); }

// Running top-3 of one row (slice), branch-free.  Scores carry the element's position inside its group in their 4 low
// mantissa bits (tag = 15 - e, so that among equal truncated values the FIRST column wins a max), which makes the whole
// update min/max arithmetic — no compare/select chains, no divergence between the 32 rows of a warp.  The tag perturbs
// a score by < 16 ulp; the certification band W carries that slack.  t3 only answers "is there a third candidate
// inside the band" (-> whole-row exact re-scan).
struct RowState {
  float t1, t2, t3;   // tagged top-3 scores
  float t4;           // fourth best: only answers "is there a fourth candidate inside the band" (-> whole-row exact re-scan)
  float thr, W;       // thr = t1 - W: pieces whose exact maximum is <= thr cannot hold a candidate
  float bexact;       // exact (untagged) running maximum: the score that carries the loss
  int j1, j2, j3;     // first column of the groups t1 / t2 / t3 came from
  __device__ __forceinline__ void init(float w) {
    W = w; t1 = t2 = t3 = t4 = -3.4e38f; bexact = -3.4e38f; thr = -3.4e38f; j1 = 0; j2 = 0; j3 = 0;
  }
  // Pipe balance: only the max of each compare-exchange is an FMNMX (alu pipe); the min is recovered on the fma pipe as
  // an integer identity on the bit patterns, min = a + b - max (exact: max returns one of its inputs), written as IMADs
  // with a multiplier ptxas cannot fold (mul1 = 1, mulm1 = -1 come in through the kernel params).
  template <int G>
  __device__ __forceinline__ void insert(const uint32_t* r, int cbase, uint32_t tagmask, uint32_t mul1, uint32_t mulm1) {
    const float o1 = t1, o2 = t2, o3 = t3;
#pragma unroll
    for (int e = 0; e < G; ++e) {
      const uint32_t ku = (r[e] & tagmask) | static_cast<uint32_t>(15 - e);
      const float n1 = fmaxf(t1, __uint_as_float(ku));
      const uint32_t lo1 = __float_as_uint(n1) * mulm1 + (__float_as_uint(t1) * mul1 + ku);
      const float n2 = fmaxf(t2, __uint_as_float(lo1));
      const uint32_t lo2 = __float_as_uint(n2) * mulm1 + (__float_as_uint(t2) * mul1 + lo1);
      const float n3 = fmaxf(t3, __uint_as_float(lo2));
      const uint32_t lo3 = __float_as_uint(n3) * mulm1 + (__float_as_uint(t3) * mul1 + lo2);
      t4 = fmaxf(t4, __uint_as_float(lo3));
      t1 = n1;
      t2 = n2;
      t3 = n3;
    }
    // Where did t1 / t2 / t3 come from: an old slot (its group) or this group?  Both lists are sorted, so a greedy walk
    // attributes them: a new slot equal to the next unconsumed old value takes that old slot's group, anything else is from
    // this group.  (An equal tagged score in this group is then attributed to the old slot first and to this group after —
    // every reported column stays a distinct real candidate.)
    const int k1 = j1, k2 = j2, k3 = j3;
    const bool m1 = t1 == o1;
    j1 = m1 ? k1 : cbase;
    const float q2 = m1 ? o2 : o1;
    const bool m2 = t2 == q2;
    j2 = m2 ? (m1 ? k2 : k1) : cbase;
    const int used = static_cast<int>(m1) + static_cast<int>(m2);
    const float q3 = used == 0 ? o1 : (used == 1 ? o2 : o3);
    j3 = (t3 == q3) ? (used == 0 ? k1 : (used == 1 ? k2 : k3)) : cbase;
    thr = t1 - W;
  }
  __device__ __forceinline__ void piece(const uint32_t (&r)[16], int cbase, uint32_t tagmask, uint32_t mul1, uint32_t mulm1) {
    insert<16>(r, cbase, tagmask, mul1, mulm1);
  }
  static __device__ __forceinline__ int col(float t, int j) { return j + group_col(15 - static_cast<int>(__float_as_uint(t) & 15u)); }
};

struct MergeSlot { float t1, t2, t3, t4, bexact; int i0, i1, i2; };

// Result of merging the column slices of a row: the candidates (tagged scores inside the band W below the tagged maximum,
// best first, ties towards the lower index), how many there are (n; indices are valid for the first min(n, 3)) and the
// exact winning score.
struct RowResult { int i0, i1, i2, n; float best; };

struct Top3 {
  float v0 = -3.4e38f, v1 = -3.4e38f, v2 = -3.4e38f;
  int i0 = 0, i1 = 0, i2 = 0;
  __device__ __forceinline__ void offer(float v, int i) {   // keep the three best (value desc, index asc)
    if (v > v0 || (v == v0 && i < i0)) { v2 = v1; i2 = i1; v1 = v0; i1 = i0; v0 = v; i0 = i; }
    else if (v > v1 || (v == v1 && i < i1)) { v2 = v1; i2 = i1; v1 = v; i1 = i; }
    else if (v > v2 || (v == v2 && i < i2)) { v2 = v; i2 = i; }
  }
};

__device__ __forceinline__ void publish(MergeSlot* slot, const RowState& st) {
  slot->t1 = st.t1; slot->t2 = st.t2; slot->t3 = st.t3; slot->t4 = st.t4; slot->bexact = st.bexact;
  slot->i0 = RowState::col(st.t1, st.j1); slot->i1 = RowState::col(st.t2, st.j2); slot->i2 = RowState::col(st.t3, st.j3);
}

// merge this thread's slice with `nslots` published slices of the same row (stride = distance between them)
__device__ __forceinline__ RowResult merge_slices(const RowState& st, const MergeSlot* slots, int nslots, int stride) {
  // pass 1: exact best, tagged best and its column, number of candidates inside the band
  float best = st.bexact, tb = st.t1;
  int ib = RowState::col(st.t1, st.j1);
  for (int q = 0; q < nslots; ++q) {
    const MergeSlot& m = slots[q * stride];
    best = fmaxf(best, m.bexact);
    const bool take = m.t1 > tb || (m.t1 == tb && m.i0 < ib);
    tb = take ? m.t1 : tb;
    ib = take ? m.i0 : ib;
  }
  const float band = tb - st.W;
  int n = (st.t1 > band) + (st.t2 > band) + (st.t3 > band) + (st.t4 > band);
  for (int q = 0; q < nslots; ++q) {
    const MergeSlot& m = slots[q * stride];
    n += (m.t1 > band) + (m.t2 > band) + (m.t3 > band) + (m.t4 > band);
  }
  RowResult r;
  r.i0 = ib; r.i1 = 0; r.i2 = 0; r.n = n; r.best = best;
  if (n >= 2) {  // rare (~0.1 % of the rows): the three best candidates over all slices
    Top3 top;
    top.offer(st.t1, RowState::col(st.t1, st.j1));
    top.offer(st.t2, RowState::col(st.t2, st.j2));
    top.offer(st.t3, RowState::col(st.t3, st.j3));
    for (int q = 0; q < nslots; ++q) {
      const MergeSlot& m = slots[q * stride];
      top.offer(m.t1, m.i0);
      top.offer(m.t2, m.i1);
      top.offer(m.t3, m.i2);
    }
    r.i0 = top.i0; r.i1 = top.i1; r.i2 = top.i2;
  }
  return r;
}

// The hot loop (see the header comment).  G = columns per group.  The queue of live groups is a separate thread-local
// array (dynamically indexed -> local memory); keeping it out of this struct keeps the scalars below in registers.
template <int G>
struct ScanQueue {
  static constexpr int CAP = 4;      // live groups kept; one more = overflow -> the row is re-scanned exactly
  uint4 v[CAP + 1][G / 4];           // raw scores of the live groups (+ one spare slot for branch-free stores)
  int c[CAP + 1];                    // first column of each
};

template <int G>
struct ScanState {
  static constexpr int CAP = ScanQueue<G>::CAP;
  float t1;      // exact running maximum of this thread's slice
  float thr;     // max(own, partner slice) running maximum - W
  float kill;    // t1 + W: a group maximum above it makes every queued group irrelevant
  float W;
  int cnt;       // queued groups (CAP + 1 = overflow)

  __device__ __forceinline__ void init(float w) {
    W = w; t1 = -3.4e38f; thr = -3.4e38f; kill = -3.4e38f; cnt = 0;
  }
  // the partner thread of this row (other column half) has reached `other`: nothing <= other - W can be a candidate
  __device__ __forceinline__ void raise(float other) { thr = fmaxf(thr, other - W); }

  // Scalars are updated unconditionally (m <= thr changes none of them), only the stores are predicated: lanes
  // without a candidate cause no memory traffic and the warp does not diverge.
  __device__ __forceinline__ void push(ScanQueue<G>& q, const uint32_t* r, int col, float m, bool p) {
    const int c0 = (m > kill) ? 0 : cnt;
    const int slot = min(c0, CAP);          // overflow lands in the spare slot
    if (p) {
#pragma unroll
      for (int e = 0; e < G; e += 4) q.v[slot][e >> 2] = make_uint4(r[e], r[e + 1], r[e + 2], r[e + 3]);
      q.c[slot] = col;
    }
    cnt = p ? min(c0 + 1, CAP + 1) : cnt;
    t1 = fmaxf(t1, m);
    thr = fmaxf(thr, t1 - W);
    kill = t1 + W;
  }

  // One warp-uniform branch per 16-column piece (32 rows per warp: at K ~ 1e3 some lane holds a running-maximum
  // record in most pieces, so what counts is that the taken path is short and free of divergence).
  template <bool BRANCH = true>
  __device__ __forceinline__ void scan16(ScanQueue<G>& q, const uint32_t (&r)[16], int cbase) {
    float m[16 / G];
    bool any = false;
#pragma unroll
    for (int g = 0; g < 16 / G; ++g) {
      m[g] = max_group<G>(r + g * G);
      any |= m[g] > thr;
    }
    if (!BRANCH || __any_sync(0xffffffffu, any)) {
#pragma unroll
      for (int g = 0; g < 16 / G; ++g) push(q, r + g * G, cbase + g * G, m[g], m[g] > thr);
    }
  }

  // Rebuild the exact tagged top-3 of this slice from the live groups (typically one).
  __device__ __forceinline__ void finish(const ScanQueue<G>& q, RowState& st, uint32_t tagmask, uint32_t mul1, uint32_t mulm1) {
    const float w = W;
    st.init(w);
    st.bexact = t1;
    const float live = t1 - w;
    const int n = min(cnt, CAP);
    for (int i = 0; i < n; ++i) {
      uint32_t v[G];
#pragma unroll
      for (int e = 0; e < G; e += 4) {
        const uint4 u = q.v[i][e >> 2];
        v[e] = u.x; v[e + 1] = u.y; v[e + 2] = u.z; v[e + 3] = u.w;
      }
      if (max_group<G>(v) > live) st.template insert<G>(v, q.c[i], tagmask, mul1, mulm1);
    }
    if (cnt > CAP) { st.t2 = st.t1; st.t3 = st.t1; st.t4 = st.t1; }  // overflow: more live groups than the queue holds -> >= 3 candidates
  }
};

// live[e] = pred ? r[e] : live[e] as PREDICATED IMADs (r * one + 0, `one` = 1 from the kernel parameters so that ptxas
// cannot fold it into a SEL / MOV): the copy then runs on the fma pipe, which idles in the epilogue, instead of the alu
// pipe that bounds it (FMNMX / SEL issue at half rate there).
__device__ __forceinline__ void cond_copy8(uint32_t* live, const uint32_t* r, bool pred, uint32_t one) {
  asm("{\n"
      ".reg .pred q;\n"
      "setp.ne.u32 q, %16, 0;\n"
      "@q mad.lo.u32 %0, %8, %17, 0;\n"
      "@q mad.lo.u32 %1, %9, %17, 0;\n"
      "@q mad.lo.u32 %2, %10, %17, 0;\n"
      "@q mad.lo.u32 %3, %11, %17, 0;\n"
      "@q mad.lo.u32 %4, %12, %17, 0;\n"
      "@q mad.lo.u32 %5, %13, %17, 0;\n"
      "@q mad.lo.u32 %6, %14, %17, 0;\n"
      "@q mad.lo.u32 %7, %15, %17, 0;\n"
      "}"
      : "+r"(live[0]), "+r"(live[1]), "+r"(live[2]), "+r"(live[3]), "+r"(live[4]), "+r"(live[5]), "+r"(live[6]), "+r"(live[7])
      : "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]), "r"(r[4]), "r"(r[5]), "r"(r[6]), "r"(r[7]),
        "r"(static_cast<uint32_t>(pred)), "r"(one));
}

// Register-resident variant of the hot loop: the (almost always single) live group of 16 columns is kept in registers
// and replaced with predicated moves; only a second live group inside the band (a near tie) goes to the thread-local queue.
struct ScanReg {
  static constexpr int CAP = ScanQueue<16>::CAP;
  float t1, thr, kill, W;
  int cnt;            // groups in the queue besides `live` (CAP + 1 = overflow)
  int lcol;           // first column of the live group (-1: none yet)
  uint32_t live[16];

  __device__ __forceinline__ void init(float w) {
    W = w; t1 = -3.4e38f; thr = -3.4e38f; kill = -3.4e38f; cnt = 0; lcol = -1;
#pragma unroll
    for (int e = 0; e < 16; ++e) live[e] = 0xFF7FFFFFu;  // -FLT_MAX
  }
  __device__ __forceinline__ void raise(float other) { thr = fmaxf(thr, other - W); }

  template <bool BRANCH = true, bool IMAD = false>
  __device__ __forceinline__ void scan16(ScanQueue<16>& q, const uint32_t (&r)[16], int cbase, uint32_t one = 1u) {
    const float m = max_group<16>(r);
    const bool p = m > thr;
    if (!BRANCH || __any_sync(0xffffffffu, p)) {
      const bool reset = m > kill;             // beats everything seen so far by more than W (implies p)
      const bool tie = p && !reset;            // a second live group: rare
      if (__any_sync(0xffffffffu, tie)) {
        if (tie) {
          const int slot = min(cnt, CAP);
#pragma unroll
          for (int e = 0; e < 16; e += 4) q.v[slot][e >> 2] = make_uint4(r[e], r[e + 1], r[e + 2], r[e + 3]);
          q.c[slot] = cbase;
          cnt = min(cnt + 1, CAP + 1);
        }
      }
      if (IMAD) {
        cond_copy8(live, r, reset, one);
        cond_copy8(live + 8, r + 8, reset, one);
      } else {
#pragma unroll
        for (int e = 0; e < 16; ++e) live[e] = reset ? r[e] : live[e];
      }
      lcol = reset ? cbase : lcol;
      cnt = reset ? 0 : cnt;
      t1 = fmaxf(t1, m);
      thr = fmaxf(thr, t1 - W);
      kill = t1 + W;
    }
  }

  __device__ __forceinline__ void finish(const ScanQueue<16>& q, RowState& st, uint32_t tagmask, uint32_t mul1, uint32_t mulm1) {
    const float w = W;
    st.init(w);
    st.bexact = t1;
    if (lcol >= 0) st.template insert<16>(live, lcol, tagmask, mul1, mulm1);
    const float lv = t1 - w;
    const int n = min(cnt, CAP);
    for (int i = 0; i < n; ++i) {
      uint32_t v[16];
#pragma unroll
      for (int e = 0; e < 16; e += 4) {
        const uint4 u = q.v[i][e >> 2];
        v[e] = u.x; v[e + 1] = u.y; v[e + 2] = u.z; v[e + 3] = u.w;
      }
      if (max_group<16>(v) > lv) st.template insert<16>(v, q.c[i], tagmask, mul1, mulm1);
    }
    if (cnt > CAP) { st.t2 = st.t1; st.t3 = st.t1; st.t4 = st.t1; }
  }
};

}  // namespace vqb
