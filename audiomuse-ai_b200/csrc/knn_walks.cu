// Candidate post-processing on the stored rows of the k-NN index (knn.cu), each one kernel behind one host call: the
// duplicate filter, the radius walk, and the by-vector chain's requests -- the song path's jobs, Song Alchemy and the
// plain similar-tracks queries.  The duplicate filter and the chain's requests walk their lists through one filter window
// (FilterWindow) and one per-item walk (walk_list).
#include "host_call.cuh"
#include "knn.cuh"

#include <math_constants.h>

#include <algorithm>

namespace am {

// ---------------------------------------------------------------- distances
// a . b, |a|^2, |b|^2 and |a - b|^2 between a (stored row or float64 centroid) and stored row b, one warp, float64
// accumulation
struct Moments {
  double dot, na, nb, d2;
};

template <class T>
__device__ __forceinline__ Moments warp_moments(const T* a, const float* b, int d, int lane) {
  double dot = 0.0, na = 0.0, nb = 0.0, d2 = 0.0;
  for (int t = lane; t < d; t += 32) {
    const double av = (double)__ldg(&a[t]), bv = (double)__ldg(&b[t]);
    dot = fma(av, bv, dot);
    na = fma(av, av, na);
    nb = fma(bv, bv, nb);
    const double df = av - bv;
    d2 = fma(df, df, d2);
  }
  return {warp_sum(dot), warp_sum(na), warp_sum(nb), warp_sum(d2)};
}

// get_direct_distance (voyager_manager.py:99-140) between stored rows a and b: euclidean ||a - b||, otherwise 1 - cos
// (+inf when either row is zero)
__device__ __forceinline__ double direct_distance(const float* a, const float* b, int d, int metric, int lane) {
  const Moments m = warp_moments(a, b, d, lane);
  if (metric == kMetricL2) return sqrt(m.d2);
  const double den = sqrt(m.na) * sqrt(m.nb);
  return den == 0.0 ? INFINITY : 1.0 - fmin(1.0, fmax(-1.0, m.dot / den));
}


// ---------------------------------------------------------------- the filter window and the per-item walk
// _filter_by_distance (voyager_manager.py:526-617) + :487-524 (_compute_distance_batch) over one list in order: an item
// whose DIRECT distance to a recently kept item is below the threshold is dropped, and so is an item without a vector.
// "Recently kept": lists of <= `batch` items compare with the last `lookback` kept items; longer lists are cut into
// batches of `batch`, and an item is compared with the last `lookback` items kept BEFORE its batch plus everything kept
// so far inside the batch.  With no lookback the reference returns the list unchanged: nothing is compared and every
// item passes.  Every thread holds the same counts and admits every item; thread 0 writes the kept list.
struct FilterWindow {
  const float* X;
  int64_t N;
  int d, metric;
  double threshold;
  int lookback, batch;
  bool batched;      // the list is longer than one batch
  int* kept;         // the kept items' positions in the list
  int n = 0;         // kept so far
  int at_batch = 0;  // kept when the current batch started

  __device__ FilterWindow(const float* X, int64_t N, int d, int metric, double threshold, int lookback, int batch,
                          int L, int* kept)
      : X(X), N(N), d(d), metric(metric), threshold(threshold), lookback(lookback), batch(batch), batched(L > batch),
        kept(kept) {}

  // the first kept position item i is compared with (n: none)
  __device__ __forceinline__ int start(int i) {
    if (batched && i % batch == 0) at_batch = n;
    return lookback > 0 ? max(0, (batched ? at_batch : n) - lookback) : n;
  }

  // whether item i passes the filter; valid: it has a vector, close: it came within the threshold of the window
  __device__ __forceinline__ bool admit(int i, bool valid, bool close) {
    if (lookback <= 0) return true;
    if (!valid || close) return false;
    if (threadIdx.x == 0) kept[n] = i;
    ++n;
    return true;
  }
};

constexpr int kClose = 1;  // walk flag: the item came within the threshold of the filter window

// The walk over a list of L items, one item at a time, three barriers an item.  row_of(i) is item i's stored row (-1 or
// >= N: no vector).  Between the first two barriers every warp computes the item's distances to the window and then
// extra(row, valid, slot) runs on every thread: the caller's own per-item work, whose distance slots continue the
// window's (slot is the first this warp takes, when valid), so that all the item's distances are spread over the warps
// as one range; it returns the flag bits above kClose that the thread found.  After the second barrier every thread
// admits the item to the window and thread 0 runs decide(i, row, valid, passed the filter, flags), which keeps the
// books and returns true to end the walk.
struct NoExtra {
  __device__ int operator()(int64_t, bool, int) const { return 0; }
};

template <class RowOf, class Extra, class Decide>
__device__ __forceinline__ void walk_list(FilterWindow& w, int L, RowOf row_of, Extra extra, Decide decide) {
  __shared__ int s_flags;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (int i = 0; i < L; ++i) {
    const int64_t row = row_of(i);
    const bool valid = row >= 0 && row < w.N;  // the reference skips items whose vector is missing
    const int f0 = w.start(i);
    if (threadIdx.x == 0) s_flags = 0;
    __syncthreads();
    int flags = 0, t = f0 + warp;  // slot t - f0
    if (valid)
      for (; t < w.n; t += warps) {
        const double dist = direct_distance(w.X + row * w.d, w.X + row_of(w.kept[t]) * w.d, w.d, w.metric, lane);
        if (lane == 0 && dist < w.threshold) flags = kClose;
      }
    flags |= extra(row, valid, t - w.n);
    if (flags) atomicOr(&s_flags, flags);
    __syncthreads();
    const int f = s_flags;
    const bool pass = w.admit(i, valid, f & kClose);
    bool stop = false;
    if (threadIdx.x == 0) stop = decide(i, row, valid, pass, f);
    if (__syncthreads_or(stop)) break;
  }
}

// One CTA per list, the comparisons of one item spread over the warps.
constexpr int kFilterThreads = 256;
constexpr int kFilterCap = 4096;  // items per list

__global__ void __launch_bounds__(kFilterThreads)
filter_by_distance_kernel(const float* __restrict__ X, int64_t N, int d, int metric, const int64_t* __restrict__ ids,
                          int n, double threshold, int lookback, int batch, unsigned char* __restrict__ keep) {
  __shared__ int s_kept[kFilterCap];
  const int64_t* my_ids = ids + (int64_t)blockIdx.x * n;
  unsigned char* my_keep = keep + (int64_t)blockIdx.x * n;
  FilterWindow w(X, N, d, metric, threshold, lookback, batch, n, s_kept);
  walk_list(w, n, [&](int i) { return my_ids[i]; }, NoExtra{}, [&](int i, int64_t, bool, bool pass, int) {
    my_keep[i] = pass ? 1 : 0;
    return false;
  });
}


// ---------------------------------------------------------------- radius walk on device
// voyager_manager.py:941-1367 (_execute_radius_walk) over the candidates _radius_walk_get_candidates (:842-938) leaves,
// in one CTA.  The reference's steps and the state that restates each:
//   * anchor distances (:927, get_direct_distance) in float64, one warp per candidate; the stable sort by that distance
//     (:968) is a bitonic sort of (distance bits, input position) keys -- distances are >= 0 or +inf, so their bit
//     patterns order like the values, and the position breaks ties the way a stable sort keeps them;
//   * buckets of 50 in that order (:956, :970-974), walked one after the other until the playlist holds n songs (what
//     the window-doubling loop at :1261-1281 amounts to);
//   * the first song is sorted[0] (:1008-1013); its artist counts (:1041-1047) but not per bucket;
//   * each bucket starts at its first unused candidate (:1091-1103; in bucket 0 that skips sorted[0]), accepted if it
//     passes the artist rules and otherwise only dropped from the bucket (:1140-1163);
//   * then greedily: score = 0.7 d(prev, cand) + 0.3 float32(d(anchor, cand)) (:1222), the first strict minimum in
//     bucket order wins (:1223), prev is the last song APPENDED (:1174), and the bucket ends when no candidate passes;
//   * the artist rules (:1120-1136, :1188-1211) apply when eliminate_duplicates and the cap is > 0: one song per artist
//     per bucket, and an artist already in 2 buckets or at the cap is refused;
//   * once the playlist holds n songs nothing later changes it (:1146, :1237, :1262), so the walk stops there;
//   * _avoid_triple_adjacent (:1287-1318) on the final order.
// Per-candidate state lives in global scratch (sort keys, per-artist counters, the playlist); only the distances from
// the current song to the <= 50 candidates of the bucket are in shared memory.  Warp 0 keeps the books, every warp
// computes distances.
constexpr int kWalkThreads = 1024;
constexpr int kWalkBucket = 50;    // BUCKET_SIZE, voyager_manager.py:956
constexpr unsigned long long kWalkMissing = ~0ull;  // sort key of a candidate that is not in the index: after +inf

__device__ __forceinline__ double walk_key_dist(unsigned long long k) { return __longlong_as_double((long long)k); }

// artists[c] of input position c (-1: no artist); count / buckets / mark: per artist, the songs taken, the buckets it
// has a song in, and the last bucket it took a song in
__device__ __forceinline__ bool walk_artist_ok(int a, int bucket, int cap, const int* count, const int* buckets,
                                               const int* mark) {
  return a < 0 || !(mark[a] == bucket || buckets[a] >= 2 || count[a] >= cap);
}

__global__ void __launch_bounds__(kWalkThreads)
radius_walk_kernel(const float* __restrict__ X, int64_t N, int d, int metric, const float* __restrict__ anchor,
                   const int64_t* __restrict__ rows, const int32_t* __restrict__ artists, int n_cand, int n,
                   int artist_rules, int cap, int64_t npad, unsigned long long* key, int* ord, int* count,
                   int* buckets, int* mark, int* playlist, int32_t* __restrict__ out_pos,
                   double* __restrict__ out_dist, int32_t* __restrict__ out_count) {
  __shared__ double s_dprev[kWalkBucket];
  __shared__ unsigned long long s_elig;  // candidates of the bucket that may be taken next
  __shared__ int s_valid, s_len, s_prev_pos;  // valid candidates, playlist length, input position of the last song
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = kWalkThreads / 32;
  if (threadIdx.x == 0) s_valid = 0;
  __syncthreads();

  // ---- anchor distances and sort keys (padding sorts after every candidate)
  for (int64_t i = warp; i < npad; i += warps) {
    unsigned long long k = kWalkMissing;
    const int64_t row = i < n_cand ? rows[i] : -1;
    if (row >= 0 && row < N) {
      k = (unsigned long long)__double_as_longlong(direct_distance(X + row * d, anchor, d, metric, lane));
      if (lane == 0) atomicAdd(&s_valid, 1);
    }
    if (lane == 0) {
      key[i] = k;
      ord[i] = (int)i;
    }
  }
  __syncthreads();
  // ---- bitonic sort of (key, position) ascending
  for (int64_t kk = 2; kk <= npad; kk <<= 1) {
    for (int64_t j = kk >> 1; j > 0; j >>= 1) {
      for (int64_t i = threadIdx.x; i < npad; i += kWalkThreads) {
        const int64_t l = i ^ j;
        if (l > i) {
          const unsigned long long ki = key[i], kl = key[l];
          const int oi = ord[i], ol = ord[l];
          const bool i_after = ki > kl || (ki == kl && oi > ol);
          if (i_after == ((i & kk) == 0)) {
            key[i] = kl;
            key[l] = ki;
            ord[i] = ol;
            ord[l] = oi;
          }
        }
      }
      __syncthreads();
    }
  }

  // ---- the walk; sorted index s -> input position ord[s], anchor distance key[s]
  const int m = s_valid;
  if (threadIdx.x == 0) {
    s_len = 0;
    if (m > 0 && n > 0) {  // the first song (:1008-1013, :1041-1047)
      playlist[0] = 0;
      s_len = 1;
      s_prev_pos = ord[0];
      const int a = artists[ord[0]];
      if (a >= 0) count[a] += 1;
    }
  }
  __syncthreads();
  for (int b = 0;; ++b) {
    const bool go = (int64_t)b * kWalkBucket < m && s_len < n;  // read by every thread before warp 0 writes again
    __syncthreads();
    if (!go) break;
    const int base = b * kWalkBucket, nb = min(kWalkBucket, m - base);
    // warp 0's books for this bucket: candidates still available, playlist length, the artist of each lane's two
    // candidates (j = lane, lane + 32)
    unsigned long long avail = ((1ull << nb) - 1) & ~(b == 0 ? 1ull : 0ull);  // bucket 0 holds the first song
    int len = 0, art[2] = {-1, -1};
    // the candidates that may be taken next (a warp-wide ballot)
    auto eligible = [&]() {
      unsigned long long e = 0;
      for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        const bool ok = j < nb && ((avail >> j) & 1) &&
                        (!artist_rules || walk_artist_ok(art[h], b, cap, count, buckets, mark));
        e |= (unsigned long long)__ballot_sync(0xffffffffu, ok) << (32 * h);
      }
      return e;
    };
    // take sorted index base + j (the bookkeeping of :1141-1161 / :1232-1253); lane 0 writes, the warp reads back
    auto accept = [&](int j) {
      avail &= ~(1ull << j);
      if (lane == 0) {
        if (len < n) {
          playlist[len] = base + j;
          s_prev_pos = ord[base + j];
        }
        const int a = artists[ord[base + j]];
        if (a >= 0) {
          count[a] += 1;
          if (mark[a] != b) {
            mark[a] = b;
            buckets[a] += 1;
          }
        }
      }
      if (len < n) ++len;
      __syncwarp();
    };
    if (warp == 0) {
      len = s_len;
      for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        if (j < nb) art[h] = artists[ord[base + j]];
      }
      if (avail) {  // the start (:1105-1163): the first available candidate, taken if the artist rules allow it
        const int start = __ffsll((long long)avail) - 1;
        if ((eligible() >> start) & 1) accept(start);
        else avail &= ~(1ull << start);
      }
      const unsigned long long e = len < n ? eligible() : 0ull;
      if (lane == 0) {
        s_len = len;
        s_elig = e;
      }
    }
    // greedy steps (:1166-1253): every warp computes d(prev, cand) for the eligible candidates, warp 0 picks
    for (;;) {
      __syncthreads();  // s_elig / s_prev_pos published
      const unsigned long long e = s_elig;
      if (e == 0) break;
      const float* prev = X + rows[s_prev_pos] * d;
      for (int j = warp; j < nb; j += warps)
        if ((e >> j) & 1) {
          const double dist = direct_distance(X + rows[ord[base + j]] * d, prev, d, metric, lane);
          if (lane == 0) s_dprev[j] = dist;
        }
      __syncthreads();  // distances ready
      if (warp == 0) {
        double best = INFINITY;  // a score must be strictly below +inf and below every earlier one (:1179, :1223)
        int best_j = INT_MAX;
        for (int h = 0; h < 2; ++h) {
          const int j = lane + 32 * h;
          if (j < nb && ((e >> j) & 1)) {
            const double a32 = (double)(float)walk_key_dist(key[base + j]);  // the bucket's float32 array (:983)
            const double score = __dadd_rn(__dmul_rn(0.7, s_dprev[j]), __dmul_rn(0.3, a32));
            if (score < best) {
              best = score;
              best_j = j;
            }
          }
        }
        for (int o = 16; o > 0; o >>= 1) {  // the first minimum in bucket order
          const double ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oj = __shfl_xor_sync(0xffffffffu, best_j, o);
          if (ob < best || (ob == best && oj < best_j)) {
            best = ob;
            best_j = oj;
          }
        }
        unsigned long long next = 0;
        if (best_j != INT_MAX) {
          accept(best_j);
          if (len < n) next = eligible();
        }
        if (lane == 0) {
          s_len = len;
          s_elig = next;
        }
      }
    }
  }

  // ---- _avoid_triple_adjacent (:1287-1318) on the playlist, then the outputs
  const int L = s_len;
  if (threadIdx.x == 0) {
    auto author = [&](int t) { return artists[ord[playlist[t]]]; };
    int i = 0;
    while (i <= L - 3) {
      const int a1 = author(i);
      if (a1 >= 0 && a1 == author(i + 1) && a1 == author(i + 2)) {
        int j = i + 3;
        while (j < L && author(j) == a1) ++j;
        if (j < L) {  // swap the third with the first later song by another artist, then look at i again
          const int t = playlist[i + 2];
          playlist[i + 2] = playlist[j];
          playlist[j] = t;
          continue;
        }
      }
      ++i;
    }
    *out_count = L;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < L; t += kWalkThreads) {
    out_pos[t] = ord[playlist[t]];
    out_dist[t] = walk_key_dist(key[playlist[t]]);
  }
}


// ---------------------------------------------------------------- the by-vector chain
// find_nearest_neighbors_by_vector (voyager_manager.py:1589-1657) after its k-NN query, for the song path's jobs, Song
// Alchemy and the plain similar-tracks requests: one item at a time in k-NN order (walk_list), each stage looking only at
// what came before it.
//   * _filter_by_distance (:526-617) in the VOYAGER_METRIC distance: the filter window;
//   * same-song dedupe (:1625-1636): an item without details, or whose signature this list already let through, is out;
//   * the mood stage of find_nearest_neighbors_by_id (:1512, _filter_by_mood_similarity): the caller's verdict, taken
//     after the signature is marked (the reference's dedupe marks a song the mood filter then drops); the by-vector
//     callers pass true;
//   * the raw-author cap (:1638-1653, only when eliminate_duplicates and the cap is > 0; falsy authors are out).
// step() is thread 0's decision and books for the stages after the filter.
struct ByVectorChain {
  const int64_t* row;  // [n_cand] stored row, -1: no vector
  const int32_t* sig;  // [n_cand] (title, author) signature key, -1: no details
  const int32_t* raw;  // [n_cand] raw author key, -1: falsy author
  int32_t* kept;       // [longest list] scratch: the filter window's kept positions
  int32_t* seen;       // [n_sig] scratch: the list that last let the signature through, -1 initially
  int32_t* raw_mark;   // [n_raw] scratch: the list that last counted the raw author, -1 initially
  int32_t* raw_count;  // [n_raw] scratch

  // candidate p of list `list`: pass = it passed the filter, mood = it passes the mood stage.  True when it passes every
  // stage.
  __device__ __forceinline__ bool step(int list, int p, bool pass, bool mood, int cap) const {
    const int s = sig[p], r = raw[p];  // both loads in flight before the books' dependent ones
    if (!pass || s < 0 || seen[s] == list) return false;
    seen[s] = list;
    if (!mood) return false;
    if (cap > 0) {
      if (r < 0) return false;
      if (raw_mark[r] != list) {
        raw_mark[r] = list;
        raw_count[r] = 0;
      }
      if (raw_count[r] >= cap) return false;
      raw_count[r] += 1;
    }
    return true;
  }
};


// ---------------------------------------------------------------- song path walk on device
// path_manager.py:180-317 (_find_best_songs_for_job) over the chain find_nearest_neighbors_by_vector
// (voyager_manager.py:1547-1657) runs on each job's k-NN prefix, for a sequence of jobs, in one CTA.  One pass over a
// job's candidates in k-NN order does every stage, because each stage only looks at what came before it:
//   * the by-vector chain (ByVectorChain, each job a list of its own);
//   * [:n]: the pass ends after the n-th item that got this far;
//   * acceptance (path_manager.py:211-291): used rows and signatures, the normalised-author cap, then the lookbacks
//     against the path's last songs and this job's found songs, in PATH_DISTANCE_METRIC; the job ends once it has
//     its songs.  A job that falls short gives back what it took (:294-312).
// Per candidate the walk's extra work is the path window's and the found window's distances, and the threads' look
// for the row among the used rows.
constexpr int kPathThreads = 512;
constexpr int kPathClose = 2, kFoundClose = 4, kUsed = 8;  // walk flags

// get_distance (path_manager.py:27-52): euclidean ||a - b||, angular arccos(clip(cos)) / pi (+inf when either row is
// zero).  cos = 1 - (1 - cos) is exact for cos >= 0.5, which covers every distance below the thresholds.
__device__ __forceinline__ double path_distance(const float* a, const float* b, int d, int metric, int lane) {
  const double dd = direct_distance(a, b, d, metric, lane);
  if (metric == kMetricL2 || dd == INFINITY) return dd;
  return acos(1.0 - dd) / CUDART_PI;
}

struct SongPathArgs {
  const float* X;
  int64_t N;
  int d;
  int n_jobs;
  const int32_t* job_off;     // [n_jobs + 1] candidate ranges
  const int32_t* job_n;       // [n_jobs] the by-vector n (k_search)
  const int32_t* job_need;    // [n_jobs] num_to_find
  ByVectorChain chain;        // the candidates, kept: [max candidates per job]
  const int32_t* cand_author; // normalised author key
  int64_t* used_row;          // [n_used + sum(need)] in / out
  int32_t* n_used;
  unsigned char* used_sig;    // [n_sig] in / out
  int32_t* author_count;      // [n_author] in / out
  int64_t* path_row;          // [n_path + sum(need)] in / out: the start song first
  int32_t* n_path;
  int64_t end_row;
  am_song_path_cfg cfg;
  int32_t* found;             // [max candidates per job] scratch: the job's found songs, by position in its list
  int32_t* out_found;         // [n_jobs]
  int32_t* out_pos;           // [sum(need)] accepted candidates, in path order
  int32_t* out_failed;        // first failed job when stopping on failure, else -1
  double* out_dist;           // [n_path + sum(need)] distances between consecutive songs of the path and the end song
};

__global__ void __launch_bounds__(kPathThreads) song_path_kernel(const SongPathArgs a) {
  __shared__ int s_found, s_n_used, s_n_path;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, warps = kPathThreads / 32;
  const am_song_path_cfg& c = a.cfg;
  const ByVectorChain& chain = a.chain;
  for (int j = tid; j < a.n_jobs; j += kPathThreads) a.out_found[j] = 0;  // jobs after a stop are not run
  int n_out = 0;  // thread 0: songs taken so far
  if (tid == 0) {
    s_n_used = *a.n_used;
    s_n_path = *a.n_path;
    *a.out_failed = -1;
  }
  __syncthreads();
  for (int j = 0; j < a.n_jobs; ++j) {
    const int base = a.job_off[j], m = a.job_off[j + 1] - base, n = a.job_n[j], need = a.job_need[j];
    const int64_t* rows = chain.row + base;
    int found = 0, prod = 0;  // thread 0: songs found, items through the chain
    if (tid == 0) s_found = 0;
    const int used0 = s_n_used;  // thread 0: the rows this job adds are given back by truncation
    FilterWindow w(a.X, a.N, a.d, c.voyager_metric, c.filter_threshold, c.filter_lookback, c.filter_batch, m,
                   chain.kept);
    walk_list(
        w, m, [&](int i) { return rows[i]; },
        [&](int64_t row, bool valid, int slot) {
          int flags = 0;
          if (valid) {
            const int np = s_n_path, nfound = s_found, npw = min(c.path_lookback, np), nq = min(c.path_lookback, nfound);
            for (int u = slot; u < npw + nq; u += warps) {
              const int64_t other = u < npw ? a.path_row[np - npw + u] : rows[a.found[nfound - nq + (u - npw)]];
              const double dist = path_distance(a.X + row * a.d, a.X + other * a.d, a.d, c.path_metric, lane);
              if (lane == 0 && dist < c.path_threshold) flags |= u < npw ? kPathClose : kFoundClose;
            }
          }
          for (int t = tid; t < s_n_used; t += kPathThreads)
            if (a.used_row[t] == row) flags |= kUsed;
          return flags;
        },
        [&](int i, int64_t row, bool valid, bool pass, int flags) {
          const int p = base + i;
          if (!chain.step(j, p, pass, true, c.voyager_cap)) return false;
          ++prod;
          const int sig = chain.sig[p], au = a.cand_author[p];
          const bool ok = !(flags & kUsed) && !a.used_sig[sig] && !(c.path_cap > 0 && a.author_count[au] >= c.path_cap) &&
                          valid && !(flags & (kPathClose | kFoundClose));
          if (ok) {
            a.used_row[s_n_used++] = row;
            a.used_sig[sig] = 1;
            a.author_count[au] += 1;
            a.out_pos[n_out + found] = p;
            a.found[found++] = i;
            s_found = found;
          }
          return found >= need || prod >= n;
        });
    bool failed = false;
    if (tid == 0) {
      if (found < need) {  // roll back (:294-312)
        for (int t = 0; t < found; ++t) {
          const int p = base + a.found[t];
          a.used_sig[chain.sig[p]] = 0;
          int& cnt = a.author_count[a.cand_author[p]];
          cnt = max(0, cnt - 1);
        }
        s_n_used = used0;
        a.out_found[j] = 0;
        if (c.stop_on_failure) {
          *a.out_failed = j;
          failed = true;
        }
      } else {
        for (int t = 0; t < found; ++t) a.path_row[s_n_path++] = rows[a.found[t]];
        n_out += found;
        a.out_found[j] = found;
      }
    }
    if (__syncthreads_or(failed)) break;
  }
  // distances between consecutive songs of the path, the end song last
  const int np = s_n_path;
  for (int t = warp; t < np; t += warps) {
    const int64_t r0 = a.path_row[t], r1 = t + 1 < np ? a.path_row[t + 1] : a.end_row;
    const double dist = path_distance(a.X + r0 * a.d, a.X + r1 * a.d, a.d, c.path_metric, lane);
    if (lane == 0) a.out_dist[t] = dist;
  }
  if (tid == 0) {
    *a.n_used = s_n_used;
    *a.n_path = np;
  }
}

// ---------------------------------------------------------------- Song Alchemy on device
// song_alchemy (tasks/song_alchemy.py:371-1115) between its centroids and its projection, in one CTA:
//   * the by-vector chain (ByVectorChain) over the add centroid's k-NN list, cut at [:n] (n = 3 n_results,
//     voyager_manager.py:1657); skipped for the single-song temperature-0 branch (:423-427), whose list is the
//     reference's find_nearest_neighbors_by_id;
//   * the add and subtract song rows are taken out (:441-446);
//   * the subtract filter (:448-486): d(sub, v) >= threshold keeps the candidate, otherwise it is filtered out;
//   * the distance to the add centroid (:916-930).
// The centroids are float64, as the reference's means of float64 copies are.  Both distances are song_alchemy's own
// (not get_distance's): angular arccos(clip(c / (|c| or 1) . v / (|v| or 1))) / pi, so a zero vector is at 0.5, and
// euclidean ||c - v||, in float64 from the stored rows.  The chain is the walk; the rest is one warp per chain survivor.
constexpr int kAlchemyThreads = 512;

struct AlchemyArgs {
  const float* X;
  int64_t N;
  int d;
  int m;                    // candidates
  const double* add_c;      // [d]
  const double* sub_c;      // [d] or null: no subtract filter
  ByVectorChain chain;      // kept: [m]
  const int64_t* excl_row;  // [n_excl]
  int n_excl;
  am_alchemy_cfg cfg;
  int32_t* out_count;       // the chain's survivors
  int32_t* out_pos;         // [min(m, n)] their positions in the candidate arrays, in order
  unsigned char* out_status;  // [min(m, n)] 0 taken out, 1 kept, 2 filtered out
  double* out_dsub;         // [min(m, n)]
  double* out_dadd;         // [min(m, n)]
  float* out_rows;          // [min(m, n), d] or null
};

// song_alchemy's distance from centroid c (float64) to stored row v, one warp
__device__ __forceinline__ double alchemy_distance(const double* c, const float* v, int d, int metric, int lane) {
  const Moments m = warp_moments(c, v, d, lane);
  if (metric == kMetricL2) return sqrt(m.d2);
  const double nc = sqrt(m.na), nv = sqrt(m.nb);
  const double cs = m.dot / ((nc == 0.0 ? 1.0 : nc) * (nv == 0.0 ? 1.0 : nv));
  return acos(fmin(1.0, fmax(-1.0, cs))) / CUDART_PI;
}

__global__ void __launch_bounds__(kAlchemyThreads) alchemy_kernel(const AlchemyArgs a) {
  __shared__ int s_n;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, warps = kAlchemyThreads / 32;
  const am_alchemy_cfg& c = a.cfg;
  if (c.skip_chain) {
    for (int i = tid; i < a.m; i += kAlchemyThreads) a.out_pos[i] = i;
    if (tid == 0) s_n = a.m;
  } else {
    int n = 0;  // thread 0: survivors
    FilterWindow w(a.X, a.N, a.d, c.voyager_metric, c.filter_threshold, c.filter_lookback, c.filter_batch, a.m,
                   a.chain.kept);
    walk_list(w, a.m, [&](int i) { return a.chain.row[i]; }, NoExtra{}, [&](int i, int64_t, bool, bool pass, int) {
      if (a.chain.step(0, i, pass, true, c.voyager_cap)) a.out_pos[n++] = i;
      return n >= c.n;
    });
    if (tid == 0) s_n = n;
  }
  __syncthreads();
  const int n = s_n;
  for (int t = warp; t < n; t += warps) {
    const int64_t row = a.chain.row[a.out_pos[t]];
    bool out = row < 0 || row >= a.N;  // no vector: the subtract filter skips it (:465), the distances do (:921)
    for (int e = 0; e < a.n_excl && !out; ++e) out = a.excl_row[e] == row;
    unsigned char status = 0;
    double dsub = 0.0, dadd = 0.0;
    if (!out) {
      const float* v = a.X + row * a.d;
      dadd = alchemy_distance(a.add_c, v, a.d, c.path_metric, lane);
      status = 1;
      if (a.sub_c) {
        dsub = alchemy_distance(a.sub_c, v, a.d, c.path_metric, lane);
        if (!(dsub >= c.subtract_threshold)) status = 2;
      }
      if (a.out_rows)
        for (int k = lane; k < a.d; k += 32) a.out_rows[(int64_t)t * a.d + k] = v[k];
    }
    if (lane == 0) {
      a.out_status[t] = status;
      a.out_dsub[t] = dsub;
      a.out_dadd[t] = dadd;
    }
  }
  if (tid == 0) *a.out_count = n;
}


// ---------------------------------------------------------------- plain similar-tracks requests on device
// find_nearest_neighbors_by_id without the radius walk (voyager_manager.py:1493-1545) and
// find_nearest_neighbors_by_vector (:1589-1657) after their k-NN query, in one CTA: the by-vector chain (ByVectorChain)
// over the request's list in k-NN order, stopping once n items have passed ([:n]).  A by-id request differs in three
// places:
//   * its target goes first into _filter_by_distance at distance 0 (:1497-1502): it is item 0 of the walk, a member of
//     the window only (the list it heads is one longer, which moves the batch boundaries) and never output (:1505);
//   * the dedupe starts with the target's signature already seen (:662-665);
//   * the mood stage (:1508-1514, _filter_by_mood_similarity :714-822) runs between the dedupe and the cap when the
//     caller passes a mood table: a candidate without parsed features is dropped, otherwise its mood distance
//     sum(|target[f] - cand[f]|) / 6 over the six features, summed in float64 as Python's sum() does (mood_distance),
//     must be <= the threshold.
constexpr int kSimilarThreads = 512;
constexpr int kMoodFeatures = 6;  // danceable, aggressive, happy, party, relaxed, sad (:775)

struct SimilarArgs {
  const float* X;
  int64_t N;
  int d;
  int m;                          // candidates
  int n;                          // the request's n
  int64_t target_row;             // -1: a by-vector request
  int target_sig;                 // the signature seen before the first candidate, -1: none
  ByVectorChain chain;            // kept: [m + 1]
  const double* mood;             // [m, 6] the candidates' features, or null: no mood stage
  const unsigned char* mood_ok;   // [m] 1: the candidate's features parsed
  const double* target_mood;      // [6]
  am_similar_cfg cfg;
  int32_t* out_count;
  int32_t* out_pos;               // [min(m, n)] the survivors' positions in the candidate arrays, in order
  double* out_mood;               // [min(m, n)] their mood distances (mood stage only)
};

// the normalised mood distance of :789-795, sum(|t - c|) / 6, with Python's sum() of floats and no contraction:
// CPython >= 3.12 (compensated = 1) starts from the first term and adds the others with Neumaier's compensation, added
// back at the end when it is non-zero and finite; older versions add left to right.
__device__ __forceinline__ double mood_distance(const double* t, const double* c, int compensated) {
  double s = fabs(__dsub_rn(t[0], c[0])), comp = 0.0;
#pragma unroll
  for (int f = 1; f < kMoodFeatures; ++f) {
    const double x = fabs(__dsub_rn(t[f], c[f])), u = __dadd_rn(s, x);
    if (compensated)
      comp = __dadd_rn(comp, fabs(s) >= fabs(x) ? __dadd_rn(__dsub_rn(s, u), x) : __dadd_rn(__dsub_rn(x, u), s));
    s = u;
  }
  if (comp != 0.0 && isfinite(comp)) s = __dadd_rn(s, comp);
  return __ddiv_rn(s, (double)kMoodFeatures);
}

__global__ void __launch_bounds__(kSimilarThreads) similar_kernel(const SimilarArgs a) {
  const am_similar_cfg& c = a.cfg;
  const int by_id = a.target_row >= 0 ? 1 : 0;
  const int L = a.m + by_id;  // the list _filter_by_distance sees
  int n = 0;                  // thread 0: survivors
  if (threadIdx.x == 0 && a.target_sig >= 0) a.chain.seen[a.target_sig] = 0;
  FilterWindow w(a.X, a.N, a.d, c.metric, c.filter_threshold, c.filter_lookback, c.filter_batch, L, a.chain.kept);
  walk_list(
      w, L, [&](int i) { return by_id && i == 0 ? a.target_row : a.chain.row[i - by_id]; }, NoExtra{},
      [&](int i, int64_t, bool, bool pass, int) {
        const int p = i - by_id;
        if (p < 0) return false;  // the target
        bool mood = true;
        double md = 0.0;
        if (a.mood) {
          mood = a.mood_ok[p] != 0;
          if (mood) {
            md = mood_distance(a.target_mood, a.mood + (int64_t)p * kMoodFeatures, c.mood_sum);
            mood = md <= c.mood_threshold;
          }
        }
        if (a.chain.step(0, p, pass, mood, c.cap)) {
          a.out_pos[n] = p;
          if (a.out_mood) a.out_mood[n] = md;
          ++n;
        }
        return n >= a.n;
      });
  if (threadIdx.x == 0) *a.out_count = n;
}

}  // namespace am


using namespace am;

extern "C" int am_knn_filter_by_distance(const am_index* idx, const int64_t* ids, int n_lists, int n, float threshold,
                                         int lookback, int batch, unsigned char* keep) {
  AM_CHECK(idx && (ids || n_lists * n == 0) && (keep || n_lists * n == 0), "am_knn_filter_by_distance: NULL argument");
  AM_CHECK(n_lists >= 0 && n >= 0 && n <= kFilterCap, "am_knn_filter_by_distance: list length %d exceeds %d", n, kFilterCap);
  AM_CHECK(batch > 0, "am_knn_filter_by_distance: batch must be positive");
  if (n_lists == 0 || n == 0) return AM_OK;
  if (lookback <= 0) {  // the reference returns the list unchanged
    std::memset(keep, 1, (size_t)n_lists * n);
    return AM_OK;
  }
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, kStageLimit, HostCall::Memory::Pool);
  int64_t* d_ids;
  unsigned char* d_keep;
  call.up(&d_ids, ids, (size_t)n_lists * n);
  call.down(&d_keep, (size_t)n_lists * n, keep);
  AM_TRY(call.start());
  AM_LAUNCH(filter_by_distance_kernel, n_lists, kFilterThreads, 0, st, idx->X.p, idx->N, idx->d, idx->metric, d_ids, n,
            (double)threshold, lookback, batch, d_keep);
  return call.finish();
}

extern "C" int am_knn_radius_walk(const am_index* idx, const float* anchor, const int64_t* rows, const int32_t* artists,
                                  int n_cand, int n, int eliminate_duplicates, int max_songs_per_artist, int metric,
                                  int32_t* out_pos, double* out_dist, int32_t* out_count) {
  AM_CHECK(idx && anchor && out_count && (n_cand == 0 || (rows && artists)) && (n == 0 || (out_pos && out_dist)),
           "am_knn_radius_walk: NULL argument");
  AM_CHECK(n_cand >= 0 && n >= 0, "am_knn_radius_walk: negative size (n_cand = %d, n = %d)", n_cand, n);
  AM_CHECK(metric == kMetricCos || metric == kMetricL2, "am_knn_radius_walk: metric %d is not 0 (angular) or 1 (euclidean)",
           metric);
  *out_count = 0;
  if (n_cand == 0 || n == 0) return AM_OK;
  int n_art = 0;
  for (int i = 0; i < n_cand; ++i) {
    AM_CHECK(artists[i] >= -1, "am_knn_radius_walk: artist id %d at %d is below -1", artists[i], i);
    n_art = std::max(n_art, artists[i] + 1);
  }
  int64_t npad = 1;
  while (npad < n_cand) npad <<= 1;
  const int n_out = std::min(n, n_cand);
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, HostCall::kAlways, HostCall::Memory::Pool);
  float* d_anchor;
  int64_t* d_rows;
  int32_t *d_art, *d_cnt, *d_pos;
  double* d_dist;
  unsigned long long* d_key;
  int *d_ord, *d_count, *d_buckets, *d_mark, *d_playlist;
  call.up(&d_anchor, anchor, (size_t)idx->d);
  call.up(&d_rows, rows, (size_t)n_cand);
  call.up(&d_art, artists, (size_t)n_cand);
  call.down(&d_cnt, 1);
  call.down(&d_pos, (size_t)n_out);
  call.down(&d_dist, (size_t)n_out);
  call.device(&d_key, (size_t)npad);
  call.device(&d_ord, (size_t)npad);
  call.device(&d_count, (size_t)n_art, 0);
  call.device(&d_buckets, (size_t)n_art, 0);
  call.device(&d_mark, (size_t)n_art, 0xff);  // -1: no bucket yet
  call.device(&d_playlist, (size_t)n_out);
  AM_TRY(call.start());
  const int rules = eliminate_duplicates && max_songs_per_artist > 0;
  AM_LAUNCH(radius_walk_kernel, 1, kWalkThreads, 0, st, idx->X.p, idx->N, idx->d, metric, d_anchor, d_rows, d_art,
            n_cand, n_out, rules, max_songs_per_artist, npad, d_key, d_ord, d_count, d_buckets, d_mark, d_playlist, d_pos,
            d_dist, d_cnt);
  AM_TRY(call.finish());
  const int32_t cnt = *call.mirror(d_cnt);
  call.get(out_pos, d_pos, (size_t)cnt);
  call.get(out_dist, d_dist, (size_t)cnt);
  *out_count = cnt;
  return AM_OK;
}

// The by-vector chain's candidates of one host call: check() validates them with the chain's metric and filter batch,
// declare() puts their uploads and the chain's scratch on the call.
struct ChainHost {
  const char* fn;  // the entry point, for messages
  int n_cand;
  const int64_t* rows;
  const int32_t* sig;  // -1: no details, else < n_sig
  const int32_t* raw;  // -1: falsy author
  int n_sig;
  int n_raw = 0;  // raw-author keys, found by check()

  int check(int metric, int filter_batch) {
    AM_CHECK(metric == kMetricCos || metric == kMetricL2, "%s: metric %d is not 0 (angular) or 1 (euclidean)", fn,
             metric);
    AM_CHECK(filter_batch > 0, "%s: filter_batch must be positive", fn);
    AM_CHECK(n_cand >= 0 && n_sig >= 0, "%s: negative size", fn);
    AM_CHECK(n_cand == 0 || (rows && sig && raw), "%s: NULL candidates", fn);
    for (int i = 0; i < n_cand; ++i) {
      AM_CHECK(sig[i] >= -1 && sig[i] < n_sig && raw[i] >= -1, "%s: candidate %d has a key out of range", fn, i);
      n_raw = std::max(n_raw, raw[i] + 1);
    }
    return AM_OK;
  }

  // n_kept: the longest list the filter window walks
  void declare(HostCall& call, ByVectorChain* c, size_t n_kept) const {
    call.up(&c->row, rows, (size_t)n_cand);
    call.up(&c->sig, sig, (size_t)n_cand);
    call.up(&c->raw, raw, (size_t)n_cand);
    call.device(&c->kept, n_kept);
    call.device(&c->seen, (size_t)n_sig, 0xff);  // -1: no list let the signature through yet
    call.device(&c->raw_mark, (size_t)n_raw, 0xff);
    call.device(&c->raw_count, (size_t)n_raw);
  }
};

extern "C" int am_knn_song_path(const am_index* idx, const am_song_path_cfg* cfg, int n_jobs, const int32_t* job_off,
                                const int32_t* job_n, const int32_t* job_need, const int64_t* cand_rows,
                                const int32_t* cand_sig, const int32_t* cand_author, const int32_t* cand_author_raw,
                                int n_sig, int n_author, int64_t* used_rows, int32_t* n_used, unsigned char* used_sig,
                                int32_t* author_count, int64_t* path_rows, int32_t* n_path, int64_t end_row,
                                int32_t* out_found, int32_t* out_pos, int32_t* out_failed, double* out_dist) {
  AM_CHECK(idx && cfg && n_used && n_path && out_failed && (n_jobs == 0 || (job_off && job_n && job_need && out_found)),
           "am_knn_song_path: NULL argument");
  AM_CHECK(n_jobs >= 0 && n_sig >= 0 && n_author >= 0 && *n_used >= 0 && *n_path >= 1,
           "am_knn_song_path: negative size, or no start song in the path");
  AM_CHECK(cfg->path_metric == kMetricCos || cfg->path_metric == kMetricL2, "am_knn_song_path: path_metric %d",
           cfg->path_metric);
  AM_CHECK(end_row >= 0 && end_row < idx->N, "am_knn_song_path: end row %lld out of range", (long long)end_row);
  AM_CHECK(n_jobs == 0 || job_off[0] == 0, "am_knn_song_path: job_off[0] must be 0");
  int64_t total_need = 0;
  int max_m = 0;
  for (int j = 0; j < n_jobs; ++j) {
    AM_CHECK(job_off[j + 1] >= job_off[j] && job_n[j] >= 1 && job_need[j] >= 1,
             "am_knn_song_path: job %d: bad range, n or num_to_find", j);
    total_need += job_need[j];
    max_m = std::max(max_m, job_off[j + 1] - job_off[j]);
  }
  const int n_cand = n_jobs ? job_off[n_jobs] : 0;
  ChainHost chain{"am_knn_song_path", n_cand, cand_rows, cand_sig, cand_author_raw, n_sig};
  AM_TRY(chain.check(cfg->voyager_metric, cfg->filter_batch));
  AM_CHECK(n_cand == 0 || cand_author, "am_knn_song_path: NULL candidates");
  AM_CHECK(total_need == 0 || out_pos, "am_knn_song_path: NULL out_pos");
  for (int i = 0; i < n_cand; ++i)
    AM_CHECK(cand_author[i] >= 0 && cand_author[i] < n_author, "am_knn_song_path: candidate %d has a key out of range", i);
  const int nu = *n_used, np = *n_path;
  for (int t = 0; t < np; ++t)
    AM_CHECK(path_rows[t] >= 0 && path_rows[t] < idx->N, "am_knn_song_path: path row %d out of range", t);
  const int64_t cap_used = nu + total_need, cap_path = np + total_need;
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, HostCall::kAlways, HostCall::Memory::Pool);
  SongPathArgs a{idx->X.p, idx->N, idx->d, n_jobs};
  a.end_row = end_row;
  a.cfg = *cfg;
  int32_t* d_hdr;  // n_used, n_path, failed
  const int32_t hdr[4] = {nu, np, -1, 0};
  call.up(&a.job_off, job_off, n_jobs ? (size_t)n_jobs + 1 : 0);
  call.up(&a.job_n, job_n, (size_t)n_jobs);
  call.up(&a.job_need, job_need, (size_t)n_jobs);
  call.up(&a.cand_author, cand_author, (size_t)n_cand);
  chain.declare(call, &a.chain, (size_t)max_m);
  call.both(&d_hdr, hdr, 4, 4);
  call.both(&a.used_row, used_rows, (size_t)nu, (size_t)cap_used);
  call.both(&a.path_row, path_rows, (size_t)np, (size_t)cap_path);
  call.both(&a.author_count, author_count, (size_t)n_author, (size_t)n_author, author_count);
  call.both(&a.used_sig, used_sig, (size_t)n_sig, (size_t)n_sig, used_sig);
  call.down(&a.out_found, (size_t)n_jobs, out_found);
  call.down(&a.out_pos, (size_t)total_need);
  call.down(&a.out_dist, (size_t)cap_path);
  call.device(&a.found, (size_t)max_m);
  AM_TRY(call.start());
  a.n_used = d_hdr;
  a.n_path = d_hdr + 1;
  a.out_failed = d_hdr + 2;
  AM_LAUNCH(song_path_kernel, 1, kPathThreads, 0, st, a);
  AM_TRY(call.finish());
  const int32_t* out_hdr = call.mirror(d_hdr);
  int64_t taken = 0;
  for (int j = 0; j < n_jobs; ++j) taken += out_found[j];
  AM_CHECK(out_hdr[0] >= nu && out_hdr[0] <= cap_used && out_hdr[1] >= np && out_hdr[1] <= cap_path && taken <= total_need,
           "am_knn_song_path: inconsistent result (used %d of %lld, path %d of %lld, taken %lld of %lld)", out_hdr[0],
           (long long)cap_used, out_hdr[1], (long long)cap_path, (long long)taken, (long long)total_need);
  *n_used = out_hdr[0];
  *n_path = out_hdr[1];
  *out_failed = out_hdr[2];
  call.get(out_pos, a.out_pos, (size_t)taken);
  call.get(used_rows, a.used_row, (size_t)out_hdr[0]);
  call.get(path_rows, a.path_row, (size_t)out_hdr[1]);
  call.get(out_dist, a.out_dist, (size_t)out_hdr[1]);
  return AM_OK;
}

extern "C" int am_knn_alchemy(const am_index* idx, const am_alchemy_cfg* cfg, const double* add_centroid,
                              const double* sub_centroid, int n_cand, const int64_t* cand_rows, const int32_t* cand_sig,
                              const int32_t* cand_author_raw, int n_sig, int n_excl, const int64_t* excl_rows,
                              int32_t* out_count, int32_t* out_pos, unsigned char* out_status, double* out_dsub,
                              double* out_dadd, float* out_rows) {
  AM_CHECK(idx && cfg && add_centroid && out_count && (n_excl == 0 || excl_rows), "am_knn_alchemy: NULL argument");
  AM_CHECK(cfg->path_metric == kMetricCos || cfg->path_metric == kMetricL2, "am_knn_alchemy: path_metric %d",
           cfg->path_metric);
  AM_CHECK(cfg->n >= 1 && cfg->n <= AM_ALCHEMY_MAX_N, "am_knn_alchemy: n = %d is outside [1, %d]", cfg->n,
           AM_ALCHEMY_MAX_N);
  AM_CHECK(n_cand >= 0 && n_cand <= AM_ALCHEMY_MAX_CANDIDATES && (!cfg->skip_chain || n_cand <= cfg->n),
           "am_knn_alchemy: %d candidates (at most %d, and at most n without the chain)", n_cand,
           AM_ALCHEMY_MAX_CANDIDATES);
  AM_CHECK(n_excl >= 0, "am_knn_alchemy: negative size");
  ChainHost chain{"am_knn_alchemy", n_cand, cand_rows, cand_sig, cand_author_raw, n_sig};
  AM_TRY(chain.check(cfg->voyager_metric, cfg->filter_batch));
  const int n_out = std::min(n_cand, cfg->n);
  AM_CHECK(n_out == 0 || (out_pos && out_status && out_dsub && out_dadd), "am_knn_alchemy: NULL output");
  *out_count = 0;
  if (n_cand == 0) return AM_OK;
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, HostCall::kAlways, HostCall::Memory::Pool);
  AlchemyArgs a{idx->X.p, idx->N, idx->d, n_cand};
  a.n_excl = n_excl;
  a.cfg = *cfg;
  call.up(&a.add_c, add_centroid, (size_t)idx->d);
  call.up(&a.sub_c, sub_centroid, sub_centroid ? (size_t)idx->d : 0);
  chain.declare(call, &a.chain, (size_t)n_cand);
  call.up(&a.excl_row, excl_rows, (size_t)n_excl);
  call.down(&a.out_count, 1);
  call.down(&a.out_pos, (size_t)n_out);
  call.down(&a.out_status, (size_t)n_out);
  call.down(&a.out_dsub, (size_t)n_out);
  call.down(&a.out_dadd, (size_t)n_out);
  call.down(&a.out_rows, out_rows ? (size_t)n_out * idx->d : 0);
  AM_TRY(call.start());
  if (!sub_centroid) a.sub_c = nullptr;
  if (!out_rows) a.out_rows = nullptr;
  AM_LAUNCH(alchemy_kernel, 1, kAlchemyThreads, 0, st, a);
  AM_TRY(call.finish());
  const int32_t cnt = *call.mirror(a.out_count);
  AM_CHECK(cnt >= 0 && cnt <= n_out, "am_knn_alchemy: inconsistent result (%d of at most %d)", cnt, n_out);
  call.get(out_pos, a.out_pos, (size_t)cnt);
  call.get(out_status, a.out_status, (size_t)cnt);
  call.get(out_dsub, a.out_dsub, (size_t)cnt);
  call.get(out_dadd, a.out_dadd, (size_t)cnt);
  if (out_rows) call.get(out_rows, a.out_rows, (size_t)cnt * idx->d);
  *out_count = cnt;
  return AM_OK;
}

extern "C" int am_knn_similar(const am_index* idx, const am_similar_cfg* cfg, int64_t target_row, int target_sig,
                              int n_cand, const int64_t* cand_rows, const int32_t* cand_sig,
                              const int32_t* cand_author_raw, int n_sig, const double* mood, const unsigned char* mood_ok,
                              const double* target_mood, int n, int32_t* out_count, int32_t* out_pos,
                              double* out_mood) {
  AM_CHECK(idx && cfg && out_count, "am_knn_similar: NULL argument");
  ChainHost chain{"am_knn_similar", n_cand, cand_rows, cand_sig, cand_author_raw, n_sig};
  AM_TRY(chain.check(cfg->metric, cfg->filter_batch));
  AM_CHECK(target_row >= -1 && target_row < idx->N, "am_knn_similar: target row %lld out of range",
           (long long)target_row);
  AM_CHECK(target_sig >= -1 && target_sig < n_sig, "am_knn_similar: target signature %d out of range", target_sig);
  AM_CHECK(!mood || (mood_ok && target_mood), "am_knn_similar: a mood table needs its flags and the target's features");
  const int n_out = std::max(0, std::min(n_cand, n));
  AM_CHECK(n_out == 0 || (out_pos && (!mood || out_mood)), "am_knn_similar: NULL output");
  *out_count = 0;
  if (n_out == 0) return AM_OK;
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, HostCall::kAlways, HostCall::Memory::Pool);
  SimilarArgs a{idx->X.p, idx->N, idx->d, n_cand, n, target_row, target_sig};
  a.cfg = *cfg;
  chain.declare(call, &a.chain, (size_t)n_cand + 1);
  call.up(&a.mood, mood, mood ? (size_t)n_cand * kMoodFeatures : 0);
  call.up(&a.mood_ok, mood_ok, mood ? (size_t)n_cand : 0);
  call.up(&a.target_mood, target_mood, mood ? (size_t)kMoodFeatures : 0);
  call.down(&a.out_count, 1);
  call.down(&a.out_pos, (size_t)n_out);
  call.down(&a.out_mood, mood ? (size_t)n_out : 0);
  AM_TRY(call.start());
  if (!mood) {
    a.mood = a.target_mood = nullptr;
    a.mood_ok = nullptr;
    a.out_mood = nullptr;
  }
  AM_LAUNCH(similar_kernel, 1, kSimilarThreads, 0, st, a);
  AM_TRY(call.finish());
  const int32_t cnt = *call.mirror(a.out_count);
  AM_CHECK(cnt >= 0 && cnt <= n_out, "am_knn_similar: inconsistent result (%d of at most %d)", cnt, n_out);
  call.get(out_pos, a.out_pos, (size_t)cnt);
  if (mood) call.get(out_mood, a.out_mood, (size_t)cnt);
  *out_count = cnt;
  return AM_OK;
}
