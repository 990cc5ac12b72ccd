/*
 * audiomuse_b200.h -- C ABI of libaudiomuse_b200.so (sm_90a).
 *
 * The reference (NeptuneHub/AudioMuse-AI) has no FFI of its own: the hot path is Python
 * calling third-party wheels (librosa, onnxruntime, voyager, cuML).  Each entry point below
 * replaces one of those call sites; the Python-side binding a maintainer adds (ctypes) is
 * shown in INTEGRATION.md and lives in audiomuse-ai_b200/_lib.py.
 *
 * Conventions
 *   - every function returns 0 on success or a negative am_status; am_last_error() gives a
 *     thread-local message.  "out of memory" appears in the message for allocation failures
 *     so the reference's OOM-retry wrapper (tasks/memory_utils.py:327-426) keeps working.
 *   - `*_dev` variants take DEVICE pointers and a cudaStream_t (as void*), do not synchronise
 *     and never touch host memory; the plain variants take HOST pointers, stage through
 *     pinned buffers and return after the result is in the caller's buffer.
 *   - caller owns all buffers; opaque handles are freed by the matching *_free.
 *   - no CUDA work happens at library load: the context is created lazily by am_init or the
 *     first call (RQ workers fork per job, rq_worker.py:48-55).
 */
#ifndef AUDIOMUSE_B200_H
#define AUDIOMUSE_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define AM_API __attribute__((visibility("default")))
#else
#define AM_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef enum am_status {
  AM_OK = 0,
  AM_ERR_INVALID = -1,     /* bad argument / unsupported configuration */
  AM_ERR_CUDA = -2,        /* CUDA runtime error (message has the cudaError string) */
  AM_ERR_OOM = -3,         /* allocation failed: message contains "out of memory" */
  AM_ERR_NO_DEVICE = -4,   /* no sm_90 device visible */
  AM_ERR_IO = -5,          /* weight file unreadable / malformed */
  AM_ERR_RECALL = -6       /* fewer than k neighbours exist (voyager.RecallError) */
} am_status;

/* ------------------------------------------------------------------ lifecycle */
AM_API int am_init(int device_ordinal /* -1 = current device */);
AM_API void am_shutdown(void);
AM_API const char* am_last_error(void);
AM_API int am_version(void);
/* kernels launched by this library in the calling process since load (bench.py gpu_launches) */
AM_API uint64_t am_launch_count(void);

/* Per-launch CUDA-event timing of this library's kernels (off by default).  am_profile_report
 * writes {"kernel": {"ms": device_ms, "count": n}, ...} for the launches recorded since the last
 * report and clears them; it returns the byte length needed (call with cap = 0 to size). */
AM_API void am_profile_enable(int on);
AM_API int am_profile_report(char* buf, int cap);
/* ------------------------------------------------------------------ K1: log-mel
 * Replaces librosa.feature.melspectrogram + power_to_db as called by
 * tasks/clap_analyzer.py:438-454 (compute_mel_spectrogram).  Parameters mirror
 * config.CLAP_AUDIO_* (config.py:386-392). */
typedef struct am_mel_cfg {
  int sr;         /* 48000 */
  int n_fft;      /* 2048 (student), 1024 (teacher, config.py:384) or 512; win_length == n_fft, periodic Hann,
                   * center=True, reflect pad */
  int hop;        /* 480 */
  int n_mels;     /* 128 */
  float fmin;     /* 0 */
  float fmax;     /* 14000 */
  int transpose;  /* 0: [B, n_mels, T] (student)   1: [B, T, n_mels] (teacher layout) */
} am_mel_cfg;

typedef struct am_mel_plan am_mel_plan;
AM_API int am_mel_plan_create(const am_mel_cfg* cfg, am_mel_plan** out);
AM_API void am_mel_plan_free(am_mel_plan* plan);
/* host-only (no GPU): the dense filterbank f32[n_mels, n_fft/2+1] the plan uploads
 * (librosa.filters.mel(htk=False, norm='slaney') semantics) */
AM_API int am_mel_filterbank(const am_mel_cfg* cfg, float* out);
/* frames for a segment of n_samples: 1 + n_samples / hop */
AM_API int am_mel_num_frames(const am_mel_cfg* cfg, int n_samples);

/* host: pcm f32[B, n_samples] -> out f32[B, n_mels, T] (or [B, T, n_mels]) */
AM_API int am_mel_batch(const float* pcm, int B, int n_samples, const am_mel_cfg* cfg, float* out);
/* host: PCM16 windows as produced by am_pcm_to_segments (value q means q / 32767.0f) */
AM_API int am_mel_batch_i16(const int16_t* pcm, int B, int n_samples, const am_mel_cfg* cfg, float* out);
/* device: pcm_is_i16 selects int16 (q/32767) or float32 samples */
AM_API int am_mel_batch_dev(const am_mel_plan* plan, const void* pcm_dev, int pcm_is_i16, int B,
                     int n_samples, float* out_dev, void* stream);

/* Sibling front end on the same kernel (SURVEY 8(f) row 4): tasks/analysis.py:371-375 feeds MusiCNN with
 * librosa.feature.melspectrogram(sr=16000, n_fft=512, hop_length=256, n_mels=96, center=False, norm='slaney') and
 * log10(1 + 10000 x).  center: 1 = reflect pad n_fft/2 (T = 1 + n/hop), 0 = frame t starts at t*hop
 * (T = 1 + (n - n_fft)/hop); log_mode: 0 = 10 log10(max(1e-10, x)), 1 = log10(1 + 10000 x). */
AM_API int am_mel_plan_create_ex(const am_mel_cfg* cfg, int center, int log_mode, am_mel_plan** out);
AM_API int am_mel_num_frames_ex(const am_mel_cfg* cfg, int center, int n_samples);
AM_API int am_mel_batch_ex(const float* pcm, int B, int n_samples, const am_mel_cfg* cfg, int center, int log_mode,
                           float* out);

/* tasks/clap_analyzer.py:502-523: clip to [-1,1], *32767 -> int16 (truncation), then the
 * 10 s / 5 s-hop windowing incl. the right-aligned tail window.  Host-side.
 * audio f32[L] -> seg i16[S, 480000]; returns S through *n_seg.  seg may be NULL to query S. */
AM_API int am_pcm_to_segments(const float* audio, int64_t L, int16_t* seg, int max_seg, int* n_seg);

/* ------------------------------------------------------------------ front end: decode + resample (SURVEY 8(f) row 1)
 * What tasks/analysis.py:170-250 (robust_load_audio_with_fallback -> librosa.load(path, sr=48000, mono=True,
 * duration=AUDIO_LOAD_TIMEOUT)) does before tasks/clap_analyzer.py:495 sees a waveform, for RIFF/WAVE files: PCM 8 /
 * 16 / 24 / 32 bit and IEEE float 32 / 64 (also WAVE_FORMAT_EXTENSIBLE), any channel count, any sample rate.  Other
 * containers stay with the reference's own pydub / ffmpeg loader.  Host-only (no GPU) unless noted. */
/* bits < 0: IEEE float of -bits bits */
AM_API int am_wav_info(const char* path, int* sample_rate, int* channels, int64_t* frames, int* bits);
/* mono float32 by the channel mean (librosa.to_mono), integers scaled by 1 / 2^(bits-1) (libsndfile's float read);
 * at most max_frames frames (< 0: all; librosa's `duration`).  out == NULL: only *n_frames / *sample_rate are set. */
AM_API int am_wav_decode_mono(const char* path, int64_t max_frames, float* out, int64_t cap, int64_t* n_frames,
                              int* sample_rate);
/* 48 kHz WAV file -> the reference's int16 windows in one call (decode + am_pcm_to_segments; no GPU).  seg == NULL: only
 * *n_seg / *duration_sec.  AM_ERR_INVALID ("needs resampling") for any other rate. */
AM_API int am_wav_to_segments(const char* path, double max_seconds, int16_t* seg, int max_seg, int* n_seg,
                              double* duration_sec);
/* Device polyphase resampler: the algorithm of scipy.signal.resample_poly(x, up, down) with up / down = sr_out / sr_in
 * reduced (44.1 kHz -> 48 kHz: 160 / 147), Kaiser(5.0)-windowed sinc of half length 10 max(up, down), float64
 * accumulation.  librosa resamples with soxr_hq, which cannot be installed here: parity is pinned against scipy, NOT
 * against librosa, for files that are not already at 48 kHz. */
typedef struct am_resample_plan am_resample_plan;
AM_API int am_resample_plan_create(int sr_in, int sr_out, am_resample_plan** out);
AM_API void am_resample_plan_free(am_resample_plan* plan);
AM_API int64_t am_resample_out_len(const am_resample_plan* plan, int64_t n_in); /* ceil(n_in * up / down) */
/* host-only: the plan's polyphase table poly f32[up, taps] (poly == NULL: sizes only) and its output offset; output
 * sample k is sum_i poly[t % up, i] * x[t / up - i] with t = (k + pre_remove) * down */
AM_API int am_resample_filter(int sr_in, int sr_out, float* poly, int cap, int* up, int* down, int* taps,
                              int64_t* pre_remove);
AM_API int am_resample_dev(const am_resample_plan* plan, const float* x_dev, int64_t n_in, float* y_dev, void* stream);
AM_API int am_resample(const float* x, int64_t n_in, int sr_in, int sr_out, float* y, int64_t cap, int64_t* n_out);
/* windows a waveform of L samples at 48 kHz produces (tasks/clap_analyzer.py:510-521) */
AM_API int am_num_segments(int64_t L);
/* device form of am_pcm_to_segments: audio f32[L] in HBM -> seg i16[S, 480000] in HBM (clip, * 32767, truncation,
 * 10 s windows every 5 s + the right-aligned tail window); seg_dev == NULL only reports S */
AM_API int am_audio_to_segments_dev(const float* audio_dev, int64_t L, int16_t* seg_dev, int max_seg, int* n_seg,
                                    void* stream);

/* ------------------------------------------------------------------ K2+K3: audio encoder
 * Replaces onnxruntime.InferenceSession(CLAP_AUDIO_MODEL_PATH).run(None, {'mel_spectrogram': mel})
 * (tasks/clap_analyzer.py:109-116,534) plus the numpy pooling at :552-562.
 *
 * am_clap_load takes the file the reference deploys: an ONNX ModelProto as written by
 * torch.onnx.export(opset 17, constant folding, input 'mel_spectrogram' f32[1,1,n_mels,T];
 * student_clap/models/student_onnx_model.py:611-626), with tensor data inline or in an external-data file next
 * to it (the `model.onnx.data` case of clap_analyzer.py:132-147).  The graph is read by hand (no onnx / protobuf
 * dependency) and LOWERED, node by node, to the engine's layer program (csrc/onnx_model.cu lists the supported
 * operators and patterns); a node outside that set fails the load with its name and operator in am_last_error().
 * A private "AMW1" blob (audiomuse-ai_b200/weights.py, from a StudentCLAPAudio state_dict) is accepted too. */
typedef struct am_model am_model;
AM_API int am_clap_load(const char* model_path, am_model** out);
/* same from memory (ONNX bytes without external data, or an AMW1 blob) */
AM_API int am_clap_load_mem(const void* blob, size_t nbytes, am_model** out);
/* host-only, needs no GPU: parses + lowers `model_path` and writes one text line per layer / head operation of the
 * resulting program into buf (NUL terminated, truncated to cap); returns the size needed, or a negative am_status */
AM_API int am_clap_describe_file(const char* model_path, char* buf, int cap);
/* frees the model's workspace (activations, staging buffers); weights stay.  The cleanup step of the reference's
 * OOM retry (tasks/clap_analyzer.py:536-549, memory_utils.py:327-426): clean up, then run the same call once more */
AM_API int am_clap_release_workspace(am_model* m);
AM_API void am_clap_free(am_model* m);
AM_API int am_clap_embedding_dim(const am_model* m);
AM_API int am_clap_n_mels(const am_model* m);
/* 2 * multiply-accumulates of one segment of T frames (for tensor-roofline accounting) */
AM_API double am_clap_flops_per_segment(const am_model* m, int T);

/* flops of one window executed by the GEMM kernel; the fused-block share (flops, and the algorithmic HBM
 * bytes of fused blocks) is 0 on sm_90, where every block runs layer by layer */
AM_API int am_clap_flops_split(const am_model* m, int T, double* gemm_flops, double* fused_flops,
                               double* fused_bytes);

/* host: mel f32[B,1,n_mels,T] -> out f32[B, dim], each row L2-normalised (student_onnx_model.py:285) */
AM_API int am_clap_embed(am_model* m, const float* mel, int B, int T, float* out);
AM_API int am_clap_embed_dev(am_model* m, const float* mel_dev, int B, int T, float* out_dev, void* stream);

/* Fused path: PCM16 windows -> mel -> encoder -> per-track mean + L2.
 * pcm i16[S_total, n_samples]; seg_offsets i32[n_tracks+1] (prefix sums of windows per track);
 * out f32[n_tracks, dim].  A track with zero windows yields a zero row (clap_analyzer.py:561-562). */
AM_API int am_clap_embed_tracks(am_model* m, const am_mel_cfg* cfg, const int16_t* pcm, int n_samples,
                         const int32_t* seg_offsets, int n_tracks, float* out);
/* Pipelined form of am_clap_embed_tracks for bulk analysis: _submit enqueues one batch (H2D, kernels, D2H into
 * pinned staging) and returns; _collect blocks until the OLDEST submitted batch is done and fills its `out`.
 * At most two batches in flight: the next batch's copies and early blocks overlap the previous one's tail.
 * `pcm` must stay valid until the batch is collected (pin it for a truly asynchronous H2D). */
AM_API int am_clap_embed_tracks_submit(am_model* m, const am_mel_cfg* cfg, const int16_t* pcm, int n_samples,
                                       const int32_t* seg_offsets, int n_tracks, float* out);
AM_API int am_clap_embed_tracks_collect(am_model* m);
AM_API int am_clap_embed_tracks_dev(am_model* m, const am_mel_plan* plan, const int16_t* pcm_dev,
                             int n_samples, const int32_t* seg_offsets_dev, int n_tracks,
                             int n_segments, float* out_dev, void* stream);

/* ------------------------------------------------------------------ K4: exact k-NN index
 * Replaces the voyager.Index object (voyager==2.1.0) used at tasks/voyager_manager.py:183,
 * 341-346,1397,1447,1580,1681 and tasks/clap_text_search.py:173,242,263,493.
 * metric: 0 cosine (rows are stored unit-normalised; distance = 1 - cos),
 *         1 euclidean (distance = squared L2, hnswlib convention), 2 inner product (1 - dot). */
typedef struct am_index am_index;
AM_API int am_knn_build(const float* X, int64_t N, int d, int metric, am_index** out);
AM_API int am_knn_build_dev(const float* X_dev, int64_t N, int d, int metric, void* stream, am_index** out);
AM_API void am_knn_free(am_index* idx);
AM_API int64_t am_knn_size(const am_index* idx);
AM_API int am_knn_dim(const am_index* idx);
AM_API int am_knn_get_vector(const am_index* idx, int64_t id, float* out /* [d] */);
/* Q f32[nq,d] -> ids i64[nq,k], dist f32[nq,k]; ascending distance, ties by lower id.
 * Exact: candidates are re-ranked with float64 accumulation.  Re-entrant. */
AM_API int am_knn_query(const am_index* idx, const float* Q, int nq, int k, int64_t* ids, float* dist);
/* mode: 0 auto, 1 force fp32 scoring pass, 2 force bf16 tensor-core filter pass */
AM_API int am_knn_query_ex(const am_index* idx, const float* Q, int nq, int k, int mode, int64_t* ids,
                    float* dist);
/* Device version of voyager_manager.py:526-617 (_filter_by_distance, with :487-524 for lists longer than `batch`):
 * ids i64[n_lists, n] are row ids in result order (rows outside [0, N) are dropped like missing vectors);
 * keep u8[n_lists, n] receives 1 for the items the reference's greedy walk keeps.  threshold / lookback are
 * config.DUPLICATE_DISTANCE_THRESHOLD_* / DUPLICATE_DISTANCE_CHECK_LOOKBACK (config.py:550-552), batch is
 * BATCH_SIZE_VECTOR_OPS (voyager_manager.py:63).  Distances are the reference's get_direct_distance (:99-140)
 * for the index metric (cosine / inner product: 1 - cos; euclidean: ||a - b||), in float64.  n <= 4096. */
AM_API int am_knn_filter_by_distance(const am_index* idx, const int64_t* ids, int n_lists, int n, float threshold,
                                     int lookback, int batch, unsigned char* keep);
/* Direct distances (voyager_manager.py:99-140, get_direct_distance for the index metric) between all pairs of
 * the n stored rows `ids`: out f32[n, n], symmetric; +inf where a row id is outside [0, N).  Serves the radius
 * walk / path scoring (voyager_manager.py:1166-1258) without per-candidate get_vector round trips.  n <= 8192. */
AM_API int am_knn_pairwise(const am_index* idx, const int64_t* ids, int n, float* out);
/* n stored rows in one device gather + one copy: out f32[n, d] */
AM_API int am_knn_get_vectors(const am_index* idx, const int64_t* ids, int n, float* out);
AM_API int am_knn_query_dev(const am_index* idx, const float* Q_dev, int nq, int k, int mode,
                     int64_t* ids_dev, float* dist_dev, void* stream);

/* ------------------------------------------------------------------ K5: k-means
 * Replaces cuml.cluster.KMeans(...).fit_predict (tasks/clustering_gpu.py:100-123).
 * init_centers may be NULL (k-means++ seeding from `seed`) or f32[k,d]. */
AM_API int am_kmeans_fit(const float* X, int64_t N, int d, int k, int n_init, int max_iter, float tol,
                  uint64_t seed, const float* init_centers, float* centers, int32_t* labels,
                  float* inertia, int* n_iter);
/* One Lloyd assignment pass on device data (multi-GPU hosts all-reduce sums/counts between
 * passes): labels i32[N], sums f32[k,d], counts f32[k], inertia f32[1] are OVERWRITTEN. */
AM_API int am_kmeans_assign_dev(const float* X_dev, int64_t N, int d, const float* centers_dev, int k,
                         int32_t* labels_dev, float* sums_dev, float* counts_dev,
                         float* inertia_dev, void* stream);

/* ------------------------------------------------------------------ PCA / DBSCAN (SURVEY 8(f4))
 * Replace cuml.decomposition.PCA / cuml.cluster.DBSCAN behind GPUPCA / GPUDBSCAN (tasks/clustering_gpu.py:151-278);
 * scikit-learn's results are the bar (its CPU classes are the reference's own fallback).
 * am_pca_moments: column means f64[d] and the covariance f64[d, d] (n - 1 normalisation), float64 accumulation on the
 * device; the d x d eigenproblem is the host's (LAPACK).  am_pca_project: Y f32[N, k] = (X - mean) components^T, the
 * centring done in float64 against the float64 mean. */
AM_API int am_pca_moments(const float* X, int64_t N, int d, double* mean, double* cov);
AM_API int am_pca_project(const float* X, int64_t N, int d, const double* mean, const float* components, int k, float* Y);
/* Exact brute-force DBSCAN (euclidean, eps-neighbourhood includes the point itself): labels i32[N] numbered like
 * sklearn.cluster.DBSCAN (clusters in order of their lowest core index, border points take the smallest label among
 * their core neighbours, noise -1).  A pair is a neighbour pair when its float64 squared distance is <= eps * eps in
 * float64, as in scikit-learn on the float64 copy of X.  N <= 2^20 (the neighbourhood bit matrix is N^2 / 8 bytes). */
AM_API int am_dbscan(const float* X, int64_t N, int d, double eps, int min_samples, int32_t* labels, int* n_clusters);
/* Clustering scores of tasks/clustering_helper.py:462-470 (sklearn.metrics silhouette_score, davies_bouldin_score,
 * calinski_harabasz_score; euclidean).  X f32[N, d] (1 <= d <= 8192); labels i32[N] in [0, n_labels), every label
 * present, 2 <= n_labels <= N - 1 (scikit-learn's LabelEncoder output: DBSCAN's -1 is an ordinary label there);
 * which = bit 0 silhouette, bit 1 Davies-Bouldin, bit 2 Calinski-Harabasz; scores f64[3] in that order (entries not
 * asked for are left alone); samples f32[N] optional: the per-row silhouette, caller's row order.  Silhouette runs
 * as split-bf16 tensor-core distance tiles reduced per cluster in the epilogue (only f64[N, n_labels] is stored);
 * DB / CH accumulate in float64.  Limits: N <= 2^31 - 129 (int32 permutation), and N * n_labels <= 2^31 when bit 0 is
 * set; AM_ERR_INVALID beyond them. */
AM_API int am_cluster_scores(const float* X, int64_t N, int d, const int32_t* labels, int n_labels, int which,
                             double* scores, float* samples);

/* Iterative form for Lloyd loops on device data (multi-GPU: one plan per rank over its row shard, the host all-reduces
 * sums / counts between steps; tasks/clustering_gpu.py:108-124 is the call this serves).  The plan keeps a split-bf16
 * copy of the rows so each step is one tensor-core assignment pass + one partial-sum pass (k <= 128; larger k runs on
 * CUDA cores).  X_dev must stay valid while the plan lives.  am_kmeans_plan_step is stream-ordered (no sync):
 * labels i32[N]; sums f32[k,d], counts f32[k], inertia f32[1] (each optional) are OVERWRITTEN; dist f32[N] (optional)
 * receives the squared distance of every row to its centre. */
typedef struct am_kmeans_plan am_kmeans_plan;
AM_API int am_kmeans_plan_create(const float* X_dev, int64_t N, int d, int k, void* stream, am_kmeans_plan** out);
AM_API int am_kmeans_plan_step(am_kmeans_plan* plan, const float* centers_dev, int32_t* labels_dev, float* sums_dev,
                               float* counts_dev, float* inertia_dev, float* dist_dev, void* stream);
AM_API int am_kmeans_plan_uses_tensor_cores(const am_kmeans_plan* plan);
/* diagnostic: rows the last step re-checked in exact fp32 (near-ties within the tensor-core error band); synchronises */
AM_API int am_kmeans_plan_last_recheck(am_kmeans_plan* plan, void* stream, int* n_rows);
AM_API void am_kmeans_plan_free(am_kmeans_plan* plan);

/* ------------------------------------------------------------------ spectral clustering (graph + eigensolver)
 * Replaces sklearn.cluster.SpectralClustering(affinity='nearest_neighbors') behind GPUSpectralClustering
 * (tasks/clustering_gpu.py:312-335).  The plan holds, on the device, X's k-NN graph W = 0.5 (C + C^T) without its
 * diagonal (C = kneighbors_graph(X, n_neighbors, include_self=True): exact euclidean lists of am_knn_query), dd =
 * sqrt(row sums of W) and S = D^-1/2 W D^-1/2 in float64, and a block V f64[N, block] seeded from `seed`.  The
 * host runs the subspace iteration (audiomuse-ai_b200/clustering_gpu.py, spectral_embedding): it only sees block x block
 * matrices and length-block vectors.  Every call is synchronous; a plan is used by one thread at a time.
 *   _create      X f32[N, d] (host), 2 <= n_neighbors <= N, 1 <= block <= N, N < 2^31
 *   _info        nnz of W, the block width, SpMMs run so far, device ms of the k-NN stage and of the CSR build
 *   _graph       W as CSR: indptr i64[N + 1], indices i32[nnz] (ascending per row), data f32[nnz] (0.5 or 1), and
 *                dd f64[N]; each pointer optional
 *   _iterate     Q f64[block, block] (row-major, optional): V <- V Q first.  Then V <- p(S) V, p the scaled Chebyshev
 *                polynomial of `degree` that damps [-1, cut] and is 1 at 1 (degree 0: no filter).  Returns
 *                G = V^T V and H = V^T S V, f64[block, block]
 *   _residuals   Q f64[block, ncols], theta f64[ncols]: res[c] = ||S V q_c - theta_c V q_c|| / ||V q_c|| and, optional,
 *                norms[c] = ||V q_c||, for the V of the last _iterate
 *   _embed       out f64[N, ncols] = (V Q)[i, c] / dd[i], Q f64[block, ncols] */
typedef struct am_spectral_plan am_spectral_plan;
AM_API int am_spectral_plan_create(const float* X, int64_t N, int d, int n_neighbors, int block, uint64_t seed,
                                   am_spectral_plan** out);
AM_API int am_spectral_plan_info(const am_spectral_plan* plan, int64_t* nnz, int* block, int64_t* n_spmm,
                                 float* knn_ms, float* graph_ms);
AM_API int am_spectral_plan_graph(am_spectral_plan* plan, int64_t* indptr, int32_t* indices, float* data, double* dd);
AM_API int am_spectral_plan_iterate(am_spectral_plan* plan, const double* Q, int degree, double cut, double* G,
                                    double* H);
AM_API int am_spectral_plan_residuals(am_spectral_plan* plan, const double* Q, const double* theta, int ncols,
                                      double* res, double* norms);
AM_API int am_spectral_plan_embed(am_spectral_plan* plan, const double* Q, int ncols, double* out);
AM_API void am_spectral_plan_free(am_spectral_plan* plan);
/* A plan over a given symmetric graph instead of a k-NN graph: indptr i64[N + 1], indices i32[nnz], weights f64[nnz]
 * (host; every row non-empty, every weight finite and > 0, the matrix symmetric).  dd = sqrt(row sums) and S are
 * computed in float64; _iterate / _residuals / _embed work as above (_info reports no k-NN or CSR time, and _graph
 * copies no data: the caller owns the graph).  Serves UMAP's spectral initialisation. */
AM_API int am_spectral_plan_create_csr(const int64_t* indptr, const int32_t* indices, const double* weights, int64_t N,
                                       int block, uint64_t seed, am_spectral_plan** out);

/* ------------------------------------------------------------------ UMAP graph + layout
 * Replaces umap.UMAP(n_components=2).fit_transform behind tasks/song_alchemy._project_with_umap (:272-287).  The plan
 * holds umap-learn 0.5's fuzzy simplicial set of X, pruned for n_epochs, and runs the SGD layout; the host fits a, b and
 * computes the spectral initialisation (audiomuse-ai_b200/projection.py).  Every call is synchronous; a plan is used by
 * one thread at a time.
 *   _create      X f32[N, d] (host), N >= 2, 1 <= n_neighbors <= N (the row itself counts as its first neighbour),
 *                n_epochs >= 1 (no seed: nothing in the graph is random; _layout takes it).  k-NN: exact euclidean (am_knn_query), distances recomputed in float64.  rho, sigma:
 *                smooth_knn_dist (local_connectivity 1); W = A + A^T - A o A^T; entries with w < max(w) / n_epochs
 *                dropped; epochs_per_sample = n_epochs / (n_epochs w / max(w))
 *   _info        nnz of the pruned W, n_neighbors, n_epochs, device ms of the k-NN, the graph and the last layout
 *   _graph       the pruned W as CSR (indptr i64[N + 1], indices i32[nnz] ascending per row, weights f64[nnz]), rho and
 *                sigma f64[N], epochs_per_sample f64[nnz]; each pointer optional
 *   _layout      emb f32[N, 2] in/out: the first `epochs` epochs (0 <= epochs <= n_epochs) of the n_epochs schedule,
 *                learning rate alpha0 (1 - n / n_epochs), curve a, b, repulsion gamma, neg_rate negative samples per
 *                sample.  Per-vertex updates from the previous epoch's embedding, negative samples from a hash of
 *                (seed, epoch, entry, sample): one seed gives bit-identical output on every call */
typedef struct am_umap_plan am_umap_plan;
AM_API int am_umap_plan_create(const float* X, int64_t N, int d, int n_neighbors, int n_epochs, am_umap_plan** out);
AM_API int am_umap_plan_info(const am_umap_plan* plan, int64_t* nnz, int* n_neighbors, int* n_epochs, float* knn_ms,
                             float* graph_ms, float* layout_ms);
AM_API int am_umap_plan_graph(am_umap_plan* plan, int64_t* indptr, int32_t* indices, double* weights, double* rho,
                              double* sigma, double* epochs_per_sample);
AM_API int am_umap_plan_layout(am_umap_plan* plan, float* emb, int epochs, double a, double b, double gamma,
                               double alpha0, double neg_rate, uint64_t seed);
AM_API void am_umap_plan_free(am_umap_plan* plan);

/* ------------------------------------------------------------------ artist-similarity GMM sweep
 * Replaces tasks/artist_gmm_manager.select_optimal_gmm_components (:63-126), which fit_artist_gmm (:129-216) calls:
 * for every artist and every K of its range, GaussianMixture(K, covariance_type='diag', max_iter, n_init,
 * random_state=42).fit and bic, float64 arithmetic on float32 rows (oracle/artist_gmm.py states it).  Synchronous.
 *   rows         f32[n_rows, d], the artists' rows one after the other; offsets i64[n_artists + 1] (0 .. n_rows, every
 *                artist >= 1 row); 1 <= d <= AM_ARTIST_GMM_MAX_D; every value finite
 *   k_lo, k_hi   i32[n_artists]: the K tried, 1 <= k_lo, k_hi <= AM_ARTIST_GMM_MAX_K (k_hi < k_lo: none); a K above
 *                the artist's row count fails, as scikit-learn's fit raises
 *   draws        f64[n_draws]: MT19937(seed).random_sample() in order; init i of a K-fit uses the
 *                1 + (K - 1)(2 + floor(ln K)) doubles from i times that count (at least n_init times it for the
 *                largest K)
 *   per artist   chosen_k i32 (0: every K failed), bic f64[16] and failed u8[16] per K (bic NaN where failed or not
 *                tried), lower_bound f64, n_iter i32, converged u8 [16, n_init] per (K, init) (NaN / 0 for an init
 *                that never ran), and the chosen fit's weights f32[16], means and covariances f32[16, d] (first K rows)
 *   kpp          optional i32[n_artists, 16, n_init, 16]: the k-means++ centre rows (within the artist)
 *   labels       optional i32[16, n_init, n_rows]: the k-means labels each (K, init) starts EM from
 *   phase_ms     optional f32[2]: device ms of the fits and of the selection, from CUDA events
 * Rows are staged in shared memory when n d 4 <= AM_ARTIST_GMM_SMEM_BYTES. */
#define AM_ARTIST_GMM_MAX_K 16
#define AM_ARTIST_GMM_MAX_D 1024
#define AM_ARTIST_GMM_SMEM_BYTES 98304
AM_API int am_artist_gmm_fit(const float* rows, int64_t n_rows, int d, const int64_t* offsets, int n_artists,
                             const int32_t* k_lo, const int32_t* k_hi, int n_init, int max_iter, double tol,
                             double reg_covar, const double* draws, int64_t n_draws, int32_t* chosen_k, double* bic,
                             uint8_t* failed, double* lower_bound, int32_t* n_iter, uint8_t* converged,
                             float* weights, float* means, float* covariances, int32_t* kpp, int32_t* labels,
                             float* phase_ms);

#ifdef __cplusplus
}
#endif
#endif /* AUDIOMUSE_B200_H */
