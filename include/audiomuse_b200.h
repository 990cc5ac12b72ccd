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
  int n_fft;      /* 2048 (student), 1024 (teacher, config.py:384) or 512; win_length == n_fft, periodic Hann */
  int hop;        /* 480 */
  int n_mels;     /* 128 */
  float fmin;     /* 0 */
  float fmax;     /* 14000 */
  int transpose;  /* 0: [B, n_mels, T] (student)   1: [B, T, n_mels] (teacher layout) */
  /* Zero is CLAP's mel in both trailing fields.  The MusiCNN front end of tasks/analysis.py:371-375
   * (librosa.feature.melspectrogram(sr=16000, n_fft=512, hop_length=256, n_mels=96, center=False, norm='slaney'),
   * then log10(1 + 10000 x)) is framing 1, log_mode 1; onset_strength's melspectrogram is framing 2. */
  int framing;    /* 0: reflect pad n_fft/2 (librosa center=True), T = 1 + n/hop, n > n_fft/2;
                   * 1: no padding (center=False), frame t starts at t*hop, T = 1 + (n - n_fft)/hop, n >= n_fft;
                   * 2: zero pad n_fft/2 (pad_mode='constant'), T = 1 + n/hop, n >= 1 */
  int log_mode;   /* 0: 10 log10(max(1e-10, x)) (power_to_db)   1: log10(1 + 10000 x) */
} am_mel_cfg;

typedef struct am_mel_plan am_mel_plan;
/* AM_ERR_INVALID for a framing or log_mode outside the values above */
AM_API int am_mel_plan_create(const am_mel_cfg* cfg, am_mel_plan** out);
AM_API void am_mel_plan_free(am_mel_plan* plan);
/* host-only (no GPU): the dense filterbank f32[n_mels, n_fft/2+1] the plan uploads
 * (librosa.filters.mel(htk=False, norm='slaney') semantics) */
AM_API int am_mel_filterbank(const am_mel_cfg* cfg, float* out);
/* host-only: frames T of a window of n_samples under cfg's framing; AM_ERR_INVALID for a window shorter than the
 * framing accepts */
AM_API int am_mel_num_frames(const am_mel_cfg* cfg, int n_samples);

/* pcm_is_i16 selects int16 (q / 32767.0f: PCM16 windows as produced by am_pcm_to_segments) or float32 samples.
 * host: pcm[B, n_samples] -> out f32[B, n_mels, T] (or [B, T, n_mels]) */
AM_API int am_mel_batch(const void* pcm, int pcm_is_i16, int B, int n_samples, const am_mel_cfg* cfg, float* out);
/* device: the same on a plan, stream-ordered */
AM_API int am_mel_batch_dev(const am_mel_plan* plan, const void* pcm_dev, int pcm_is_i16, int B,
                     int n_samples, float* out_dev, void* stream);

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
 * against librosa, for files that are not already at 48 kHz.
 * x f32[n_in] at sr_in -> y f32[*n_out] at sr_out, *n_out = ceil(n_in * up / down) <= cap. */
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

/* ------------------------------------------------------------------ CLAP text encoder
 * Replaces the onnxruntime session over CLAP_TEXT_MODEL_PATH (tasks/clap_analyzer.py:168-240) that
 * get_text_embedding (:577-628) and get_text_embeddings_batch (:631-687) run on
 * {'input_ids', 'attention_mask'} int64 [B, T] -> 'text_embedding' f32[B, dim].
 *
 * am_text_load takes the deployed clap_text_model.onnx (TextCLAPWrapper of query/pythorch.sh:95-127: RoBERTa, its
 * pooler, Linear -> ReLU -> Linear and F.normalize; torch.onnx.export opset 17 with constant folding), with tensor
 * data inline or in `<name>.onnx.data` next to it.  The graph is lowered to the text program (csrc/text_model.cu
 * lists the accepted patterns, eager and SDPA attention among them); any other node fails the load with its name and
 * operator in am_last_error().  No CUDA work happens before the first load. */
typedef struct am_text_model am_text_model;
AM_API int am_text_load(const char* model_path, am_text_model** out);
/* same from memory (ONNX bytes with inline tensor data) */
AM_API int am_text_load_mem(const void* blob, size_t nbytes, am_text_model** out);
/* host-only, needs no GPU: parses + lowers `model_path` and writes the program (dimensions, attention form, one line
 * per layer, pooler and projection) into buf (NUL terminated, truncated to cap); returns the size needed, or a
 * negative am_status */
AM_API int am_text_describe_file(const char* model_path, char* buf, int cap);
AM_API int am_text_embedding_dim(const am_text_model* m);
/* frees the per-(B, T) workspace; weights stay */
AM_API int am_text_release_workspace(am_text_model* m);
AM_API void am_text_free(am_text_model* m);
/* host: ids, mask int64 [B, T] -> out f32[B, dim], each row L2-normalised as the graph's F.normalize does.
 * T + pad id must stay below the model's position count (RoBERTa: T <= 512).  Same (B, T) input, same bits. */
AM_API int am_text_embed(am_text_model* m, const int64_t* ids, const int64_t* mask, int B, int T, float* out);

/* ------------------------------------------------------------------ K4: exact k-NN index
 * Replaces the voyager.Index object (voyager==2.1.0) used at tasks/voyager_manager.py:183,
 * 341-346,1397,1447,1580,1681 and tasks/clap_text_search.py:173,242,263,493.
 * metric: 0 cosine (rows are stored unit-normalised; distance = 1 - cos),
 *         1 euclidean (distance = squared L2, hnswlib convention), 2 inner product (1 - dot). */
typedef struct am_index am_index;
AM_API int am_knn_build(const float* X, int64_t N, int d, int metric, am_index** out);
AM_API int am_knn_build_dev(const float* X_dev, int64_t N, int d, int metric, void* stream, am_index** out);
AM_API void am_knn_free(am_index* idx);
/* Q f32[nq,d] -> ids i64[nq,k], dist f32[nq,k]; ascending distance, ties by lower id.
 * Exact: candidates are re-ranked with float64 accumulation.  Re-entrant.
 * mode: 0 auto, 1 force fp32 scoring pass, 2 force bf16 tensor-core filter pass */
AM_API int am_knn_query(const am_index* idx, const float* Q, int nq, int k, int mode, int64_t* ids, float* dist);
/* Device version of voyager_manager.py:526-617 (_filter_by_distance, with :487-524 for lists longer than `batch`):
 * ids i64[n_lists, n] are row ids in result order (rows outside [0, N) are dropped like missing vectors);
 * keep u8[n_lists, n] receives 1 for the items the reference's greedy walk keeps.  threshold / lookback are
 * config.DUPLICATE_DISTANCE_THRESHOLD_* / DUPLICATE_DISTANCE_CHECK_LOOKBACK (config.py:550-552), batch is
 * BATCH_SIZE_VECTOR_OPS (voyager_manager.py:63).  Distances are the reference's get_direct_distance (:99-140)
 * for the index metric (cosine / inner product: 1 - cos; euclidean: ||a - b||), in float64.  n <= 4096. */
AM_API int am_knn_filter_by_distance(const am_index* idx, const int64_t* ids, int n_lists, int n, float threshold,
                                     int lookback, int batch, unsigned char* keep);
/* The similar-tracks radius walk, voyager_manager.py:941-1367 (_execute_radius_walk), in one call: anchor f32[d];
 * rows i64[n_cand] the candidates' stored rows in the order _radius_walk_get_candidates (:842-938) leaves them (-1 or
 * any row outside [0, N): not in the index, dropped like a missing vector at :920-921); artists i32[n_cand] a dense id
 * per distinct truthy author, -1 for a falsy one.  Sorts by the anchor distance (stable, :968), walks buckets of 50
 * greedily on 0.7 d(prev) + 0.3 d(anchor) (:1166-1253) under the artist rules (one per artist per bucket, at most two
 * buckets below the cap, the cap itself; only when eliminate_duplicates and max_songs_per_artist > 0, :1120-1136),
 * stops at n songs and applies _avoid_triple_adjacent (:1287-1318).  metric: config.VOYAGER_METRIC as
 * get_direct_distance reads it (:138-142), 0 angular (1 - cos) or 1 euclidean (||a - b||), from the stored rows in
 * float64 whatever the index space.  out_pos i32[n] receives positions in `rows` in walk order, out_dist f64[n] their
 * anchor distances, *out_count how many were written (<= n).  Re-entrant. */
AM_API int am_knn_radius_walk(const am_index* idx, const float* anchor, const int64_t* rows, const int32_t* artists,
                              int n_cand, int n, int eliminate_duplicates, int max_songs_per_artist, int metric,
                              int32_t* out_pos, double* out_dist, int32_t* out_count);
/* The configuration path_manager.py and voyager_manager.py read at call time, for am_knn_song_path.  Metrics are
 * 0 angular or 1 euclidean: voyager_metric is config.VOYAGER_METRIC as get_direct_distance reads it (1 - cos),
 * path_metric config.PATH_DISTANCE_METRIC as get_distance reads it (arccos(cos) / pi). */
typedef struct am_song_path_cfg {
  int voyager_metric;
  int path_metric;
  int filter_lookback;     /* voyager_manager.DUPLICATE_DISTANCE_CHECK_LOOKBACK (<= 0: no distance filter) */
  int filter_batch;        /* voyager_manager.BATCH_SIZE_VECTOR_OPS */
  int path_lookback;       /* path_manager.DUPLICATE_DISTANCE_CHECK_LOOKBACK (<= 0: no path lookback) */
  int voyager_cap;         /* the by-vector raw-author cap: MAX_SONGS_PER_ARTIST when eliminate_duplicates, else 0 */
  int path_cap;            /* path_manager.MAX_SONGS_PER_ARTIST (<= 0: off) */
  int stop_on_failure;     /* path_fix_size: stop at the first failed job instead of skipping it */
  double filter_threshold; /* DUPLICATE_DISTANCE_THRESHOLD_* for voyager_metric */
  double path_threshold;   /* DUPLICATE_DISTANCE_THRESHOLD_* for path_metric */
} am_song_path_cfg;

/* The song path's centroid jobs, path_manager.py:180-317 (_find_best_songs_for_job) over the by-vector chain
 * (voyager_manager.py:1589-1657), in one call.  Job j's candidates are entries job_off[j] .. job_off[j+1] of the
 * candidate arrays, its k-NN prefix in order; job_n[j] is its k_search, job_need[j] its num_to_find (both >= 1).
 * Per candidate: cand_rows its stored row (-1: no vector), cand_sig a dense key of its (title, author) signature after
 * strip().lower() (-1: no details), cand_author a dense key of its normalised author, cand_author_raw a dense key of
 * its raw author (-1: falsy).  The carried state, read and updated: used_rows[*n_used] the rows taken (start and end
 * song included), used_sig[n_sig] a flag per signature, author_count[n_author] songs per normalised author,
 * path_rows[*n_path] the path so far, start song first.  used_rows and path_rows have room for sum(job_need) more.
 * Jobs run in order; a failed job gives back what it took and stops the call when cfg->stop_on_failure, else the
 * next job runs.  out_found[j] receives the songs job j took (0: failed or not run), out_pos the accepted candidates
 * (entries of the candidate arrays) in path order, *out_failed the job that stopped the call or -1, and out_dist
 * f64[*n_path] the path_metric distances between consecutive rows of path_rows followed by end_row, in float64 from
 * the stored rows.  Re-entrant. */
AM_API int am_knn_song_path(const am_index* idx, const am_song_path_cfg* cfg, int n_jobs, const int32_t* job_off,
                            const int32_t* job_n, const int32_t* job_need, const int64_t* cand_rows,
                            const int32_t* cand_sig, const int32_t* cand_author, const int32_t* cand_author_raw,
                            int n_sig, int n_author, int64_t* used_rows, int32_t* n_used, unsigned char* used_sig,
                            int32_t* author_count, int64_t* path_rows, int32_t* n_path, int64_t end_row,
                            int32_t* out_found, int32_t* out_pos, int32_t* out_failed, double* out_dist);
/* The configuration song_alchemy and voyager_manager.py read at call time, for am_knn_alchemy.  Metrics as in
 * am_song_path_cfg; path_metric is config.PATH_DISTANCE_METRIC as song_alchemy reads it (:456, :923). */
#define AM_ALCHEMY_MAX_N 600            /* 3 x config.ALCHEMY_MAX_N_RESULTS (200) */
#define AM_ALCHEMY_MAX_CANDIDATES 3000  /* the by-vector query for n = 600 with eliminate_duplicates: 600 + 4 x 600 */
typedef struct am_alchemy_cfg {
  int voyager_metric;
  int path_metric;
  int filter_lookback;        /* voyager_manager.DUPLICATE_DISTANCE_CHECK_LOOKBACK (<= 0: no distance filter) */
  int filter_batch;           /* voyager_manager.BATCH_SIZE_VECTOR_OPS */
  int voyager_cap;            /* the by-vector raw-author cap: MAX_SONGS_PER_ARTIST when eliminate_duplicates, else 0 */
  int n;                      /* the by-vector n, 3 x n_results: the chain stops at n survivors */
  int skip_chain;             /* the candidates are the final neighbour list (the single-song temperature-0 branch) */
  double filter_threshold;    /* DUPLICATE_DISTANCE_THRESHOLD_* for voyager_metric */
  double subtract_threshold;  /* the subtract filter keeps a candidate at distance >= this from the subtract centroid */
} am_alchemy_cfg;

/* Song Alchemy's candidate list, tasks/song_alchemy.py:420-486 and :916-930, in one call.  The candidates are the add
 * centroid's k-NN list in order (the by-vector chain of voyager_manager.py:1589-1657 runs on them and stops at cfg->n
 * survivors), or with cfg->skip_chain the neighbour list itself (n_cand <= cfg->n).  Per candidate: cand_rows its stored
 * row (-1: no vector), cand_sig the dense key of its (title, author) signature after strip().lower() (-1: no details),
 * cand_author_raw a dense key of its raw author (-1: falsy).  excl_rows[n_excl] are the add and subtract songs' rows:
 * they are taken out of the survivors.  add_centroid f64[d]; sub_centroid f64[d] or NULL (no subtract filter).
 * *out_count receives the chain's survivors (<= min(n_cand, cfg->n)); for each, in order: out_pos its entry in the
 * candidate arrays, out_status 1 kept, 2 filtered out (d(sub) < subtract_threshold) or 0 taken out (excluded or without
 * a vector), out_dsub and out_dadd its song_alchemy distances to the centroids in float64 (0 where not computed), and
 * out_rows f32[d] its stored row (out_rows may be NULL: nothing gathered; rows of entries taken out are not written).
 * Re-entrant. */
AM_API int am_knn_alchemy(const am_index* idx, const am_alchemy_cfg* cfg, const double* add_centroid,
                          const double* sub_centroid, int n_cand, const int64_t* cand_rows, const int32_t* cand_sig,
                          const int32_t* cand_author_raw, int n_sig, int n_excl, const int64_t* excl_rows,
                          int32_t* out_count, int32_t* out_pos, unsigned char* out_status, double* out_dsub,
                          double* out_dadd, float* out_rows);
/* The configuration voyager_manager.py reads at call time, for am_knn_similar.  metric: config.VOYAGER_METRIC as
 * get_direct_distance reads it, 0 angular (1 - cos) or 1 euclidean (||a - b||). */
typedef struct am_similar_cfg {
  int metric;
  int filter_lookback;      /* DUPLICATE_DISTANCE_CHECK_LOOKBACK (<= 0: no distance filter) */
  int filter_batch;         /* BATCH_SIZE_VECTOR_OPS */
  int cap;                  /* the raw-author cap: MAX_SONGS_PER_ARTIST when eliminate_duplicates, else 0 (off) */
  int mood_sum;             /* how the mood distance sums, as Python's sum() of floats: 1 compensated (CPython >= 3.12,
                               Neumaier), 0 left to right (older versions) */
  double filter_threshold;  /* DUPLICATE_DISTANCE_THRESHOLD_* for metric */
  double mood_threshold;    /* MOOD_SIMILARITY_THRESHOLD */
} am_similar_cfg;

/* A plain similar-tracks request after its k-NN query, in one call: find_nearest_neighbors_by_id without the radius
 * walk (voyager_manager.py:1493-1545) when target_row >= 0, find_nearest_neighbors_by_vector (:1589-1657) when it is -1.
 * The candidates are the query's list in order: cand_rows their stored rows (-1: no vector), cand_sig the dense key of
 * their (title, author) signature after strip().lower() (-1: no details), cand_author_raw a dense key of their raw
 * author (-1: falsy).  Runs the distance filter (a by-id request's target heads the list, as the first kept item of the
 * window, and is never output), the same-song dedupe (starting with signature target_sig already seen, -1: none), the
 * mood stage when mood is not NULL, the raw-author cap, and stops after n survivors.  Mood stage: mood f64[n_cand, 6]
 * holds each candidate's danceable, aggressive, happy, party, relaxed and sad (0 where missing), mood_ok u8[n_cand] 1
 * where its features parsed (0: the candidate is dropped), target_mood f64[6] the target's; a candidate is kept when
 * sum(|target - candidate|) / 6, summed in that order in float64 as cfg->mood_sum says, is <= cfg->mood_threshold.  *out_count receives the
 * survivors (<= min(n_cand, n)); out_pos their entries in the candidate arrays in order, out_mood (mood stage only)
 * their mood distances.  Re-entrant. */
AM_API int am_knn_similar(const am_index* idx, const am_similar_cfg* cfg, int64_t target_row, int target_sig,
                          int n_cand, const int64_t* cand_rows, const int32_t* cand_sig, const int32_t* cand_author_raw,
                          int n_sig, const double* mood, const unsigned char* mood_ok, const double* target_mood, int n,
                          int32_t* out_count, int32_t* out_pos, double* out_mood);
/* get_max_distance_for_id (voyager_manager.py:1660-1702) in one pass over the stored rows: of the distances
 * am_knn_query would return for `query` f32[d] with k = N, the largest float32 one, skipping exclude_row (-1: none);
 * among rows at that float32 value the one query() lists first (smaller float64 distance, then smaller row).
 * *out_row receives its row and *out_dist that float32 distance; with no other row, -1 and 0.  Deterministic. */
AM_API int am_knn_farthest(const am_index* idx, const float* query, int64_t exclude_row, int64_t* out_row,
                           float* out_dist);
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
/* Many small k-means fits at once: the clustering task's RQ batches (tasks/clustering.py:175-227, one
 * KMeans(k, init='k-means++', n_init=10) per iteration through tasks/clustering_helper.py:261-335).  Problem p has
 * N_p = row_offsets[p + 1] - row_offsets[p] rows of dims[p] features, packed row-major after problem p - 1's
 * (row_offsets i64[n_problems + 1] from 0 to n_rows), k = ks[p] and seed seeds[p].  Each problem's centres
 * f32[k, d] land at centers + center_offsets[p] (center_offsets i64[n_problems + 1], steps of k * d), its labels i32 at
 * labels + row_offsets[p], inertia f32[p] and n_iter i32[p]; kpp_rows (optional) receives the k-means++ rows,
 * i32[n_init, k] per problem, problem after problem.  Every problem's result is am_kmeans_fit's definition with the
 * same seed (column-mean shift, sklearn's tolerance, greedy k-means++ on the same SplitMix draws, Lloyd with
 * sklearn's empty-cluster rule, the first init with the strictly lowest inertia), computed by one CTA per
 * (problem, init) with every reduction in a fixed order: deterministic, and independent of the other problems of
 * the batch.  Limits per problem: 1 <= k <= N <= AM_KMEANS_BATCH_MAX_ROWS, d >= 1 and
 * max(k, 8) * (d + 1) <= AM_KMEANS_BATCH_MAX_KD (centres and sums in shared memory); AM_ERR_INVALID beyond them, as for
 * NaN / inf rows.  am_kmeans_fit serves larger problems. */
#define AM_KMEANS_BATCH_MAX_KD 24576
#define AM_KMEANS_BATCH_MAX_ROWS 1048576
AM_API int am_kmeans_fit_batch(const float* rows, const int64_t* row_offsets, int64_t n_rows, const int32_t* dims,
                               const int32_t* ks, int n_problems, int n_init, int max_iter, float tol,
                               const uint64_t* seeds, float* centers, const int64_t* center_offsets, int32_t* labels,
                               float* inertia, int32_t* n_iter, int32_t* kpp_rows);

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
 * copy of the rows so each step is one tensor-core assignment pass + one partial-sum pass when the shape allows it
 * (kmeans_use_tensor_cores in csrc/kmeans.cu; k > 128 or d > 4096 runs on CUDA cores).  X_dev must stay valid while the plan lives.  am_kmeans_plan_step is stream-ordered (no sync):
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

/* ------------------------------------------------------------------ clustering-task Gaussian mixture
 * GaussianMixture(K, covariance_type, init_params='k-means++', n_init, max_iter, tol, reg_covar).fit_predict
 * (tasks/clustering_helper._apply_clustering_model, method 'gmm'; config.GMM_COVARIANCE_TYPE, which
 * tasks/clustering_gpu.py:284-309, 385-392 and tasks/clustering_helper.py:295-302 hand to scikit-learn) in float64.
 * Synchronous.
 *   X            f64[N, d], K <= N, 1 <= d <= AM_GMM_MAX_D, 1 <= K <= AM_GMM_MAX_K,
 *                n_init K <= AM_GMM_MAX_COMPONENTS (the components of all inits are one launch dimension)
 *   covariance_type  AM_GMM_FULL, AM_GMM_DIAG, AM_GMM_TIED or AM_GMM_SPHERICAL; any other value is AM_ERR_INVALID
 *   draws        f64[n_draws]: the generator's random_sample() in order; init i uses the 1 + (K - 1)(2 + floor(ln K))
 *                doubles from i times that count (at least n_init times it)
 *   outputs      the best init's (first strictly greatest final lower bound) weights f64[K], means f64[K, d],
 *                covariances and precisions_cholesky (shapes below), lower_bounds f64[max_iter] (NaN after n_iter),
 *                n_iter, converged, best_init, labels i64[N] (argmax of one more E-step)
 *   ill_defined  1 when a full or tied Cholesky pivot of any init was <= 0 or not finite, or a diag or spherical
 *                variance was <= 0 (scikit-learn's ValueError); the other outputs are then not written
 *   optional     kpp i32[n_init, K] (k-means++ rows), init_lower_bounds f64[n_init, max_iter], init_n_iter and
 *                init_converged i32[n_init], phase_ms f32[5] (device ms of seeding, E-step, normaliser, M-step,
 *                Cholesky and inverse, from CUDA events)
 * The workspace (about n_init K (N + 3 d^2) doubles for 'full') is allocated per call on the call's own stream.
 *   covariance_type      covariances              precisions_cholesky
 *   AM_GMM_FULL          f64[K, d, d]             f64[K, d, d]          upper triangular
 *   AM_GMM_DIAG          f64[K, d]                f64[K, d]             1 / sqrt(cov), elementwise
 *   AM_GMM_TIED          f64[d, d]                f64[d, d]             upper triangular, as 'full'
 *   AM_GMM_SPHERICAL     f64[K]                   f64[K] */
#define AM_GMM_MAX_D 256
#define AM_GMM_MAX_K 512
#define AM_GMM_MAX_COMPONENTS 65535
#define AM_GMM_FULL 0
#define AM_GMM_DIAG 1
#define AM_GMM_TIED 2
#define AM_GMM_SPHERICAL 3
AM_API int am_gmm_fit(const double* X, int64_t N, int d, int K, int covariance_type, int n_init, int max_iter,
                      double tol, double reg_covar, const double* draws, int64_t n_draws, double* weights,
                      double* means, double* covariances, double* precisions_cholesky, double* lower_bounds,
                      int32_t* n_iter, int32_t* converged, int32_t* best_init, int64_t* labels, int32_t* ill_defined,
                      int32_t* kpp, double* init_lower_bounds, int32_t* init_n_iter, int32_t* init_converged,
                      float* phase_ms);

/* ------------------------------------------------------------------ track features: tempo, energy, chroma
 * The three librosa 0.11.0 calls of tasks/analysis.py:344-348 (analyze_track) for a batch of tracks:
 * beat.beat_track(y, sr)'s tempo (beat positions are not computed), feature.rms(y) and feature.chroma_stft(y, sr), all
 * with n_fft 2048, hop 512, periodic Hann, center=True and zero padding, so a track of n samples has T = 1 + n / 512
 * frames.  oracle/track_features.py states every step in float64.  A plan per sample rate; the call is synchronous.
 *   samples      f32, the tracks one after the other; offsets i64[n_tracks + 1] (offsets[0] = 0, every track >= 1
 *                sample, every sample finite: AM_ERR_INVALID before any device work otherwise)
 *   what         AM_TF_TEMPO | AM_TF_RMS | AM_TF_CHROMA: which outputs to compute (the others are not touched)
 *   tempo        f64[n_tracks]: the tempo estimate in bpm, 0 when the onset envelope is all zero
 *   rms          f32[sum T]: per-frame RMS, track i at frame offset F_i = sum_{j<i} T_j
 *   chroma       f32[12 sum T]: track i's (12, T_i) row-major chromagram at 12 F_i
 *   optional     (NULL: not returned) tuning f64[n_tracks] (the estimate_tuning result the filterbank used; with
 *                AM_TF_CHROMA), onset_env f32[sum T] and tempogram f64[n_tracks, win] (the tempogram's mean over frames;
 *                with AM_TF_TEMPO), histogram i32[n_tracks, 100] (pitch_tuning's residual counts) and threshold
 *                f32[n_tracks] (the median peak magnitude; both with AM_TF_CHROMA)
 * Bit-identical between calls, and a track's results do not depend on the other tracks of the batch.
 * am_track_features_plan_info: win = floor(8 sr / 512) tempogram lags, piptrack's bins [kmin, kmax). */
#define AM_TF_TEMPO 1
#define AM_TF_RMS 2
#define AM_TF_CHROMA 4
#define AM_TRACK_FEATURES_MIN_SR 8000
#define AM_TRACK_FEATURES_MAX_SR 48000
typedef struct am_track_features_plan am_track_features_plan;
AM_API int am_track_features_plan_create(int sr, am_track_features_plan** out);
AM_API void am_track_features_plan_free(am_track_features_plan* plan);
AM_API int am_track_features_plan_info(const am_track_features_plan* plan, int* win, int* kmin, int* kmax);
AM_API int am_track_features(const am_track_features_plan* plan, const float* samples, const int64_t* offsets,
                             int n_tracks, int what, double* tempo, float* rms, float* chroma, double* tuning,
                             float* onset_env, double* tempogram, int32_t* histogram, float* threshold);

#ifdef __cplusplus
}
#endif
#endif /* AUDIOMUSE_B200_H */
