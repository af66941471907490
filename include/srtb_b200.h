/* srtb_b200.h — C ABI of libsrtb_b200.so: the H100-native drop-in for srtb's
 * baseband -> single-pulse hot path
 *   unpack -> fft_1d_r2c -> rfi_mitigation_s1 -> dedisperse -> watfft_1d_c2c
 *          -> rfi_mitigation_s2 -> signal_detect
 * (wired in the reference at userspace/src/main.cpp:170-204).
 *
 * Every entry point replaces one reference operator (file:line cited per function,
 * paths relative to /root/reference/userspace/include/srtb/). Conventions:
 *   - plain pointers and sizes only; `d_` = device pointer, `h_` = host pointer;
 *   - every call is stream-ordered on the ctx's CUDA stream and returns without
 *     synchronising, except srtb_b200_signal_detect / srtb_b200_process_block, whose
 *     outputs are host-visible (the reference `.wait()`s after every kernel; the C++
 *     pipe wrappers in include/srtb/ restore that contract in drop-in mode);
 *   - the library never allocates or frees user buffers; scratch lives in the ctx and is
 *     re-sized when a call's size differs (mirrors fft_wrapper::set_size re-planning,
 *     fft/fft_wrapper.hpp:106-113);
 *   - return value 0 = ok, negative = srtb_b200_status; text via srtb_b200_last_error.
 *   - alignment: a complex64 (float2) pointer must be 8-byte aligned, so any element of a cudaMalloc'd array
 *     (x + 1 included) is accepted; a misaligned one returns SRTB_B200_E_INVALID before any launch. 16-byte
 *     alignment only selects the faster 16-byte-load / TMA routes. Stricter rules are stated per entry below.
 *   - there is NO CPU fallback: without a CUDA device ctx_create fails;
 *   - a ctx may be shared by several host threads (the reference copies one sycl::queue into every pipe): each entry
 *     locks the ctx while it plans and enqueues, waits (synchronize, collect_block) run unlocked;
 *   - a ctx spreads the data streams of a block over two CUDA streams of its own ("lanes": its stream for the even
 *     streams, a private one for the odd ones); results are complete when process_block / collect_block returns.
 *     SRTB_B200_LANES=1 keeps everything on the ctx's stream.
 */
#ifndef SRTB_B200_H
#define SRTB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct srtb_b200_ctx srtb_b200_ctx;

typedef enum {
  SRTB_B200_OK = 0,
  SRTB_B200_E_INVALID = -1,     /* bad argument (null pointer, zero size...)          */
  SRTB_B200_E_SIZE = -2,        /* size not a power of two ("n must be a power of 2",
                                   fft/naive_fft_wrapper.hpp:52-56)                   */
  SRTB_B200_E_UNSUPPORTED = -3, /* unsupported baseband_input_bits / format
                                   (pipeline/unpack_pipe.hpp:123-127,411-412)         */
  SRTB_B200_E_CUDA = -4,        /* CUDA runtime error                                 */
  SRTB_B200_E_NOMEM = -5
} srtb_b200_status;

/* baseband formats, io/backend_registry.hpp:36-181 + pipeline/unpack_pipe.hpp:392-413 */
typedef enum {
  SRTB_B200_FORMAT_SIMPLE = 0,         /* 1 stream  (unpack_pipe)                        */
  SRTB_B200_FORMAT_INTERLEAVED_2 = 1,  /* "1 2 1 2" (unpack.hpp:221-244)                 */
  SRTB_B200_FORMAT_NAOCPSR_SNAP1 = 2,  /* "1 1 2 2" int8 (unpack.hpp:255-283)            */
  SRTB_B200_FORMAT_GZNUPSR_A1_2 = 3,   /* 4-sample words, 2 streams (unpack.hpp:338-369) */
  SRTB_B200_FORMAT_GZNUPSR_A1_4 = 4    /* 4-sample words, 4 streams, ^0x80 (:293-336)    */
} srtb_b200_format;

/* FFT windows fused into unpack, fft/fft_window.hpp:52-83 (default = rectangle) */
typedef enum { SRTB_B200_WINDOW_RECTANGLE = 0, SRTB_B200_WINDOW_HANN = 1, SRTB_B200_WINDOW_HAMMING = 2 } srtb_b200_window;

#define SRTB_B200_MAX_BOXCARS 32

/* result of signal_detect_pipe_2 (pipeline/signal_detect_pipe.hpp:252-442).
 * entry 0 is the mean-removed time series (boxcar 1), entry i the boxcar 2^i series. */
typedef struct {
  uint64_t zero_count;        /* channels whose first sample is exactly zero (:261-284)   */
  uint64_t time_series_count; /* L' = L - reserved (:288-299)                             */
  int32_t detect_enabled;     /* zero_count < channel_threshold * C (:344-345)            */
  int32_t n_boxcars;          /* entries used below                                       */
  uint64_t boxcar_length[SRTB_B200_MAX_BOXCARS];
  uint64_t series_length[SRTB_B200_MAX_BOXCARS];
  uint64_t signal_count[SRTB_B200_MAX_BOXCARS]; /* count_signal (signal_detect.hpp:32-72) */
  float variance[SRTB_B200_MAX_BOXCARS];        /* mean(v^2)                              */
  float threshold[SRTB_B200_MAX_BOXCARS];       /* snr * sqrt(variance)                   */
} srtb_b200_detect_result;

/* ---- context ------------------------------------------------------------------- */
/* replaces the `sycl::queue q` every pipe is constructed with (pipeline/framework/pipe.hpp:148-161).
 * cuda_stream: a cudaStream_t (NULL = the legacy default stream). */
int srtb_b200_ctx_create(int device, void* cuda_stream, srtb_b200_ctx** out);
int srtb_b200_ctx_destroy(srtb_b200_ctx* ctx);
int srtb_b200_ctx_set_stream(srtb_b200_ctx* ctx, void* cuda_stream);
int srtb_b200_synchronize(srtb_b200_ctx* ctx);
const char* srtb_b200_last_error(const srtb_b200_ctx* ctx); /* ctx may be NULL: last global error */
/* number of kernels this ctx has launched so far (bench.py's gpu_launches) */
uint64_t srtb_b200_launch_count(const srtb_b200_ctx* ctx);

/* ---- optional per-stage timing (SURVEY 8b: srtb_b200_stage_stats) ------------------------
 * When enabled, every stage entry point below records a CUDA-event pair around its launches on the
 * ctx stream. srtb_b200_stage_stats waits for the LAST call of `stage` and returns its duration and
 * the algorithmic bytes it moved (SURVEY 8d: unpack N*b/8 + 4N, fft_r2c 8N, rfi_s1 12N, dedisperse 8N,
 * watfft 8N, rfi_s2 4N, signal_detect 4N, N = real samples of the block), so achieved GB/s =
 * bytes / ms / 1e6. The reference has no per-pipe device timing (its pipes only .wait()); this is the
 * measurement hook SURVEY 8b proposes for the drop-in. */
typedef enum {
  SRTB_B200_STAGE_UNPACK = 0,
  SRTB_B200_STAGE_FFT_R2C = 1,
  SRTB_B200_STAGE_RFI_S1 = 2,
  SRTB_B200_STAGE_DEDISPERSE = 3,
  SRTB_B200_STAGE_WATFFT = 4,
  SRTB_B200_STAGE_RFI_S2 = 5,
  SRTB_B200_STAGE_SIGNAL_DETECT = 6,
  /* groups of the fused block path (srtb_b200_process_block / submit_block), per stream, with the bytes each
   * group MUST move (compulsory traffic of the fused form): */
  SRTB_B200_STAGE_FUSED_R2C = 7,        /* unpack + R2C + split + power mean: N*b/8 read, 4N written           */
  SRTB_B200_STAGE_FUSED_WATERFALL = 8,  /* manual zap, s1, chirp, waterfall FFT, SK, column sums: 4N + 4N        */
  SRTB_B200_STAGE_FUSED_DETECT_TAIL = 9,/* column-sum reduction, scan, boxcars (reads the partial sums only)   */
  SRTB_B200_STAGE_COUNT = 10
} srtb_b200_stage;
int srtb_b200_stage_stats_enable(srtb_b200_ctx* ctx, int on);
int srtb_b200_stage_stats(srtb_b200_ctx* ctx, int stage, double* ms, double* bytes);
const char* srtb_b200_version(void);

/* ---- unpack: srtb::unpack::unpack<BITS> and the multi-stream unpackers --------------
 * (unpack.hpp:171-197,221-244,255-283,293-403; bits dispatch pipeline/unpack_pipe.hpp:72-127)
 * bits: 1,2,4,8 unsigned; -8 int8; 16/-16; 32 float; 64 double.
 * out_count: samples PER OUTPUT STREAM; d_out[s] must hold out_count (+2 for in-place R2C) floats.
 * Alignment (else SRTB_B200_E_INVALID before any launch): SIMPLE: d_in aligned to the sample width (any byte for
 * 1/2/4/8-bit samples, 2 bytes for 16-bit, 4 for 32-bit, 8 for 64-bit), d_out[0] 4-byte aligned; the multi-stream
 * formats: d_in and every d_out[s] 16-byte aligned.
 * streams written: 1 (SIMPLE), 2 (INTERLEAVED_2, SNAP1, GZNUPSR_A1_2), 4 (GZNUPSR_A1_4). */
int srtb_b200_unpack(srtb_b200_ctx* ctx, const void* d_in, size_t in_bytes, int bits, int format,
                     int window, float* const d_out[4], size_t out_count);

/* ---- fft_1d_dispatcher<R2C_1D>::process (fft/fft.hpp:146-149; naive_fft.hpp:221-261) ----
 * in place on n_real + 2 floats: X[k], k = 0..n_real/2, unnormalised, forward sign.
 * n_real: power of two, 2 .. 2^31. d_inout is read as complex64: it must be 8-byte aligned (a float
 * pointer at +4 bytes returns SRTB_B200_E_INVALID). */
int srtb_b200_fft_r2c_inplace(srtb_b200_ctx* ctx, float* d_inout, size_t n_real);

/* ---- batched C2C, unnormalised, in place (fft_1d_dispatcher<C2C_1D_*>; naive_fft.hpp:155-176) ----
 * direction +1 forward (e^-i), -1 backward (e^+i). d_x is [batch][length] complex64, 8-byte aligned.
 * length: power of two up to 2^30; batch * length up to 2^34 (else SRTB_B200_E_SIZE). */
int srtb_b200_fft_c2c(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch, int direction);

/* watfft_1d_c2c_pipe (pipeline/fft_pipe.hpp:313-371): batch backward C2C of `length` (rules of srtb_b200_fft_c2c) */
int srtb_b200_watfft_c2c_backward(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch);

/* ---- rfi_mitigation_s1_pipe (pipeline/rfi_mitigation_pipe.hpp:43-101) ---------------
 * mean m of |X|^2; X = (|X|^2 > avg_threshold*m) ? 0 : X*norm_coef; then zero the
 * inclusive bin ranges h_bin_ranges[n_ranges][2] (spectrum/rfi_mitigation.hpp:137-143).
 * d_mean_out (optional device float) receives m. d_x: 8-byte aligned complex64. */
int srtb_b200_rfi_s1(srtb_b200_ctx* ctx, void* d_x, size_t count, float avg_threshold,
                     float norm_coef, const size_t* h_bin_ranges, size_t n_ranges,
                     float* d_mean_out);

/* host helpers mirroring the reference's host-side arithmetic for this stage */
float srtb_b200_norm_coefficient(size_t in_count, size_t spectrum_channel_count); /* rfi_mitigation_pipe.hpp:61-65 */
size_t srtb_b200_eval_rfi_ranges(const char* freq_list, float* pairs, size_t max_pairs); /* rfi_mitigation.hpp:64-88 */
int srtb_b200_rfi_range_to_bins(float f1, float f2, float freq_low, float bandwidth, size_t in_count,
                                size_t* lo, size_t* hi); /* rfi_mitigation.hpp:102-143; 1 = applied */

/* ---- coherent_dedispertion (coherent_dedispersion.hpp:133-150,223-237) ---------------
 * d_x: 8-byte aligned complex64. */
int srtb_b200_dedisperse(srtb_b200_ctx* ctx, void* d_x, size_t count, float f_min, float f_c,
                         float df, float dm);
/* nsamps_reserved (coherent_dedispersion.hpp:76-128) */
size_t srtb_b200_nsamps_reserved(size_t baseband_input_count, size_t spectrum_channel_count,
                                 float freq_low, float bandwidth, float sample_rate, float dm,
                                 int reserve_sample);

/* ---- mitigate_rfi_spectral_kurtosis_method_2 (spectrum/rfi_mitigation.hpp:292-341) ----
 * d_x is [chan_count][time_count], 8-byte aligned complex64. d_sk_out (optional, chan_count floats) receives sk. */
int srtb_b200_rfi_s2_sk(srtb_b200_ctx* ctx, void* d_x, size_t time_count, size_t chan_count,
                        float sk_threshold, float* d_sk_out);

/* ---- signal_detect_pipe_2 (pipeline/signal_detect_pipe.hpp:252-442) -------------------
 * h_series: NULL, or host buffer of SRTB_B200_MAX_BOXCARS * time_count floats; row i receives
 * the series of entry i when signal_count[i] > 0 (all entries if copy_all != 0).
 * d_x: [chan_count][time_count], 8-byte aligned complex64. Synchronises the stream. */
int srtb_b200_signal_detect(srtb_b200_ctx* ctx, const void* d_x, size_t time_count,
                            size_t chan_count, size_t time_reserved_count, float snr_threshold,
                            float channel_threshold, size_t max_boxcar_length,
                            srtb_b200_detect_result* h_result, float* h_series, int copy_all);

/* ---- alternates of the refft path (defined by the reference, not wired in its main.cpp): spectra laid out
 * [time][frequency], as refft_1d_c2c_pipe leaves them (pipeline/fft_pipe.hpp:197-278) ------------------------------
 * mitigate_rfi_spectral_kurtosis_method (v1, spectrum/rfi_mitigation.hpp:181-275, normalization = false):
 * d_x is [time_counts][fft_bins]; every frequency column whose sk = M s4 / s2^2 over the time_counts spectra leaves
 * the thresholds is zeroed. d_sk_out (optional, fft_bins floats) receives sk. d_x: 8-byte aligned complex64. */
int srtb_b200_rfi_sk_v1(srtb_b200_ctx* ctx, void* d_x, size_t fft_bins, size_t time_counts, float sk_threshold,
                        float* d_sk_out);
/* signal_detect_pipe (v1, pipeline/signal_detect_pipe.hpp:51-230): SK v1 in place, masked channels counted over the
 * first spectrum, one time-series value per spectrum (sum over its count_per_batch bins of |x|^2), mean removal,
 * count_signal, boxcars 2..max (series lengths batch_size - boxcar; nothing is trimmed). h_series rows are
 * batch_size floats apart. d_x: 8-byte aligned complex64. Synchronises the stream. */
int srtb_b200_signal_detect_v1(srtb_b200_ctx* ctx, void* d_x, size_t count_per_batch, size_t batch_size,
                               float sk_threshold, float snr_threshold, float channel_threshold,
                               size_t max_boxcar_length, srtb_b200_detect_result* h_result, float* h_series,
                               int copy_all);

/* ---- the whole path on one block (main.cpp:170-204 for one work item) -----------------
 * configuration scalars = the srtb::configs fields the path reads (config.hpp:80-249). */
typedef struct {
  uint64_t baseband_input_count; /* samples per stream per block                       */
  int32_t baseband_input_bits;
  int32_t baseband_format;       /* srtb_b200_format                                   */
  int32_t window;                /* srtb_b200_window                                   */
  int32_t baseband_reserve_sample;
  float baseband_freq_low, baseband_bandwidth, baseband_sample_rate, dm;
  float mitigate_rfi_average_method_threshold;
  float mitigate_rfi_spectral_kurtosis_threshold;
  uint64_t spectrum_channel_count;
  float signal_detect_signal_noise_threshold;
  float signal_detect_channel_threshold;
  uint64_t signal_detect_max_boxcar_length;
  const float* rfi_freq_pairs;   /* MHz pairs parsed from mitigate_rfi_freq_list        */
  uint64_t n_rfi_freq_pairs;
  int32_t signal_detect_sum_streams; /* non-zero: also detect on the streams' total intensity (below); 0 = off    */
} srtb_b200_block_config;

/* ---- the detector on total intensity (signal_detect_sum_streams != 0) ---------------------------------------------
 * A block of S >= 2 streams gets one more result, computed from the streams' final dynamic spectra x_s[C][L] (after s1,
 * the chirp, the waterfall FFT and SK, as the block leaves them). Channel c is dropped when |x_s[c][0]|^2 == 0 in any
 * stream (the zero_count proxy, so a channel SK zapped in one stream is left out of every stream); K = the kept ones.
 *   v[j] = sum_{c in K} sum_s |x_s[c][j]|^2, j < L' (the streams' time_series_count), in fp32 with a fixed operation
 * order: the same bits with one lane or two, through process_block or the ring. v then goes through the block's detector
 * unchanged (mean removal, scan, boxcars, count_signal). Its header: zero_count = C - |K|, detect_enabled by the
 * reference's rule with that count, time_series_count = L'. For an unpolarised pulse with equal noise in both
 * polarisations the sum has sqrt(2) times the S/N of either stream.
 * Every stream's own header and series are bit-identical to a call with the field 0. Where the result goes:
 *   - process_block[_device], collect_block[_ex]: h_results[streams] (h_results needs streams + 1 entries); the return
 *     value stays the stream count;
 *   - the positive series: slot `streams` of h_series, [streams + 1][SRTB_B200_MAX_BOXCARS][L] floats in all (the same
 *     for srtb_b200_block_outputs.h_series; the ring's own buffer grows to that size).
 * On the device the first lane waits for the second with an event once both streams' chains are enqueued (no host
 * synchronisation); blocks with the field 0 keep the lanes free-running. Four kernels per block.
 * Before any launch: a single-stream format returns SRTB_B200_E_INVALID; the DM sweep entries
 * (srtb_b200_process_block_dm_sweep[_ex]) return SRTB_B200_E_UNSUPPORTED. */

/* h_baseband: host (ideally pinned) bytes of one block, all streams interleaved as the
 * format says; the call copies them to the device, runs every stage for every stream and
 * fills h_results[stream] (and h_results[streams] with signal_detect_sum_streams). d_spectrum_out (optional): per-stream device pointers that
 * receive the dynamic spectrum [C][L] (else it stays in ctx scratch).
 * Returns the number of streams processed (>0) or a negative status.
 * Baseband alignment (the rules of srtb_b200_unpack): a SIMPLE baseband must be aligned to its sample width (any
 * byte address for 1/2/4/8-bit samples, 2/4/8 bytes for 16/32/64-bit ones). The two- and four-stream formats
 * (INTERLEAVED_2, NAOCPSR_SNAP1, GZNUPSR_A1_2, GZNUPSR_A1_4) need a 16-byte aligned baseband pointer. A pointer that
 * breaks the rule returns SRTB_B200_E_INVALID. The same holds for submit_block_device / submit_block_ex. */
int srtb_b200_process_block(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                            const void* h_baseband, size_t baseband_bytes,
                            srtb_b200_detect_result* h_results, float* h_series, int copy_all);
/* same, input already on the device */
int srtb_b200_process_block_device(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                   const void* d_baseband, size_t baseband_bytes,
                                   srtb_b200_detect_result* h_results, float* h_series, int copy_all);
/* DM sweep on one block (BASELINE config #4): unpack + R2C once, then per trial DM the s1-apply + chirp
 * (coherent_dedispersion.hpp:223-237, out of place), waterfall FFT, SK and detector; h_results is
 * [n_dm][streams], each entry equal to process_block with cfg->dm = h_dms[j]. The reference handles one
 * DM per run (config.hpp:132); this loops its own dedisperse..detect stages over a list. */
int srtb_b200_process_block_dm_sweep(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                     const void* baseband, size_t baseband_bytes, int on_device,
                                     const float* h_dms, size_t n_dm, srtb_b200_detect_result* h_results);
/* DM search on one block: the sweep above, which ranks its trials and hands out the best one's candidate.
 * With outputs == NULL it is srtb_b200_process_block_dm_sweep (same results, same launches). Otherwise:
 *   - every trial's detector also reduces each boxcar series v (the positive one a .tim file holds) to its peak:
 *     snr[b] = max_j v[j] / sqrt(variance[b]) (0 when the variance is 0; the detector's rule is v > snr * sqrt(var), so
 *     this S/N is on the scale of signal_detect_signal_noise_threshold) and peak_index[b] = the smallest j reaching
 *     the maximum. Boxcars beyond n_boxcars, and trials with detection disabled, keep a zero record;
 *   - each stream's best trial is chosen among the trials with detect_enabled: those with some signal_count > 0 first,
 *     then the largest max_b snr[b], then the lowest trial index; trial 0 when no trial has detection enabled;
 *   - when h_series or d_spectrum is given, the best trial runs once more per stream (one extra trial per stream per
 *     block) from the stream's kept spectrum: its dynamic spectrum [C][L] lands in d_spectrum[s] and its positive
 *     series in h_series, exactly as process_block at that DM writes them. The re-run's result header must equal the
 *     trial's in h_results bit for bit; SRTB_B200_E_CUDA if it does not.
 * A null pointer among the required arguments, n_dm == 0, a d_spectrum given for some streams but not all, or one
 * that is not 16-byte aligned returns SRTB_B200_E_INVALID before any launch. Synchronises the context's stream. */
typedef struct {
  float snr[SRTB_B200_MAX_BOXCARS];
  uint64_t peak_index[SRTB_B200_MAX_BOXCARS]; /* index into that boxcar's series */
} srtb_b200_peak;
typedef struct {
  srtb_b200_peak* h_peaks; /* [n_dm][streams], or NULL                                                          */
  int32_t* h_best_trial;   /* [streams], or NULL                                                                */
  float* h_series;         /* pinned, [streams][SRTB_B200_MAX_BOXCARS][L], or NULL: the best trial's positive series */
  float* d_spectrum[4];    /* per stream: N + 2 floats, 16-byte aligned, or all NULL: the best trial's dynamic
                              spectrum                                                                            */
} srtb_b200_sweep_outputs;
int srtb_b200_process_block_dm_sweep_ex(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband,
                                        size_t baseband_bytes, int on_device, const float* h_dms, size_t n_dm,
                                        srtb_b200_detect_result* h_results, const srtb_b200_sweep_outputs* outputs);
/* pipelined ingest (the pinned-host ring of SURVEY section 8e): submit copies the block on a
 * dedicated copy stream while the previous block computes and returns a ticket (>= 0);
 * collect waits for that block and fills h_results[stream] (returns the stream count).
 * Up to SRTB_B200_RING_SLOTS blocks may be in flight; h_baseband must stay valid (and should be
 * pinned) until its block is collected.
 *
 * What a block leaves behind is what signal_detect_pipe_2 attaches to its write_signal_work
 * (pipeline/signal_detect_pipe.hpp:347-366,405-423,431-441; work.hpp:240-260):
 *   - the dynamic spectrum [C][L] of every stream, in that stream's working buffer (the reference forwards d_in);
 *   - the host copy of every boxcar series whose count_signal is positive, written straight from the detector
 *     kernel into pinned host memory at [stream][boxcar index][L] (nothing crosses PCIe for a negative block).
 * srtb_b200_block_outputs lets the caller own those buffers (a pipe hands them to its work item, zero copy);
 * members left NULL use buffers owned by the ring slot, valid until that slot is submitted again
 * (SRTB_B200_RING_SLOTS - 1 further submissions). */
#define SRTB_B200_RING_SLOTS 3
typedef struct {
  float* d_spectrum[4]; /* per stream: device buffer of baseband_input_count + 2 floats, 16-byte aligned
                           (else submit_block_ex returns SRTB_B200_E_INVALID before it enqueues anything)        */
  float* h_series;      /* pinned (cudaMallocHost / cudaHostRegister) host buffer,
                           [streams][SRTB_B200_MAX_BOXCARS][L] floats; only positive series are written          */
} srtb_b200_block_outputs;
int srtb_b200_submit_block(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                           const void* h_baseband, size_t baseband_bytes);
int srtb_b200_submit_block_device(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                  const void* d_baseband, size_t baseband_bytes); /* input already in HBM */
int srtb_b200_submit_block_ex(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband,
                              size_t baseband_bytes, int on_device, const srtb_b200_block_outputs* outputs /* or NULL */);
int srtb_b200_collect_block(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results);
/* h_series (optional): receives the block's series buffer; d_spectrum (optional): const void*[4], the streams' spectra */
int srtb_b200_collect_block_ex(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results,
                               const float** h_series, const void** d_spectrum);
/* test hook: preset the ring's submission counter (ticket wrap-around test); the ring must be empty */
int srtb_b200_debug_set_submit_count(srtb_b200_ctx* ctx, uint64_t value);
/* device pointer of stream s's dynamic spectrum after process_block (valid until next call) */
const void* srtb_b200_block_spectrum(const srtb_b200_ctx* ctx, int stream);
/* test hook: device pointer of the [C][L] dynamic spectrum of the last trial of the last stream of the most recent
   process_block_dm_sweep (valid until the next call; after a _ex call that re-ran the best trials into ctx memory, the
   last stream's best trial) */
const void* srtb_b200_sweep_spectrum(const srtb_b200_ctx* ctx);

/* ---- semi-coherent DM search on one stream's dynamic spectrum ----------------------------------------------------
 * The block path leaves x[C][L] (complex64, time contiguous), coherently dedispersed at `dm`, SK-flagged channels
 * stored as zeros. Trial DMs near dm are then searched incoherently: each channel's power is shifted by the residual
 * delay between channels and summed over channels.
 * Shifts (host, float64): f_ref = float(freq_low + bandwidth) (the chirp's f_c: the top edge for a positive
 * bandwidth, the bottom one for a negative one), f(c) = freq_low + bandwidth (c + 0.5) / C,
 *   s[d][c] = llround(4.148808e3 (DM_d - dm) (1/f(c)^2 - 1/f_ref^2) sample_rate / (2C)),
 * S+ = max(0, max s), S- = max(0, -min s) over every trial and channel.
 * srtb_b200_incoherent_shifts writes s ([n_dm][C], or shifts == NULL), S+ and S- (either may be NULL). A zero
 * chan_count, a null h_dms or n_dm == 0 returns SRTB_B200_E_INVALID; a shift that is not finite SRTB_B200_E_INVALID. */
int srtb_b200_incoherent_shifts(size_t chan_count, float freq_low, float bandwidth, float sample_rate, float dm,
                                const float* h_dms, size_t n_dm, int64_t* shifts, uint64_t* s_plus, uint64_t* s_minus);
/* The trial groups the search launches with (host only; for tests and tools): the trials stably sorted by DM, then cut
 * greedily into groups of at most 64 trials whose shift spread (max s - min s over the group's trials) is at most 1792
 * on every channel; a trial that would break either limit starts the next group. Writes the group count to *n_groups
 * and, each when not NULL: order [n_dm] (the trial of each sorted slot), groups [n_groups][2] (first sorted slot, trial
 * count), gspan [n_groups][chan_count][2] (min, max of s + S- over the group) and *spread (the largest max - min of any
 * group and channel). groups and gspan need room for n_dm groups. Refusals as srtb_b200_incoherent_shifts, and a NULL
 * n_groups returns SRTB_B200_E_INVALID. */
int srtb_b200_incoherent_groups(size_t chan_count, float freq_low, float bandwidth, float sample_rate, float dm,
                                const float* h_dms, size_t n_dm, int32_t* order, int32_t* groups, int32_t* gspan,
                                uint64_t* n_groups, uint32_t* spread);
/* The search. With ts = time_count - time_reserved_count and T = ts - S+ - S-, trial d's series is
 *   v_d[j] = sum_c |x[c][j + S- + s[d][c]]|^2, j < T (fp32, channels added in index order: two calls agree bit for bit),
 * so every trial has the same length and time origin. Each v_d goes through signal_detect_pipe_2's detector as the block
 * path runs it (zero_count and detect_enabled from the spectrum's first sample per channel, mean removal, boxcars of 1,
 * 2, 4, ... up to max_boxcar_length, each < T, at most 32; time_series_count = T) into h_results[d], and its peaks into
 * h_peaks[d] as srtb_b200_process_block_dm_sweep_ex defines them. The best trial (its rule too) goes to *h_best_trial
 * and its positive boxcar series to h_series ([SRTB_B200_MAX_BOXCARS][T] floats, rows of other boxcars untouched).
 * With a single trial at DM = dm every shift is 0 and v is the block path's column sum.
 * Three kernel launches per call whatever n_dm. Stream-ordered on the ctx's stream; synchronises it once before it
 * returns, and once more when h_series is given and the best trial has a positive boxcar.
 * Before any launch: a null ctx, d_spectrum, h_dms or h_results, n_dm == 0, a zero size or an 8-byte misaligned spectrum
 * returns SRTB_B200_E_INVALID; time_reserved_count >= time_count, T < 2, n_dm > SRTB_B200_INCOHERENT_MAX_DMS or
 * time_count > 2^30 returns SRTB_B200_E_SIZE. Any T up to that limit runs (the dedispersion kernel's CTAs take
 * several time tiles each past 65535 tiles of 256).
 * Scratch the ctx grows on demand and keeps: at most n_dm (12 C + 132 T + 1448) bytes of device memory (shift tables,
 * the series of every boxcar, the scans, headers and peaks), and the shift tables on the host. */
#define SRTB_B200_INCOHERENT_MAX_DMS 4096
int srtb_b200_incoherent_dm_search(srtb_b200_ctx* ctx, const void* d_spectrum, size_t time_count, size_t chan_count,
                                   size_t time_reserved_count, float freq_low, float bandwidth, float sample_rate,
                                   float dm, const float* h_dms, size_t n_dm, float snr, float channel_threshold,
                                   size_t max_boxcar_length, srtb_b200_detect_result* h_results /* [n_dm] */,
                                   srtb_b200_peak* h_peaks /* [n_dm] or NULL */, int32_t* h_best_trial /* or NULL */,
                                   float* h_series /* [SRTB_B200_MAX_BOXCARS][T] or NULL */);

/* ---- single-pulse events and candidates of a DM search ------------------------------------------------------------
 * An event is a maximal run [begin, end) of consecutive indices of one boxcar series v of one trial (and stream) with
 * every v[j] > threshold[b] (count_signal's strict comparison, so the lengths of a row's events add up to its
 * signal_count). peak_index is the smallest index holding the run's largest value, snr that value / sqrt(variance[b])
 * (0 when the variance is 0): srtb_b200_peak's definition, so a row's largest-snr event is its peak record. trial is an
 * index into h_dms as given, boxcar the index b (length 2^b). The rows searched are those the detector headers describe:
 * boxcars b < n_boxcars of every trial with detect_enabled, each series_length[b] long, read on the device.
 * Events are listed in (stream, trial, boxcar, begin) order, the same bytes on every call. When more than max_events
 * exist the first max_events are written and *n_events is the total. Two kernel launches per (trial group, stream): a
 * tile summary with the scan of run counts, then the events (csrc/events.cuh); the list crosses PCIe as it is written,
 * into pinned memory the ctx grows on demand and keeps (max_events per stream), and the ctx's device scratch holds 24
 * bytes per tile of 4096 samples of the rows searched. */
typedef struct {
  uint64_t begin, end;  /* the run [begin, end) in the boxcar series */
  uint64_t peak_index;  /* smallest index of the run's largest value */
  float snr;            /* that value / sqrt(variance), 0 when the variance is 0 */
  uint32_t trial;       /* index into h_dms (srtb_b200_series_events: the record index) */
  uint32_t boxcar;      /* b: boxcar length 2^b */
  uint32_t stream;
} srtb_b200_event;
/* The event pass on caller-owned series: record y's boxcar b is d_series + y trial_stride + b boxcar_stride (floats),
 * described by h_results[y] (detect_enabled, n_boxcars, series_length, threshold, variance; the other fields are not
 * read). Events carry trial = y, stream = 0. Before any launch: a null ctx, d_series, h_results or n_events, a null
 * h_events with max_events > 0, n_trials == 0 or above 65535, n_boxcars above 32, a row longer than boxcar_stride (when
 * n_boxcars > 1) or n_boxcars rows longer than trial_stride (when n_trials > 1) returns SRTB_B200_E_INVALID.
 * Synchronises the ctx's stream. */
int srtb_b200_series_events(srtb_b200_ctx* ctx, const float* d_series, size_t boxcar_stride, size_t trial_stride,
                            const srtb_b200_detect_result* h_results, size_t n_trials, srtb_b200_event* h_events,
                            size_t max_events, uint64_t* n_events);
/* srtb_b200_incoherent_dm_search, which also lists the events of every trial's series (stream 0). Indices are in the
 * searched series: spectrum sample = index + S-. Results, peaks, best trial and series are bit-identical to the plain
 * entry's; two launches more, the same synchronisations. Refusals as the plain entry, and SRTB_B200_E_INVALID for a null
 * n_events or a null h_events with max_events > 0. */
int srtb_b200_incoherent_dm_search_events(srtb_b200_ctx* ctx, const void* d_spectrum, size_t time_count,
                                          size_t chan_count, size_t time_reserved_count, float freq_low,
                                          float bandwidth, float sample_rate, float dm, const float* h_dms, size_t n_dm,
                                          float snr, float channel_threshold, size_t max_boxcar_length,
                                          srtb_b200_detect_result* h_results, srtb_b200_peak* h_peaks,
                                          int32_t* h_best_trial, float* h_series, srtb_b200_event* h_events,
                                          size_t max_events, uint64_t* n_events);
/* srtb_b200_process_block_dm_sweep_ex, which also lists the events of every trial of the loop (never of the best trial's
 * re-run): stream s's events go to h_events + s max_events (up to max_events of them), their total to n_events[s].
 * Results, peaks, best trial, spectra and series are bit-identical to _ex's; two launches more per trial and stream, the
 * same synchronisations (once, and once more when the best trial is re-run). Refusals as _ex, and SRTB_B200_E_INVALID
 * for a null n_events or a null h_events with max_events > 0. */
int srtb_b200_process_block_dm_sweep_events(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg,
                                            const void* baseband, size_t baseband_bytes, int on_device,
                                            const float* h_dms, size_t n_dm, srtb_b200_detect_result* h_results,
                                            const srtb_b200_sweep_outputs* outputs /* or NULL */,
                                            srtb_b200_event* h_events /* [streams][max_events] */, size_t max_events,
                                            uint64_t* n_events /* [streams] */);
/* Candidates: events grouped into astrophysical detections (host only, deterministic; friends of friends, no tunables).
 *   span: the base-series samples an event's boxcar windows add, [begin + o, end - 1 + o + 2^b) with o = 0 for b = 0
 *         and o = 1 otherwise (v_b[j] sums samples j+1 .. j+b of the scan);
 *   rank: a trial's position after a stable sort of h_dms by DM (repeated DMs are adjacent ranks);
 *   friends: the same stream, ranks at most 1 apart, intersecting spans. A candidate is a connected component.
 * Its representative is the member with the largest snr (ties: the smaller trial, boxcar, begin), whose snr, DM, trial,
 * boxcar length and peak_index it carries, with window = peak_index + o (the series index the boxcar's window starts
 * at); members, dm_low / dm_high over the members, and [span_begin, span_end), the union of their spans. Candidates are
 * ordered by (stream, span_begin, representative trial, boxcar, begin); the first max_candidates are written and
 * *n_candidates is the total. A sweep over the spans keeps one active event per rank, O(n log n) in the events. A null
 * n_candidates, a null h_events with n_events > 0, a null h_dms, n_dm == 0, a null h_candidates with
 * max_candidates > 0, an event with trial >= n_dm, boxcar above 31 or end <= begin returns SRTB_B200_E_INVALID. */
typedef struct {
  float snr, dm;              /* the representative's */
  float dm_low, dm_high;      /* over the members */
  uint64_t boxcar_length;     /* the representative's, 2^b */
  uint64_t peak_index;        /* the representative's, in its boxcar series */
  uint64_t window;            /* peak_index + o */
  uint64_t members;
  uint64_t span_begin, span_end;
  uint32_t trial;             /* the representative's */
  uint32_t stream;
} srtb_b200_candidate;
int srtb_b200_cluster_events(const srtb_b200_event* h_events, size_t n_events, const float* h_dms, size_t n_dm,
                             srtb_b200_candidate* h_candidates, size_t max_candidates, uint64_t* n_candidates);
/* ---- candidate cut-outs: the dedispersed frequency-time image and the DM-time plane around each candidate ------------
 * Inputs: S (1..4) spectra x_s [C][L] (complex64, time contiguous, 8-byte aligned), coherently dedispersed at dm; only
 * samples j < ts = L - time_reserved_count are data. Per request: center, DM dm_req, half-width, decimation q. Per call:
 * width W (even), nsub (divides C), n_rows.
 *   power        P(c, j) = sum_s |x_s[c][j]|^2 for 0 <= j < ts when channel c is kept, else 0. |x|^2 = x.x*x.x + x.y*x.y
 *                in fp32 without contraction, the streams added in order. A channel is kept when |x_s[c][0]|^2 != 0 in
 *                every stream (the detector's and the total-intensity sum's masking rule).
 *   k[c]         the incoherent search's shift per unit DM: (1/f(c)^2 - 1/f_ref^2) sample_rate / (2C) 4.148808e3, in
 *                double, f and f_ref as srtb_b200_incoherent_shifts defines them.
 *   shift        s(delta, c) = llround((((double)delta - (double)dm) k[c]) / q) decimated bins, half away from zero
 *                (with q = 1 the incoherent search's s[d][c]).
 *   decimated    t0 = center - (W/2) q, D(c, m) = sum_{u<q} P(c, t0 + m q + u) in fp32, added in u order.
 *   image        ft[k][i] = sum over the C/nsub channels c of subband k, in index order, of D(c, i + s(dm_req, c)), i < W.
 *   row DMs      DM_r = (float)((double)dm_req + (double)halfwidth (double)(r - n_rows/2) / (double)(n_rows/2)), so row
 *                n_rows/2 is dm_req; with n_rows == 1 the one row is dm_req.
 *   plane        dmt[r][i] = sum_{c<C}, in index order, of D(c, i + s(DM_r, c)), fp32.
 * Samples outside [0, ts) add 0: a cut-out near or past a block edge is zero-padded. Raw power sums, no scaling. So with
 * q = 1, one stream and nsub = C, ft[c][i] is |x[c][t0 + i + s]|^2 bit for bit, and with q = 1, one stream and every
 * channel kept, dmt[r] at a row DM equal to trial DM_d of srtb_b200_incoherent_dm_search is v_d[t0 + i - S-] bit for bit
 * wherever that index lies in [0, T).
 * Four kernel launches per call whatever n, S and n_rows (csrc/cutout.cuh): a plan, the decimation (reads each
 * request's span of every channel once, at most min(ts, (W + spread) q) samples), the image and the plane. Stream-ordered
 * on the ctx's stream, synchronised once; two calls write the same bytes.
 * Before any launch: a null ctx, d_spectra, spectrum, h_requests, h_ft or h_dmt, a zero time_count or chan_count,
 * streams outside 1..4, a spectrum not 8-byte aligned, n == 0, an odd W, nsub not dividing C, a decimation of 0, or a
 * non-finite dm, request DM, half-width or shift returns SRTB_B200_E_INVALID; n > 65535, W outside 2..4096, n_rows
 * outside 1..4096, a decimation above 2^20, time_reserved_count >= time_count, a shift above 2^24 bins or |center| >=
 * 2^62 returns SRTB_B200_E_SIZE.
 * Scratch the ctx grows on demand and keeps (each part rounded up to 256 bytes): 8 C + n (24 + 4 n_rows + 8 C + 8 G C +
 * 4 C Wd + 4 nsub W + 4 n_rows W) bytes of device memory, G = ceil(n_rows / 64) or more row groups (fewer rows per
 * group when a group's shifts spread over 1792 bins), Wd = W + the widest shift span of one channel over a request's
 * rows (+ 2). */
typedef struct {
  int64_t center;      /* spectrum sample at the image's bin W/2 (before decimation) */
  float dm;            /* the image's DM and the plane's centre row */
  float dm_halfwidth;  /* the plane's rows span dm +- dm_halfwidth */
  uint32_t decimation; /* q >= 1 samples per bin */
} srtb_b200_cutout_request;
int srtb_b200_candidate_cutouts(srtb_b200_ctx* ctx, const void* const* d_spectra /* [streams] */, int streams,
                                size_t time_count, size_t chan_count, size_t time_reserved_count, float freq_low,
                                float bandwidth, float sample_rate, float dm, const srtb_b200_cutout_request* h_requests,
                                size_t n, size_t width, size_t nsub, size_t n_rows, float* h_ft /* [n][nsub][W] */,
                                float* h_dmt /* [n][n_rows][W] */, float* h_row_dms /* [n][n_rows] or NULL */);
/* Events of the block path: the ring (submit_block_ex / collect_block_ex) that also lists every single pulse of each
 * block at its one DM. Everything submit_block_ex / collect_block_ex hand out is the same, bit for bit. In addition
 * every stream's detector series is searched for events (the definition above) at the end of that stream's chain, on
 * its lane, in stream order: one record of n_boxcars rows under the header the detector just wrote, read on the device.
 * With signal_detect_sum_streams the sum's series is searched on the first lane after the sum's tail; its events carry
 * stream = streams. Events carry trial = 0; indices are in the detector's series (spectrum sample = index, since the
 * detector searches samples 0 .. L' - 1 of the block).
 * Per detector (stream, and sum) two kernel launches and an 8-byte count copy, and a 256-byte memset of the lane's
 * counts where the result headers are zeroed (at the head of a chain, never between two of its kernels); no host
 * synchronisation. Every detector route of the block path feeds the pass (each ends in the detector's
 * tail). The list crosses PCIe as it is written, into pinned memory the ring slot owns: a head of 256 bytes with the
 * counts, then [streams (+1)][max_events] events (40 bytes each), grown by the ctx and kept like the slot's series.
 * Each lane's device scratch holds 24 bytes per tile of 4096 samples of the rows of one detector.
 *   submit: max_events above 2^32 returns SRTB_B200_E_INVALID before any launch; max_events == 0 lists counts only.
 *   collect: n_events[streams (+1)] receives the true totals and *h_events the slot's list, [streams (+1)][max_events]
 *            in (stream, boxcar, begin) order (the first max_events of each detector); valid until the slot is
 *            submitted again. A null n_events, a null h_events when the block was submitted with max_events > 0, or a
 *            ticket submitted through submit_block_ex returns SRTB_B200_E_INVALID and leaves the ticket to collect. */
int srtb_b200_submit_block_events(srtb_b200_ctx* ctx, const srtb_b200_block_config* cfg, const void* baseband,
                                  size_t baseband_bytes, int on_device, const srtb_b200_block_outputs* outputs,
                                  size_t max_events);
int srtb_b200_collect_block_events(srtb_b200_ctx* ctx, int ticket, srtb_b200_detect_result* h_results,
                                   const float** h_series, const void** d_spectrum, const srtb_b200_event** h_events,
                                   uint64_t* n_events /* [streams (+1)] */);

/* ---- folding at a known pulsar period --------------------------------------------------------------------------
 * Time of a spectrum sample. A block whose first baseband sample (per stream) is first_sample holds the spectrum
 * samples j < L at t_j = (first_sample + 2C j) / sample_rate; t = 0 is the first sample after input_file_offset_bytes.
 * Times are topocentric, and an arrival is referred to the chirp's f_c (the band edge coherent dedispersion aligns to).
 * Phase model. Constant period P with derivative Pdot: phi(t) = t/P - 1/2 (Pdot/P^2) t^2. Around a block it is exactly
 *   phi_j = phi0 + a j + b j^2,  phi0 = frac(phi(t_0)),  a = (1/P - Pdot t_0/P^2) D,  b = -1/2 (Pdot/P^2) D^2,
 * with D = 2C / sample_rate. srtb_b200_fold_phase computes them in float64, in exactly this order (q = Pdot / (P P)):
 *   t0 = first_sample / sample_rate; phi = t0 / P - (0.5 q) (t0 t0); phi0 = phi - floor(phi);
 *   a = (1 / P - q t0) (2C / sample_rate); b = (-0.5 q) (D D).
 * A period or sample_rate that is not finite and positive, a non-finite Pdot, a zero 2C or a null output returns
 * SRTB_B200_E_INVALID. */
int srtb_b200_fold_phase(double period, double period_derivative, double sample_rate,
                         uint64_t samples_per_spectrum_sample /* 2C */, uint64_t first_sample, double* phi0, double* a,
                         double* b);
/* Bin of a sample, with every float64 operation rounded on its own (no FMA contraction):
 *   p = (phi0 + a j) + b (j j);  f = p - floor(p);  bin = min(floor(f nbin), nbin - 1).
 * The samples j < fold_count of each stream's d_spectra[s] ([chan_count][time_count] complex64, time contiguous) are
 * folded; with nsub subbands of chan_count / nsub consecutive channels the call returns
 *   h_profile[s][k][bin] = sum over the channels of subband k and the j in bin of |x_s[c][j]|^2   (float64),
 *   h_hits[bin]          = the number of j < fold_count in bin,
 *   h_kept[s][k]         = the channels of subband k with |x_s[c][0]|^2 != 0 (the detector's zero_count rule: a masked
 *                          channel adds zeros to the profile and nothing to kept).
 * The block path folds fold_count = min((N - R) / (2C), valid_samples / (2C)) samples: the first N - R baseband samples,
 * which the overlap-save leaves uncorrupted and consecutive blocks tile without overlap (R = the reader's rewind).
 * |x|^2 is formed in fp32 and summed in float64 in a fixed order: two calls agree bit for bit. The spectra are only read
 * (S C fold_count 8 bytes), in at most three kernel launches whatever streams, nsub and nbin. Stream-ordered on the
 * ctx's stream; synchronises it once before it returns.
 * Before any launch: a null ctx, d_spectra, spectrum or output, a zero time_count or chan_count, streams outside 1..4,
 * a spectrum that is not 8-byte aligned or a non-finite phi0, a or b returns SRTB_B200_E_INVALID; fold_count of 0 or
 * above time_count, nbin outside 1..SRTB_B200_FOLD_MAX_BINS, nsub not dividing chan_count, chan_count above 2^24 or
 * fold_count above 2^40 returns SRTB_B200_E_SIZE.
 * Scratch the ctx grows on demand and keeps, with G = the largest divisor of chan_count / nsub up to 64,
 * K = streams chan_count / G CTAs and R = min(ceil(fold_count / 2048), max(1, floor(4 SMs / K))) tile ranges each:
 * 4 ceil(fold_count / 2048) 2048 + 8 nbin + 8 streams nsub nbin + 4 streams nsub bytes, plus 8 K R nbin + 4 K bytes
 * when (chan_count / nsub / G) R > 1 (each part rounded up to 256 bytes). */
#define SRTB_B200_FOLD_MAX_BINS 4096
int srtb_b200_fold(srtb_b200_ctx* ctx, const void* const* d_spectra /* [streams] */, int streams, size_t time_count,
                   size_t chan_count, size_t fold_count, double phi0, double a, double b, size_t nbin, size_t nsub,
                   double* h_profile /* [streams][nsub][nbin] */, uint64_t* h_hits /* [nbin] */,
                   uint32_t* h_kept /* [streams][nsub] */);
/* The coherence products of a stream pair, folded as srtb_b200_fold folds (the same samples j < fold_count, bins and
 * hits): with X = d_x and Y = d_y ([chan_count][time_count] complex64 each, the two feeds of one receiver) and K(k) the
 * channels c of subband k kept in both, |X[c][0]|^2 != 0 and |Y[c][0]|^2 != 0 (formed in fp32, the detector's rule),
 *   h_coherence[0][k][bin] = AA = sum over c in K(k) and the j in bin of |X[c][j]|^2,
 *   h_coherence[1][k][bin] = BB = ... |Y[c][j]|^2,
 *   h_coherence[2][k][bin] = CR = ... Re(X[c][j] conj(Y[c][j])),
 *   h_coherence[3][k][bin] = CI = ... Im(X[c][j] conj(Y[c][j])),
 *   h_hits[bin]            = the number of j < fold_count in bin (srtb_b200_fold's hits),
 *   h_kept[k]              = |K(k)|.
 * A channel masked in either stream adds nothing to any of the four (PSRCHIVE's Coherence state: AA, BB, CR, CI; no
 * calibration). Each product of two fp32 components is formed exactly in float64 and the sums run in float64 in a fixed
 * order: two calls agree bit for bit. Both spectra are read once (2 chan_count fold_count 8 bytes, less the masked
 * channels), in at most three kernel launches whatever nsub and nbin. Stream-ordered on the ctx's stream; synchronises
 * it once before it returns.
 * Before any launch: a null ctx, spectrum or output, a zero time_count or chan_count, a spectrum that is not 8-byte
 * aligned, d_x == d_y or a non-finite phi0, a or b returns SRTB_B200_E_INVALID; fold_count of 0 or above time_count,
 * nbin outside 1..SRTB_B200_FOLD_MAX_BINS, nsub not dividing chan_count, chan_count above 2^24 or fold_count above 2^40
 * returns SRTB_B200_E_SIZE.
 * Scratch the ctx grows on demand and keeps (shared with srtb_b200_fold), with G = the largest divisor of
 * chan_count / nsub up to 64, K = chan_count / G CTAs and R = min(ceil(fold_count / 2048), max(1, floor(2 SMs / K)))
 * tile ranges each: 4 ceil(fold_count / 2048) 2048 + 8 nbin + 32 nsub nbin + 16 nsub bytes, plus 32 K R nbin + 16 K
 * bytes when (chan_count / nsub / G) R > 1 (each part rounded up to 256 bytes). */
int srtb_b200_fold_coherence(srtb_b200_ctx* ctx, const void* d_x, const void* d_y, size_t time_count,
                             size_t chan_count, size_t fold_count, double phi0, double a, double b, size_t nbin,
                             size_t nsub, double* h_coherence /* [4][nsub][nbin]: AA, BB, CR, CI */,
                             uint64_t* h_hits /* [nbin] */, uint32_t* h_kept /* [nsub]: kept in both */);

/* simplify_spectrum_pipe_2 (pipeline/spectrum_pipe.hpp:82-143): resample_spectrum_3 with norm(),
 * normalize_with_average_value, generate_pixmap. d_spectrum is [in_height][in_width] complex64
 * (time contiguous, as a block leaves it); d_intensity [out_height][out_width] floats receives the
 * normalised intensity, d_pixmap the ARGB32 image; d_average (optional, 1 float) the average before scaling. */
int srtb_b200_simplify_spectrum(srtb_b200_ctx* ctx, const void* d_spectrum, size_t in_width, size_t in_height,
                                size_t out_width, size_t out_height, uint32_t argb_0, uint32_t argb_1,
                                uint32_t argb_overflow, float* d_intensity, uint32_t* d_pixmap, float* d_average);

/* ---- the baseband correlator (the reference's userspace/src/correlator.cpp:53-149) ----------------------------------
 * cross spectrum, its step (1): d_out[i] = (norm * d_a[i]) * conj(d_b[i]) for i < count, complex64, in SyclCPLX's float
 * arithmetic without contraction. d_out may be d_a or d_b (in place); any other overlap with them, a null pointer, a
 * zero count or a pointer that is not 8-byte aligned returns SRTB_B200_E_INVALID before any launch. */
int srtb_b200_cross_spectrum(srtb_b200_ctx* ctx, const void* d_a, const void* d_b, size_t count, float norm,
                             void* d_out);
/* the whole program on device bytes: d_in_1 and d_in_2 hold input_size unsigned 8-bit samples each (the smaller of the
 * two file sizes), of which real_count = 2 (input_size / 2) are read. Each is unpacked and R2C-transformed (the unpack
 * fused into the first sweep where the block path would fuse it), the cross spectrum of the first M = real_count / 2
 * bins is scaled by norm = float(pow(double(input_size), -1.5)), transformed by an unnormalised backward C2C of M
 * points, and d_out (4-byte aligned) receives its M magnitudes |y[i]| as floats.
 * Before any launch: input_size < 2, a null pointer or a misaligned d_out returns SRTB_B200_E_INVALID; real_count not
 * a power of two ("[fft] n must be a power of 2", fft/naive_fft_wrapper.hpp:52-56) or above 2^31 returns
 * SRTB_B200_E_SIZE. Working buffers (2 x (real_count + 2) floats) live in the ctx and grow on demand. Stream-ordered. */
int srtb_b200_correlate(srtb_b200_ctx* ctx, const void* d_in_1, const void* d_in_2, size_t input_size, float* d_out);

/* ---- the integrating, segment-averaged correlator (an FX correlator: the noise falls as 1/sqrt(K)) -----------------
 * Inputs: samples of width bits = 1, 2, 4, 8 (unsigned) or -8 (int8), in srtb_b200_unpack's SIMPLE order (sub-byte
 * samples MSB first within a byte). Segment size Ls: a power of two from 16 to 2^30 real samples; Ms = Ls / 2.
 * Segment s of each input is its samples [s Ls, (s + 1) Ls), with no overlap and no window; A_s and B_s are the first Ms
 * bins of each segment's real FFT (the Nyquist bin is dropped). Over K segments in all,
 *   out[j] = | sum_k ((norm / K) sum_s A_s[k] conj(B_s[k])) e^{+2 pi i j k / Ms} |, j < Ms, float32,
 *   norm = float(pow(double(Ls), -1.5)).
 * With K = 1 and Ls = input_size this is what srtb_b200_correlate computes. Lags: if input 2 is input 1 delayed by d
 * samples (|d| << Ls), the peak is at (-d / 2) mod Ms.
 *
 * accumulate: reads n_segments Ls |bits| / 8 bytes of each input (any byte address) and adds sum_s A_s conj(B_s) into
 * d_acc, Ms complex float64 values (16-byte aligned, owned by the caller); reset != 0 overwrites d_acc instead. The sum
 * within a call has a fixed grouping, so the result is deterministic. Kernels: a pack of two segments of one input per
 * complex row, one batched forward C2C of Ls points over the rows of both inputs, a split / cross-multiply /
 * accumulate; their number does not depend on n_segments. Working buffers (2 ceil(n_segments / 2) Ls complex64, plus
 * the C2C's scratch above 2^14 points) live in the ctx and grow on demand.
 * finish: scales d_acc by norm / total_segments, rounds it to complex64, runs an unnormalised backward C2C of Ms points
 * on a ctx buffer and writes the Ms magnitudes (hypotf) into d_out (4-byte aligned).
 * Both are stream-ordered and do not synchronise. Before any launch they return SRTB_B200_E_INVALID for a null
 * pointer, n_segments == 0, total_segments == 0, a d_acc not 16-byte aligned, a d_out not 4-byte aligned or bits
 * outside the set, and SRTB_B200_E_SIZE for an Ls that is not a power of two in [16, 2^30] or n_segments Ls > 2^34. */
int srtb_b200_correlate_accumulate(srtb_b200_ctx* ctx, const void* d_in_1, const void* d_in_2, int bits,
                                   size_t segment_size, size_t n_segments, void* d_acc, int reset);
int srtb_b200_correlate_finish(srtb_b200_ctx* ctx, const void* d_acc, size_t segment_size, uint64_t total_segments,
                               float* d_out);

#ifdef __cplusplus
}
#endif
#endif /* SRTB_B200_H */
