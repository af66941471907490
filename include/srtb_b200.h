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
 * streams written: 1 (SIMPLE), 2 (INTERLEAVED_2, SNAP1, GZNUPSR_A1_2), 4 (GZNUPSR_A1_4). */
int srtb_b200_unpack(srtb_b200_ctx* ctx, const void* d_in, size_t in_bytes, int bits, int format,
                     int window, float* const d_out[4], size_t out_count);

/* ---- fft_1d_dispatcher<R2C_1D>::process (fft/fft.hpp:146-149; naive_fft.hpp:221-261) ----
 * in place on n_real + 2 floats: X[k], k = 0..n_real/2, unnormalised, forward sign. */
int srtb_b200_fft_r2c_inplace(srtb_b200_ctx* ctx, float* d_inout, size_t n_real);

/* ---- batched C2C, unnormalised, in place (fft_1d_dispatcher<C2C_1D_*>; naive_fft.hpp:155-176) ----
 * direction +1 forward (e^-i), -1 backward (e^+i). d_x is [batch][length] complex64. */
int srtb_b200_fft_c2c(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch, int direction);

/* watfft_1d_c2c_pipe (pipeline/fft_pipe.hpp:313-371): batch backward C2C of `length` */
int srtb_b200_watfft_c2c_backward(srtb_b200_ctx* ctx, void* d_x, size_t length, size_t batch);

/* ---- rfi_mitigation_s1_pipe (pipeline/rfi_mitigation_pipe.hpp:43-101) ---------------
 * mean m of |X|^2; X = (|X|^2 > avg_threshold*m) ? 0 : X*norm_coef; then zero the
 * inclusive bin ranges h_bin_ranges[n_ranges][2] (spectrum/rfi_mitigation.hpp:137-143).
 * d_mean_out (optional device float) receives m. */
int srtb_b200_rfi_s1(srtb_b200_ctx* ctx, void* d_x, size_t count, float avg_threshold,
                     float norm_coef, const size_t* h_bin_ranges, size_t n_ranges,
                     float* d_mean_out);

/* host helpers mirroring the reference's host-side arithmetic for this stage */
float srtb_b200_norm_coefficient(size_t in_count, size_t spectrum_channel_count); /* rfi_mitigation_pipe.hpp:61-65 */
size_t srtb_b200_eval_rfi_ranges(const char* freq_list, float* pairs, size_t max_pairs); /* rfi_mitigation.hpp:64-88 */
int srtb_b200_rfi_range_to_bins(float f1, float f2, float freq_low, float bandwidth, size_t in_count,
                                size_t* lo, size_t* hi); /* rfi_mitigation.hpp:102-143; 1 = applied */

/* ---- coherent_dedispertion (coherent_dedispersion.hpp:133-150,223-237) --------------- */
int srtb_b200_dedisperse(srtb_b200_ctx* ctx, void* d_x, size_t count, float f_min, float f_c,
                         float df, float dm);
/* nsamps_reserved (coherent_dedispersion.hpp:76-128) */
size_t srtb_b200_nsamps_reserved(size_t baseband_input_count, size_t spectrum_channel_count,
                                 float freq_low, float bandwidth, float sample_rate, float dm,
                                 int reserve_sample);

/* ---- mitigate_rfi_spectral_kurtosis_method_2 (spectrum/rfi_mitigation.hpp:292-341) ----
 * d_x is [chan_count][time_count]. d_sk_out (optional, chan_count floats) receives sk. */
int srtb_b200_rfi_s2_sk(srtb_b200_ctx* ctx, void* d_x, size_t time_count, size_t chan_count,
                        float sk_threshold, float* d_sk_out);

/* ---- signal_detect_pipe_2 (pipeline/signal_detect_pipe.hpp:252-442) -------------------
 * h_series: NULL, or host buffer of SRTB_B200_MAX_BOXCARS * time_count floats; row i receives
 * the series of entry i when signal_count[i] > 0 (all entries if copy_all != 0).
 * Synchronises the stream. */
int srtb_b200_signal_detect(srtb_b200_ctx* ctx, const void* d_x, size_t time_count,
                            size_t chan_count, size_t time_reserved_count, float snr_threshold,
                            float channel_threshold, size_t max_boxcar_length,
                            srtb_b200_detect_result* h_result, float* h_series, int copy_all);

/* ---- alternates of the refft path (defined by the reference, not wired in its main.cpp): spectra laid out
 * [time][frequency], as refft_1d_c2c_pipe leaves them (pipeline/fft_pipe.hpp:197-278) ------------------------------
 * mitigate_rfi_spectral_kurtosis_method (v1, spectrum/rfi_mitigation.hpp:181-275, normalization = false):
 * d_x is [time_counts][fft_bins]; every frequency column whose sk = M s4 / s2^2 over the time_counts spectra leaves
 * the thresholds is zeroed. d_sk_out (optional, fft_bins floats) receives sk. */
int srtb_b200_rfi_sk_v1(srtb_b200_ctx* ctx, void* d_x, size_t fft_bins, size_t time_counts, float sk_threshold,
                        float* d_sk_out);
/* signal_detect_pipe (v1, pipeline/signal_detect_pipe.hpp:51-230): SK v1 in place, masked channels counted over the
 * first spectrum, one time-series value per spectrum (sum over its count_per_batch bins of |x|^2), mean removal,
 * count_signal, boxcars 2..max (series lengths batch_size - boxcar; nothing is trimmed). h_series rows are
 * batch_size floats apart. Synchronises the stream. */
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
} srtb_b200_block_config;

/* h_baseband: host (ideally pinned) bytes of one block, all streams interleaved as the
 * format says; the call copies them to the device, runs every stage for every stream and
 * fills h_results[stream]. d_spectrum_out (optional): per-stream device pointers that
 * receive the dynamic spectrum [C][L] (else it stays in ctx scratch).
 * Returns the number of streams processed (>0) or a negative status. */
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
  float* d_spectrum[4]; /* per stream: device buffer of baseband_input_count + 2 floats, 16-byte aligned        */
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
   process_block_dm_sweep (valid until the next call) */
const void* srtb_b200_sweep_spectrum(const srtb_b200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* SRTB_B200_H */
