/* b200dd.h -- C ABI of the H100-native delay-Doppler processor (libb200dd.so).
 *
 * This is the drop-in boundary for blah2's hot path: every entry point replaces the
 * arithmetic behind one public method of the reference's process classes, takes only
 * plain C types (pointers + sizes, no CUDA / torch types in signatures; a stream is an
 * opaque void* that may be NULL) and returns an integer status.  The C++ classes in
 * blah2_b200/dropin/ (same names, constructors and method signatures as the reference)
 * and the Python binding blah2_b200/capi.py are thin callers of this ABI.
 *
 * Reference interface each group replaces (paths relative to the blah2 repository):
 *   b200dd_caf_*     Ambiguity::Ambiguity / Ambiguity::process / getters
 *                    src/process/ambiguity/Ambiguity.h:34-58, Ambiguity.cpp:11-200
 *   b200dd_wh_*      WienerHopf::WienerHopf / WienerHopf::process
 *                    src/process/clutter/WienerHopf.h:68-78, WienerHopf.cpp:7-163
 *   b200dd_det_*     CfarDetector1D::process, Centroid::process, Interpolate::process,
 *                    Map::set_metrics
 *                    src/process/detection/CfarDetector1D.h:46-55, Centroid.h:35-44,
 *                    Interpolate.h:36-45, src/data/Map.cpp:188-206
 *   b200dd_spectrum_*   SpectrumAnalyser::SpectrumAnalyser / SpectrumAnalyser::process
 *                    src/process/spectrum/SpectrumAnalyser.h:48-57, SpectrumAnalyser.cpp:9-74
 *   b200dd_next_hamming   next_hamming, src/process/meta/HammingNumber.h:36
 *   b200dd_mapjson_*    Map::to_json + Map::delay_bin_to_km, src/data/Map.cpp:116-185 (blah2.cpp:303-304)
 *   b200dd_maxhold_*    the API's max-hold stash, api/stash/maxhold.js (served at /stash/map, api/server.js:96-97)
 *   b200dd_detjson_*    Detection::to_json + Detection::delay_bin_to_km, src/data/Detection.cpp:47-106
 *                       (blah2.cpp:312-317), and the API's detection stash, api/stash/detection.js (served at
 *                       /stash/detection, api/server.js:99-100)
 *   b200dd_tracker_*    Tracker::process + Track::to_json, src/process/tracker/Tracker.cpp, src/data/Track.cpp
 *                       (blah2.cpp:291-296, :324-328)
 *   b200dd_iqjson_*     IqData::to_json, src/data/IqData.cpp:93-125 (blah2.cpp:299-300), and the API's IQ-data
 *                       stash, api/stash/iqdata.js (served at /stash/iqdata, api/server.js:102-103)
 *
 * Data conventions
 *   host IQ      interleaved complex128 (re, im doubles) -- what IqData holds
 *                (src/data/IqData.h:26).
 *   device IQ    interleaved complex64 (float2).  Every capture format of the reference
 *                (int16 RSPduo, fc32 USRP, int8 HackRF / Kraken) is exactly representable.
 *   map          row-major [nDopplerBins][nDelayBins] complex, row k <-> doppler[k],
 *                column j <-> delay[j]: the layout of Map<complex<double>>::data
 *                (src/data/Map.h:30); complex128 on the host, complex64 on the device.
 *   detections   three parallel double arrays delay (bins) / doppler (Hz) / snr (dB)
 *                (src/data/Detection.h:17-24), in the reference's emission order.
 *
 * Threading: a handle owns one CUDA stream and scratch buffers and is NOT re-entrant
 * (the reference's objects are not either; they are called from one thread,
 * src/blah2.cpp:245).  Different handles may be used from different threads.
 *
 * There is no CPU fallback: every *_process* entry point runs CUDA kernels for sm_90a
 * and fails with B200DD_ERR_CUDA when no usable device is present.
 *
 * Environment (all optional; default plans use the device's SM count, other heuristics not re-tuned on H100):
 *   B200DD_CAF_LOG2M / B200DD_CAF_PARTS      range-correlation FFT length (2^k) / CTAs per batch
 *   B200DD_WH_LOG2M, B200DD_WH_CORR_LOG2M, B200DD_WH_APPLY_LOG2M   WienerHopf FFT plans
 * They are read when a handle is created; the plan made then alone picks every kernel the handle launches.
 * None of them changes results beyond the rounding of a different FFT factorisation.
 */
#ifndef B200DD_H
#define B200DD_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200DD_API __attribute__((visibility("default")))
#else
#define B200DD_API
#endif

#define B200DD_OK 0
#define B200DD_ERR_ARG 1         /* null pointer / size mismatch */
#define B200DD_ERR_GEOMETRY 2    /* geometry outside the supported range (see DESIGN.md "limits") */
#define B200DD_ERR_CUDA 3        /* CUDA runtime error; b200dd_last_error() has the text */
#define B200DD_ERR_CAPACITY 4    /* output capacity too small (detections, map JSON) */
#define B200DD_ERR_NONFINITE 5   /* map / detection / IQ-data JSON: a value rapidjson cannot write (a map cell or
                                    spectrum bin with |z| = 0, inf or NaN; a detection that is not finite) */
#define B200DD_FILTER_FAILED 10  /* WienerHopf: matrix not positive definite -> y left untouched
                                    (reference returns false, WienerHopf.cpp:111-122) */

/* Text of the last error raised on the calling thread ("" if none). */
B200DD_API const char *b200dd_last_error(void);

/* Library / device probe: returns number of CUDA devices (0 when none), fills optional name. */
B200DD_API int b200dd_device_count(void);
B200DD_API int b200dd_device_name(int device, char *buf, int buflen);

/* next_hamming(value): first 5-smooth number strictly greater than value
 * (src/process/meta/HammingNumber.cpp:38-48). Host arithmetic. */
B200DD_API uint32_t b200dd_next_hamming(uint32_t value);

/* ------------------------------------------------------------------ CAF / Ambiguity */

typedef struct b200dd_caf b200dd_caf;

typedef struct {
  int32_t delay_min;     /* bins  (Ambiguity.h:34 delayMin) */
  int32_t delay_max;     /* bins */
  int32_t doppler_min;   /* Hz */
  int32_t doppler_max;   /* Hz */
  uint32_t fs;           /* Hz */
  uint32_t n_samples;    /* samples per CPI per channel */
  int32_t round_hamming; /* only affects get_nfft(); the GPU FFT length is independent */
  int32_t device;        /* CUDA device ordinal, -1 = current device */
} b200dd_caf_params;

typedef struct {
  uint32_t n_delay_bins;   /* Ambiguity::get_n_delay_bins   */
  uint32_t n_doppler_bins; /* Ambiguity::get_n_doppler_bins */
  uint32_t n_corr;         /* Ambiguity::get_n_corr         */
  uint32_t nfft;           /* Ambiguity::get_nfft           */
  uint32_t n_used;         /* nDopplerBins * nCorr: samples consumed per channel (Ambiguity.cpp:105) */
  double cpi;              /* Ambiguity::get_cpi            */
  double doppler_middle;   /* Ambiguity::get_doppler_middle */
  /* implementation facts (for DESIGN / bench reporting) */
  uint32_t range_fft_len;   /* M of the segmented range FFT */
  uint32_t range_segments;  /* segments per batch */
  uint32_t range_hop;       /* new samples per segment */
  uint32_t doppler_fft_len; /* Bluestein length M2 */
  uint32_t range_parts;     /* CTAs per batch (partial range matrices summed by the Doppler kernel) */
  uint32_t range_groups;    /* always 1 (one warp group per range CTA); kept so that the layout and the readers
                               of this struct (bench.py) stay unchanged */
} b200dd_caf_geometry;

B200DD_API int b200dd_caf_create(const b200dd_caf_params *params, b200dd_caf **out);
/* The host half of b200dd_caf_create on its own -- the Ambiguity constructor's arithmetic (Ambiguity.cpp:11-66: bin
 * counts, nCorr, cpi, nfft, both axes) and the kernel plan -- without touching a device (params->device is only used
 * to look up the SM count; 132, an H100 SXM, is assumed when there is none).  delay / doppler are nullable; capacities in elements.
 * This is what lets the CPU test-suite check the PRODUCT's geometry code against the reference's golden values. */
B200DD_API int b200dd_caf_plan(const b200dd_caf_params *params, b200dd_caf_geometry *out, int32_t *delay,
                               uint32_t cap_delay, double *doppler, uint32_t cap_doppler);
B200DD_API void b200dd_caf_destroy(b200dd_caf *h);
B200DD_API int b200dd_caf_get_geometry(const b200dd_caf *h, b200dd_caf_geometry *out);
/* Map axes as the Ambiguity constructor builds them (Ambiguity.cpp:46-59):
 * delay[n_delay_bins] (bins), doppler[n_doppler_bins] (Hz). */
B200DD_API int b200dd_caf_get_axes(const b200dd_caf *h, int32_t *delay, double *doppler);

/* Ambiguity::process on HOST buffers: x, y = n interleaved complex128 samples each
 * (n >= n_used; only the first n_used are consumed, like the FIFO pops at
 * Ambiguity.cpp:108-112).  map_out = [n_doppler_bins][n_delay_bins] complex128.
 * H2D, conversion to float2, kernels and D2H all run on the handle's stream; the call
 * returns after the map is in map_out. */
B200DD_API int b200dd_caf_process_host(b200dd_caf *h, const double *x, const double *y, uint32_t n, double *map_out);

/* Device-resident variant: d_x, d_y = n float2 samples in device memory, d_map =
 * [n_doppler_bins][n_delay_bins] float2 in device memory.  Asynchronous on `stream`
 * (NULL = the handle's stream); no host synchronisation. */
B200DD_API int b200dd_caf_process_device(b200dd_caf *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                              void *stream);

/* The two stages separately, for ONE large CPI sharded over several GPUs (BASELINE config 5):
 * range stage on a contiguous block of batches (the rank's 1/world slice of the IQ), then -- after the
 * caller has all-gathered the range matrix -- the Doppler stage on a tile of delay columns.
 *   d_x, d_y : float2 samples of batches [batch0, batch0 + n_batches), i.e. n_batches * n_corr samples
 *   d_R      : out, float2 [n_batches][n_delay_bins]  (rows batch0.. of the range matrix)
 *   d_R (doppler) : in, the COMPLETE range matrix float2 [n_doppler_bins][n_delay_bins]
 *   d_map_tile    : out, float2 [n_doppler_bins][n_cols] = map[:, col0 : col0 + n_cols]
 * Symmetric Doppler windows only (the pre-rotation phase would need the global sample index). */
B200DD_API int b200dd_caf_range_device(b200dd_caf *h, const void *d_x, const void *d_y, uint32_t batch0,
                                       uint32_t n_batches, void *d_R, void *stream);
B200DD_API int b200dd_caf_doppler_device(b200dd_caf *h, const void *d_R, uint32_t col0, uint32_t n_cols,
                                         void *d_map_tile, void *stream);
/* A tile [nDop][n_cols] (as b200dd_caf_doppler_device writes it, possibly gathered from another GPU) into the delay
 * columns [col0, col0 + n_cols) of a row-major [nDop][nDel] map: one strided device copy. */
B200DD_API int b200dd_caf_place_tile_device(b200dd_caf *h, const void *d_tile, uint32_t col0, uint32_t n_cols, void *d_map,
                                            void *stream);
/* All tiles of an EQUAL split of the delay columns over n_tiles ranks (tile t = columns [t b + min(t, r), ...) with
 * b = nDel / n_tiles, r = nDel % n_tiles: the first r tiles one column wider), stored back to back in d_tiles as the
 * gather delivers them, into the row-major map: one kernel. */
B200DD_API int b200dd_caf_place_tiles_device(b200dd_caf *h, const void *d_tiles, uint32_t n_tiles, void *d_map, void *stream);

/* Profiling aid: same as b200dd_caf_process_device but brackets the range-correlation kernel and the
 * Doppler kernel with CUDA events on the launching stream and returns their durations (ms).
 * Synchronises the stream.  Used by bench.py for the roofline figures. */
B200DD_API int b200dd_caf_profile_device(b200dd_caf *h, const void *d_x, const void *d_y, uint32_t n, void *d_map,
                                         void *stream, float *ms_range, float *ms_doppler);

/* Intermediate range matrix of the last process call (row i = batch i, nDelayBins lags;
 * Ambiguity.cpp:106-149) copied to host as complex64 -- parity tests only. */
B200DD_API int b200dd_caf_debug_range_matrix(b200dd_caf *h, float *out);

/* Device pointer to the handle's last map (float2 [nDop][nDel]) for chaining detection
 * without a host round trip; valid until the next process call on this handle. */
B200DD_API void *b200dd_caf_device_map(b200dd_caf *h);
/* Handle's stream (cudaStream_t as void*). */
B200DD_API void *b200dd_caf_stream(b200dd_caf *h);

/* ------------------------------------------------------------------ WienerHopf */

typedef struct b200dd_wh b200dd_wh;

/* WienerHopf(delayMin, delayMax, nSamples): nBins = delayMax - delayMin (no +1,
 * WienerHopf.cpp:12). device = -1 -> current device. */
B200DD_API int b200dd_wh_create(int32_t delay_min, int32_t delay_max, uint32_t n_samples, int32_t device, b200dd_wh **out);
B200DD_API void b200dd_wh_destroy(b200dd_wh *h);

/* WienerHopf::process on HOST buffers.  x: n_samples complex128 (read only);
 * y: n_samples complex128, overwritten with the filtered surveillance channel.
 * Returns B200DD_OK, or B200DD_FILTER_FAILED with y untouched. */
B200DD_API int b200dd_wh_process_host(b200dd_wh *h, const double *x, double *y);

/* Device-resident variant: d_x, d_y float2[n_samples]; d_y_out float2[n_samples] (may
 * alias d_y).  Asynchronous; the success flag is written to the handle's device status
 * word and, when the solve fails, d_y_out receives d_y unchanged.  Use
 * b200dd_wh_last_status() (synchronises the stream) to read it. */
B200DD_API int b200dd_wh_process_device(b200dd_wh *h, const void *d_x, const void *d_y, void *d_y_out, void *stream);
B200DD_API int b200dd_wh_last_status(b200dd_wh *h);
/* Same with complex128 device buffers (double2) in and out -- what the host path and the
 * pipeline's host entry use so that the filter sees the caller's doubles unrounded. */
B200DD_API int b200dd_wh_process_device_f64(b200dd_wh *h, const void *d_x, const void *d_y, void *d_y_out, void *stream);
/* Profiling aid: per-stage CUDA-event durations (ms) of correlation, solve, and weight-spectrum+filter. */
B200DD_API int b200dd_wh_profile_device(b200dd_wh *h, const void *d_x, const void *d_y, void *d_y_out, void *stream,
                                        float *ms_corr, float *ms_solve, float *ms_apply);
/* Device address of the status word (0 ok, 1 failed) for kernels chained after the filter. */
B200DD_API const int *b200dd_wh_device_status(b200dd_wh *h);
/* Filter weights w[nBins] / correlations a, b of the last call as complex128 -- parity tests. */
B200DD_API int b200dd_wh_debug_weights(b200dd_wh *h, double *w, double *a, double *b);
B200DD_API uint32_t b200dd_wh_n_bins(const b200dd_wh *h);

/* ---- one CPI split over several GPUs (SURVEY.md s8e row 3): this handle filters the samples
 * [chunk_begin, chunk_begin + chunk_len) of an n_samples-sample signal (delayMin <= 0, chunk longer than the
 * filter).  The caller holds LOCAL float2 buffers with halos (b200dd_wh_chunk_halos):
 *   x_loc: x[chunk_begin - x_left .. chunk_begin + chunk_len + x_right)   (indices taken modulo n_samples on the right:
 *          the correlations are circular; the left halo of the first chunk is never read: zero filter history)
 *   y_loc: y[chunk_begin .. chunk_begin + chunk_len + y_right)            (modulo n_samples as well)
 * 1. b200dd_wh_chunk_corr_device -> d_ab = this chunk's share of (a[0..nBins), b[0..nBins)) (2 nBins complex128);
 * 2. the caller sums d_ab over the GPUs (b200dd_comm_allreduce_f64_async, 4 nBins doubles);
 * 3. b200dd_wh_chunk_filter_device solves the SAME system on every GPU and writes the chunk's chunk_len filtered
 *    samples (float2) to d_y_out.  b200dd_wh_last_status reports a failed solve as for a whole signal. */
B200DD_API int b200dd_wh_create_chunk(int32_t delay_min, int32_t delay_max, uint32_t n_samples, uint32_t chunk_begin,
                                      uint32_t chunk_len, int32_t device, b200dd_wh **out);
B200DD_API int b200dd_wh_chunk_halos(const b200dd_wh *h, uint32_t *x_left, uint32_t *x_right, uint32_t *y_right);
B200DD_API int b200dd_wh_chunk_corr_device(b200dd_wh *h, const void *d_x_loc, const void *d_y_loc, void *d_ab, void *stream);
B200DD_API int b200dd_wh_chunk_filter_device(b200dd_wh *h, const void *d_ab, const void *d_x_loc, const void *d_y_loc,
                                             void *d_y_out, void *stream);

/* The FFT plan of the two FFT stages (for measurement: transforms per CPI = corr_lag_blocks (3 corr_segments +
 * 2 corr_ctas) in the correlation kernel, (filter_partitions + 1) filter_blocks + filter_partitions in the filter
 * stage) and the solve kernel's shape.  Above 3585 taps the correlations split the lags into corr_lag_blocks blocks
 * and the filter splits the weights into filter_partitions partitions of filter_partition_taps taps (both 1 / nBins
 * below); the solve runs solve_threads threads of one CTA, solve_rows_per_thread matrix rows each (4 above 2048
 * taps: the register-resident generator kernel). */
typedef struct {
  uint32_t corr_fft_len, corr_hop, corr_segments, corr_ctas;
  uint32_t filter_fft_len, filter_hop, filter_blocks;
  uint32_t corr_lag_blocks, filter_partitions, filter_partition_taps;
  uint32_t solve_threads, solve_rows_per_thread;
} b200dd_wh_plan;
B200DD_API int b200dd_wh_get_plan(const b200dd_wh *h, b200dd_wh_plan *out);
B200DD_API void *b200dd_wh_stream(b200dd_wh *h);

/* ------------------------------------------------------------------ detection tail */

typedef struct b200dd_det b200dd_det;

typedef struct {
  double pfa;           /* CfarDetector1D(pfa, ...)          CfarDetector1D.h:46 */
  int32_t n_guard;      /* int8_t in the reference */
  int32_t n_train;      /* int8_t */
  int32_t min_delay;    /* int8_t */
  double min_doppler;
  uint32_t n_centroid_delay;   /* Centroid(nDelay, nDoppler, resolutionDoppler)  Centroid.h:35 */
  uint32_t n_centroid_doppler;
  double resolution_doppler;
  int32_t interp_delay;   /* Interpolate(doDelay, doDoppler)  Interpolate.h:36 */
  int32_t interp_doppler;
  int32_t device;
} b200dd_det_params;

B200DD_API int b200dd_det_create(const b200dd_det_params *params, uint32_t max_doppler_bins, uint32_t max_delay_bins,
                      b200dd_det **out);
B200DD_API void b200dd_det_destroy(b200dd_det *h);

/* Map::set_metrics on a device map (float2 [n_dop][n_del]): metrics[0] = noisePower,
 * metrics[1] = maxPower (Map.cpp:188-206).  Synchronises the stream. */
B200DD_API int b200dd_det_set_metrics_device(b200dd_det *h, const void *d_map, uint32_t n_dop, uint32_t n_del, double *metrics,
                                  void *stream);

/* Stage selectors for b200dd_det_process_*: run CFAR only, CFAR+Centroid, or all three. */
#define B200DD_DET_CFAR 1
#define B200DD_DET_CENTROID 2
#define B200DD_DET_INTERPOLATE 3

/* CfarDetector1D -> Centroid -> Interpolate on a device map (blah2.cpp:285-287).
 * delay[n_del] / doppler[n_dop] are the map axes (host), noise_power = Map::noisePower.
 * Outputs (host): up to `cap` detections; *n_out = number found (may exceed cap ->
 * B200DD_ERR_CAPACITY with the first cap filled). */
B200DD_API int b200dd_det_process_device(b200dd_det *h, int last_stage, const void *d_map, uint32_t n_dop, uint32_t n_del,
                              const int32_t *delay, const double *doppler, double noise_power, double *o_delay,
                              double *o_doppler, double *o_snr, uint32_t cap, uint32_t *n_out, void *stream);

/* Fully asynchronous variant for device-resident streams of CPIs: Map::set_metrics is evaluated
 * on the device first (blah2.cpp:279) and its noisePower feeds the detector without a host round
 * trip; nothing is copied back until b200dd_det_chain_fetch (which synchronises the stream).
 * last_stage = 0 runs Map::set_metrics only (detection disabled: the fetch then reports 0 detections).
 * A CFAR stage that finds more detections than the handle's list capacity (min(cells, 2^18)) makes the
 * fetch return B200DD_ERR_CAPACITY: the later stages saw a truncated list. */
B200DD_API int b200dd_det_chain_device_async(b200dd_det *h, int last_stage, const void *d_map, uint32_t n_dop,
                                             uint32_t n_del, const int32_t *delay, const double *doppler,
                                             void *stream);
B200DD_API int b200dd_det_chain_fetch(b200dd_det *h, double *metrics, double *o_delay, double *o_doppler,
                                      double *o_snr, uint32_t cap, uint32_t *n_out, void *stream);

/* Same on a HOST complex128 map (what the drop-in classes hold in Map::data). */
B200DD_API int b200dd_det_process_host(b200dd_det *h, int last_stage, const double *map, uint32_t n_dop, uint32_t n_del,
                            const int32_t *delay, const double *doppler, double noise_power, double *o_delay,
                            double *o_doppler, double *o_snr, uint32_t cap, uint32_t *n_out);

/* Centroid / Interpolate alone on a host detection list (class-level drop-ins). */
B200DD_API int b200dd_det_centroid_host(b200dd_det *h, const double *delay, const double *doppler, const double *snr,
                             uint32_t n, double *o_delay, double *o_doppler, double *o_snr, uint32_t cap,
                             uint32_t *n_out);
B200DD_API int b200dd_det_interpolate_host(b200dd_det *h, const double *delay, const double *doppler, const double *snr,
                                uint32_t n, const double *map, uint32_t n_dop, uint32_t n_del, const int32_t *mdelay,
                                const double *mdoppler, double noise_power, double *o_delay, double *o_doppler,
                                double *o_snr, uint32_t cap, uint32_t *n_out);

/* ------------------------------------------------------------------ SpectrumAnalyser
 *
 * SpectrumAnalyser(n, bandwidth) / SpectrumAnalyser::process(IqData *x)
 * (src/process/spectrum/SpectrumAnalyser.h:48-57, SpectrumAnalyser.cpp:9-74): the stage of the reference's
 * process thread that runs on the reference channel right before the clutter filter (src/blah2.cpp:263-265).
 * decimation = n / bandwidth, nSpectrum = n / decimation, nfft = nSpectrum * decimation (:16-18); the result is
 * every decimation-th bin of the fft-shifted nfft-point spectrum of the first nfft samples (:36-54), which the
 * reference stores with IqData::update_spectrum (:55).  The device kernels never form the nfft-point transform:
 * one HBM-bound folding pass over x and an nSpectrum-point DFT (blah2_b200/csrc/spectrum.cu). */
typedef struct b200dd_spectrum b200dd_spectrum;

typedef struct {
  uint32_t decimation;   /* SpectrumAnalyser.cpp:16 */
  uint32_t n_spectrum;   /* :17, number of complex bins process() produces */
  uint32_t nfft;         /* :18, samples of x consumed (read, not popped) */
  uint32_t n_frequency;  /* entries of the frequency vector the reference's loop (:57-67) produces: its uint32_t
                            counter starts at (2^32 - nSpectrum) / 2, so this is 0 for every realistic size */
  /* implementation facts */
  uint32_t fold_chunks;          /* row chunks of the folding pass (partial sums reduced in a fixed order) */
  uint32_t fold_rows_per_chunk;
} b200dd_spectrum_geometry;

/* Returns B200DD_ERR_GEOMETRY where the reference is undefined (bandwidth <= 0, NaN, or bandwidth > n, which
 * divides by zero at :17) or for more than 65536 spectrum bins. */
B200DD_API int b200dd_spectrum_create(uint32_t n, double bandwidth, int32_t device, b200dd_spectrum **out);
/* The host half of b200dd_spectrum_create on its own (no device needed): geometry and, when `frequency` is not NULL,
 * the n_frequency values of the frequency vector. */
B200DD_API int b200dd_spectrum_plan(uint32_t n, double bandwidth, b200dd_spectrum_geometry *out, double *frequency,
                                    uint32_t cap);
B200DD_API void b200dd_spectrum_destroy(b200dd_spectrum *h);
B200DD_API int b200dd_spectrum_get_geometry(const b200dd_spectrum *h, b200dd_spectrum_geometry *out);
/* The vector SpectrumAnalyser::process hands to IqData::update_frequency (n_frequency doubles, kHz). */
B200DD_API int b200dd_spectrum_get_frequency(const b200dd_spectrum *h, double *frequency, uint32_t cap);

/* SpectrumAnalyser::process on a HOST buffer: x = n >= nfft interleaved complex128 samples (only the first nfft
 * are read); spectrum_out = n_spectrum complex128.  Synchronous. */
B200DD_API int b200dd_spectrum_process_host(b200dd_spectrum *h, const double *x, uint32_t n, double *spectrum_out);
/* Device-resident variants: d_x = float2[n] (or double2[n] for _f64) in device memory; d_spectrum =
 * double2[n_spectrum] in device memory, or NULL to use the handle's own buffer (read with b200dd_spectrum_fetch).
 * Asynchronous on `stream` (NULL = the handle's stream). */
B200DD_API int b200dd_spectrum_process_device(b200dd_spectrum *h, const void *d_x, uint32_t n, void *d_spectrum,
                                              void *stream);
B200DD_API int b200dd_spectrum_process_device_f64(b200dd_spectrum *h, const void *d_x, uint32_t n, void *d_spectrum,
                                                  void *stream);
/* The spectrum of a CPI whose reference channel is spread over GPUs.  fold_slice: fold the reference-channel samples
 * [sample0, sample0 + n) -- d_x[0] is global sample sample0, float2 -- into n_spectrum complex128 column sums at
 * d_part (the fold's contribution of those samples, before the t2 phase).  Samples at or past nfft contribute
 * nothing; a slice with none writes a zero part.  Parts of slices that cover [0, nfft) exactly once, handed to
 * b200dd_spectrum_finish_device, give the CPI's spectrum.  finish: sum n_parts parts (n_parts x n_spectrum
 * complex128, back to back) in index order, apply t2 and the n_spectrum-point DFT; d_spectrum nullable = the
 * handle's own buffer, as b200dd_spectrum_process_device.  One slice [0, n >= nfft) and a one-part finish equal
 * b200dd_spectrum_process_device bit for bit; parts summed in a fixed order give a spectrum that is deterministic for
 * a given partition.  Both asynchronous on `stream` (NULL = the handle's stream).  B200DD_ERR_ARG: a null handle or
 * d_part / d_parts, a null d_x with n > 0, n_parts == 0. */
B200DD_API int b200dd_spectrum_fold_slice_device(b200dd_spectrum *h, const void *d_x, uint32_t sample0, uint32_t n,
                                                 void *d_part, void *stream);
B200DD_API int b200dd_spectrum_finish_device(b200dd_spectrum *h, const void *d_parts, uint32_t n_parts, void *d_spectrum,
                                             void *stream);
/* Copies the handle's buffer (result of the last process_device call with d_spectrum == NULL) to the host and
 * synchronises the stream. */
B200DD_API int b200dd_spectrum_fetch(b200dd_spectrum *h, double *spectrum_out, void *stream);
/* Profiling aid: CUDA-event durations (ms) of the folding pass (the HBM-streaming kernel) and of the rest
 * (reduction + nSpectrum-point DFT).  Synchronises the stream. */
B200DD_API int b200dd_spectrum_profile_device(b200dd_spectrum *h, const void *d_x, uint32_t n, void *stream,
                                              float *ms_fold, float *ms_rest);
B200DD_API void *b200dd_spectrum_stream(b200dd_spectrum *h);

/* ------------------------------------------------------------------ map JSON
 *
 * The document blah2 sends on its map socket for every CPI: the std::string returned by
 * map->delay_bin_to_km(map->to_json(timestamp), fs) (src/blah2.cpp:303-304, src/data/Map.cpp:116-185), byte for
 * byte.  Members without whitespace in the order timestamp, nRows, nCols, noisePower, maxPower, delay (km),
 * doppler (Hz), data; data[k][j] = 10 log10|map[k][j]| - noisePower.  Doubles are rapidjson's Writer text at two
 * decimal places (shortest Grisu2 digits, TRUNCATED to two fraction digits); noisePower, maxPower, doppler and
 * the cells are that text read back by rapidjson's default Reader and written again, as delay_bin_to_km does.
 * The data body is rendered on the device (blah2_b200/csrc/mapjson.cu); the header is composed on the host.
 *
 * A map cell with |z| = 0, inf or NaN has no JSON number: rapidjson's Writer stops mid-document and blah2 then
 * fails parsing the truncated text.  Here the render reports B200DD_ERR_NONFINITE and writes no bytes.
 */
typedef struct b200dd_mapjson b200dd_mapjson;

/* Axes as Map holds them: delay[n_del] bins, doppler[n_dop] Hz; fs in Hz (delay km = delay c / fs / 1000). */
B200DD_API int b200dd_mapjson_create(uint32_t n_dop, uint32_t n_del, const int32_t *delay, const double *doppler,
                                     uint32_t fs, int32_t device, b200dd_mapjson **out);
/* Exact upper bound of a document's size in bytes for this handle, for any map and metrics (every double's text
 * is at most 24 bytes). */
B200DD_API size_t b200dd_mapjson_max_bytes(const b200dd_mapjson *h);
B200DD_API void b200dd_mapjson_destroy(b200dd_mapjson *h);
/* Renders the data body of d_map ([n_dop][n_del] float2, or double2 when is_f64) with the given metrics,
 * asynchronously on `stream` (NULL = the handle's stream).  d_map may be reused once the stream has passed it. */
B200DD_API int b200dd_mapjson_render_device(b200dd_mapjson *h, const void *d_map, int is_f64, double noise_power,
                                            double max_power, void *stream);
/* Composes the header with `timestamp` and copies the body straight behind it into out (pinned memory for a fast
 * copy); *n_bytes = document length (no terminating NUL).  Synchronises `stream` (the render's stream).
 * B200DD_ERR_NONFINITE: a value has no JSON text, nothing written.  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_mapjson_fetch(b200dd_mapjson *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes,
                                    void *stream);
/* Both steps for a HOST complex128 map (what Map<complex<double>>::data holds).  Synchronous. */
B200DD_API int b200dd_mapjson_render_host(b200dd_mapjson *h, const double *map, double noise_power, double max_power,
                                          uint64_t timestamp, char *out, size_t cap, size_t *n_bytes);
/* Test entry points: the text a client receives for each of n doubles (written, read back, written again),
 * comma-separated, an empty field for a value that has none (not finite, or its text reads back above DBL_MAX).
 * _host runs the formatter on the CPU (no device needed), _device runs it in a kernel. */
B200DD_API int b200dd_mapjson_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes);
B200DD_API int b200dd_mapjson_format_doubles_device(const double *v, uint32_t n, char *out, size_t cap,
                                                    size_t *n_bytes, int32_t device);
/* Test entry point: the double of every cell, 10 log10|z| - noise_power as the render computes it, into
 * d_out[n_dop * n_del] (device memory).  Asynchronous on `stream`. */
B200DD_API int b200dd_mapjson_debug_cell_values(b200dd_mapjson *h, const void *d_map, int is_f64, double noise_power,
                                                void *d_out, void *stream);

/* ------------------------------------------------------------------ max-hold map document
 *
 * The document blah2's API serves at /stash/map (api/stash/maxhold.js, api/server.js:96-97): the latest map
 * document (b200dd_mapjson_*) parsed by JSON.parse, its `data` replaced by the per-cell maximum over the last 20
 * documents, and sent as JSON.stringify of the result.  Every number is ECMAScript's Number::toString of the parsed
 * value: shortest round-trip digits, "12" for 12.0, "0" for -0.0, integers above 2^53 rounded
 * (18446744073709551615 -> "18446744073709552000").  A cell of a map document is always k/100 for an integer k,
 * so the window is kept on the device as int32 hundredths, and the maximum is taken on those.
 *
 * Each push is accepted or rejected on the device.  A rejected push leaves the window and header unchanged; it is
 * a CPI blah2 publishes no map document for: a cell with |z| = 0, inf or NaN, a noisePower or maxPower without
 * text (B200DD_ERR_NONFINITE), or a failed clutter-filter solve in the pipeline (B200DD_FILTER_FAILED).
 * Device memory: n_dop * n_del * 88 bytes (21 ring slots of int32, the window's maximum) plus the document. */
typedef struct b200dd_maxhold b200dd_maxhold;

/* Axes as Map holds them (see b200dd_mapjson_create). */
B200DD_API int b200dd_maxhold_create(uint32_t n_dop, uint32_t n_del, const int32_t *delay, const double *doppler,
                                     uint32_t fs, int32_t device, b200dd_maxhold **out);
/* Upper bound of a document's size in bytes for this handle. */
B200DD_API size_t b200dd_maxhold_max_bytes(const b200dd_maxhold *h);
B200DD_API void b200dd_maxhold_destroy(b200dd_maxhold *h);
/* Adds one CPI's map d_map ([n_dop][n_del] float2, or double2 when is_f64) with its set_metrics values,
 * asynchronously on `stream` (NULL = the handle's stream).  A finite |noise_power| > 1e7 dB returns
 * B200DD_ERR_ARG at once (the bound keeps every cell's hundredths inside int32); a non-finite one rejects the push. */
B200DD_API int b200dd_maxhold_push_device(b200dd_maxhold *h, const void *d_map, int is_f64, double noise_power,
                                          double max_power, void *stream);
/* Renders the window and writes header and body into out; *n_bytes = document length.  Synchronises `stream`.
 * B200DD_ERR_ARG: nothing held yet.  The last push's code when that push was rejected (nothing written: blah2
 * publishes nothing for that CPI).  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_maxhold_fetch(b200dd_maxhold *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes,
                                    void *stream);
/* Test entry points: for each of n doubles, the /stash/map text of a cell whose only held value is v,
 * comma-separated, an empty field where there is none (no map-document text, or hundredths outside int32).
 * _host runs on the CPU (no device needed), _device in a kernel. */
B200DD_API int b200dd_maxhold_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap, size_t *n_bytes);
B200DD_API int b200dd_maxhold_format_doubles_device(const double *v, uint32_t n, char *out, size_t cap,
                                                    size_t *n_bytes, int32_t device);

/* ------------------------------------------------------------------ detection JSON
 *
 * The document blah2 sends on its detection socket for every CPI: the std::string returned by
 * detection->delay_bin_to_km(detection->to_json(timestamp), fs) (src/blah2.cpp:312-317,
 * src/data/Detection.cpp:47-106), byte for byte:  {"timestamp":T,"delay":[..],"doppler":[..],"snr":[..]}.
 * doppler (Hz) and snr (dB) are rapidjson's text at two decimal places read back and written again; delay is
 * 1.0 * bin * (c / fs) / 1000 km, written once.  An empty list gives "delay":[],"doppler":[],"snr":[].  A value
 * without JSON text (inf, NaN, or a km value that overflows) makes rapidjson stop mid-document and blah2's re-parse
 * fail: B200DD_ERR_NONFINITE, nothing written.
 *
 * The handle also keeps the API's detection history, /stash/detection (api/stash/detection.js, api/server.js:99-100):
 * every fetched document enters it with its timestamp; after each one the API drops documents more than 300 s older
 * than the new one with its own loop, which tests only every other document from the front and removes one from the
 * front per stale test, so stale documents can stay.  The history is sent as JSON.stringify of
 * {"timestamp":[..],"delay":[..],"doppler":[..],"snr":[..]}: the detections of the held documents in order, each
 * with its document's timestamp, every number as Number::toString (see b200dd_maxhold_*); "[]" before the first
 * document.  Every delay, Doppler and SNR text is k/100 for an integer k, so the history is a device ring of int32
 * triples holding max_held detections.  Not reproduced: the API loses its first document after start and its 100 ms
 * polling skips documents that arrive faster; every fetched document is taken here.
 *
 * Limits: a value whose hundredths lie outside int32 (|v| >= 21474836.48) cannot enter the history: its fetch writes
 * the document and returns B200DD_ERR_ARG without committing it.  When committing a document would hold more than
 * max_held detections, its fetch writes the document and returns B200DD_ERR_CAPACITY, and the history is lost:
 * b200dd_detjson_fetch_stash returns B200DD_ERR_CAPACITY from then on, for the life of the handle (for a pipeline's
 * stage, until the stage is enabled again); later documents are still written and return B200DD_OK.
 * Device memory: about 20 MB for the document, plus max_held * 72 bytes for the history.
 */
typedef struct b200dd_detjson b200dd_detjson;

/* fs in Hz (the delay's km scale); max_held in [1, 2^25] detections held by the history. */
B200DD_API int b200dd_detjson_create(uint32_t fs, uint32_t max_held, int32_t device, b200dd_detjson **out);
/* Upper bound of a detection document's size in bytes (2^18 detections, every value's text at most 24 bytes). */
B200DD_API size_t b200dd_detjson_max_bytes(const b200dd_detjson *h);
/* Upper bound of the /stash/detection document's size in bytes. */
B200DD_API size_t b200dd_detjson_stash_max_bytes(const b200dd_detjson *h);
B200DD_API void b200dd_detjson_destroy(b200dd_detjson *h);
/* Renders the document body of a device detection list: d_delay (bins), d_doppler (Hz), d_snr (dB) doubles whose
 * length is the device word *d_count, read when the kernels run (at most 2^18 entries are read).  Asynchronous on
 * `stream` (NULL = the handle's stream); the launch shape does not depend on the count, so the call can be recorded
 * in a CUDA graph.  Also writes the values' hundredths into the history's ring, where the next commit takes them. */
B200DD_API int b200dd_detjson_render_device(b200dd_detjson *h, const double *d_delay, const double *d_doppler,
                                            const double *d_snr, const uint32_t *d_count, void *stream);
/* Writes the last render's document with `timestamp` into out (*n_bytes = its length), then commits it to the
 * history and prunes it.  Synchronises `stream` (the render's stream).  Each render is fetched once; B200DD_ERR_ARG
 * when nothing was rendered since the last fetch.  B200DD_ERR_CAPACITY, nothing written or committed: the count
 * exceeds 2^18 (*n_bytes = 0), or cap < *n_bytes (the same render may be fetched again).  B200DD_ERR_NONFINITE:
 * nothing written or committed.  See the limits above for B200DD_ERR_ARG / B200DD_ERR_CAPACITY with the document
 * written (*n_bytes <= cap). */
B200DD_API int b200dd_detjson_fetch(b200dd_detjson *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes,
                                    void *stream);
/* Writes the /stash/detection document into out; *n_bytes = its length.  Synchronises `stream`.
 * B200DD_ERR_CAPACITY: cap < *n_bytes, or the history overflowed. */
B200DD_API int b200dd_detjson_fetch_stash(b200dd_detjson *h, char *out, size_t cap, size_t *n_bytes, void *stream);
/* The detection document of n HOST detections, without a handle or a device.  B200DD_ERR_NONFINITE: a value has no
 * text, nothing written.  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_detjson_render_host(const double *delay, const double *doppler, const double *snr, uint32_t n,
                                          uint64_t timestamp, uint32_t fs, char *out, size_t cap, size_t *n_bytes);

/* ------------------------------------------------------------------ IQ-data JSON
 *
 * The document blah2 sends on its IQ-data socket for every CPI: the std::string returned by x->to_json(timestamp)
 * (src/blah2.cpp:299-300, src/data/IqData.cpp:93-125), byte for byte:
 *   {"timestamp":T,"min":m,"max":M,"mean":u,"frequency":[],"spectrum":[..]}
 * Each spectrum entry is 10 log10(hypot(re, im)) of one SpectrumAnalyser bin, written once by rapidjson's Writer at two
 * decimal places (no read-back); min, max and mean are written the same way.  frequency is always empty: the
 * analyser's uint32_t loop never runs.  blah2 never assigns IqData's min, max and mean, so here they are the values
 * the caller's IqData holds, fixed when the handle is created; a non-finite one is rejected with B200DD_ERR_ARG.  A bin
 * with |s| = 0, inf or NaN makes rapidjson's Writer stop mid-document: B200DD_ERR_NONFINITE, nothing written.
 *
 * The handle also keeps the API's history, /stash/iqdata (api/stash/iqdata.js, api/server.js:102-103): the spectrum,
 * frequency and timestamp of the last 20 fetched documents, sent as JSON.stringify of the newest document with those
 * three members replaced by the arrays, {"timestamp":[..],"min":m,"max":M,"mean":u,"frequency":[[],..],
 * "spectrum":[[..],..]}, every number as Number::toString (see b200dd_maxhold_*); "[]" before the first document.
 * Every spectrum text is k/100 for an integer k, so the history is a device ring of 21 int32 rows.  Not reproduced:
 * the API loses its first document after start, its 100 ms polling skips documents that arrive faster, and after a
 * truncated document blah2's socket text runs into the next one, which the API then loses too; every fetched document
 * is taken here.  Device memory: n_spectrum * 413 bytes.
 */
typedef struct b200dd_iqjson b200dd_iqjson;

/* n_spectrum in [1, 65536] bins; min, max, mean finite (else B200DD_ERR_ARG). */
B200DD_API int b200dd_iqjson_create(uint32_t n_spectrum, double min, double max, double mean, int32_t device,
                                    b200dd_iqjson **out);
/* Upper bound of an IQ-data document's size in bytes. */
B200DD_API size_t b200dd_iqjson_max_bytes(const b200dd_iqjson *h);
/* Upper bound of the /stash/iqdata document's size in bytes. */
B200DD_API size_t b200dd_iqjson_stash_max_bytes(const b200dd_iqjson *h);
B200DD_API void b200dd_iqjson_destroy(b200dd_iqjson *h);
/* Renders the document body of a device spectrum d_spectrum = double2[n_spectrum], asynchronously on `stream` (NULL =
 * the handle's stream); the launch shape depends only on n_spectrum, so the call can be recorded in a CUDA graph.
 * Also writes the bins' hundredths into the history's free row, where the next commit takes them. */
B200DD_API int b200dd_iqjson_render_device(b200dd_iqjson *h, const void *d_spectrum, void *stream);
/* Writes the last render's document with `timestamp` into out (*n_bytes = its length), then commits it to the
 * history.  Synchronises `stream` (the render's stream).  Each render is fetched once; B200DD_ERR_ARG when nothing was
 * rendered since the last fetch.  B200DD_ERR_NONFINITE: nothing written or committed.  B200DD_ERR_CAPACITY: cap <
 * *n_bytes, nothing written or committed (the same render may be fetched again). */
B200DD_API int b200dd_iqjson_fetch(b200dd_iqjson *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes,
                                   void *stream);
/* Writes the /stash/iqdata document into out; *n_bytes = its length.  Synchronises `stream`.
 * B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_iqjson_fetch_stash(b200dd_iqjson *h, char *out, size_t cap, size_t *n_bytes, void *stream);
/* The IQ-data document of n HOST bins (complex128), without a handle or a device.  B200DD_ERR_ARG: a non-finite
 * min, max or mean.  B200DD_ERR_NONFINITE: a bin has no text, nothing written.  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_iqjson_render_host(const double *spectrum, uint32_t n, double min, double max, double mean,
                                         uint64_t timestamp, char *out, size_t cap, size_t *n_bytes);
/* Test entry point: the double of every bin, 10 log10|s| as the render computes it, into d_out[n_spectrum] (device
 * memory).  Asynchronous on `stream`. */
B200DD_API int b200dd_iqjson_debug_bin_values(b200dd_iqjson *h, const void *d_spectrum, void *d_out, void *stream);

/* ------------------------------------------------------------------ timing JSON
 *
 * The document blah2 sends on its timing socket after every CPI (src/blah2.cpp:331-345, Timing::to_json in
 * src/data/meta/Timing.cpp), byte for byte:
 *   {"timestamp":T,"nCpi":n,"uptime_s":u/1000.0,"uptime_days":u/1000.0/60/60/24,"<stage>":ms,...}
 * T = t_now, n and u = t_now - t_start (uint64, wrapping when t_now < t_start) are written as integers / doubles by
 * rapidjson's Writer at two decimal places; each stage is a name and a time in ms.  In the pipeline (see
 * b200dd_pipeline_enable_timing_json) the times come from device stamps at the chain's stage boundaries.
 */
/* The document of `count` (<= 16) stages, without a handle or a device.  B200DD_ERR_ARG: a null pointer, a name
 * that is null, 64 bytes or longer or not printable ASCII without '"' and '\\' (names are written unescaped), or a
 * non-finite time (the Writer has no text for it).  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_timing_render_host(uint64_t t_start, uint64_t t_now, uint64_t n, const char *const *names,
                                         const double *values, uint32_t count, char *out, size_t cap,
                                         size_t *n_bytes);
/* Upper bound of a timing document's size in bytes (16 stages of 63-byte names). */
B200DD_API size_t b200dd_timing_max_bytes(void);

/* ------------------------------------------------------------------ tracker
 *
 * Tracker::process + Track::to_json (src/process/tracker/Tracker.cpp, src/data/Track.cpp; blah2.cpp:291-296 and
 * :324-328), with the track state kept on the device between CPIs.  The code is reproduced as written, quirks
 * included (DESIGN.md §9): association tests every detection against delay 0, Doppler 0 rather than against the
 * prediction, so one detection -- the first inside |delay| < 1, |Doppler| < 1/cpi -- associates with every track
 * the CPI reaches; the inactivity counters belong to vector positions, not tracks; each removal skips the next track.
 * The document is {"timestamp":T,"n":..,"nTentative":..,"nAssociated":..,"nActive":..,"nCoasting":..,"data":[..]},
 * every double written once at two decimals (delays stay in bins).
 *
 * Limits: the reference has none.  max_tracks live tracks and max_history entries per track are set at creation and
 * raised by b200dd_tracker_reserve; a CPI that would exceed either puts the handle in an overflowed state in which
 * process does nothing and fetch returns B200DD_ERR_CAPACITY with *n_bytes = 0, until b200dd_tracker_reset.  Inactivity counters are 32-bit.
 * Device memory: 16 max_history + 4 ceil(max_history / 16) + 52 bytes per track slot, plus the document body
 * (grown to the largest document fetched so far).
 */
typedef struct b200dd_tracker b200dd_tracker;

typedef struct {
  uint32_t m, n;        /* process.tracker.initiate.M / .N: promote when m of the last n states associate */
  uint32_t n_delete;    /* process.tracker.delete */
  double cpi;           /* Ambiguity::get_cpi() (s) */
  double max_acc_init;  /* process.tracker.initiate.maxAcc (Hz/s) */
  uint32_t fs, fc;      /* capture.fs, capture.fc (Hz): rangeRes = c / fs, lambda = c / fc */
} b200dd_tracker_params;

/* Host only.  *n_hypotheses = 2 nAcc + 1, the tracks each unassociated detection starts, nAcc =
 * (uint16_t)((int)max_acc_init / (1 / (cpi cpi))); *max_bytes = the document size bound; *device_bytes = the device
 * memory of the track state (all nullable).  B200DD_ERR_ARG when a conversion is undefined ((int)max_acc_init outside
 * int, the uint16 conversion of a NaN or of a value outside (-1, 65536)), nAcc > 4096, fs or fc of 0, max_tracks
 * outside [1, 2^24], max_history outside [1, 2^16], or a document bound of 2^32 bytes or more. */
B200DD_API int b200dd_tracker_plan(const b200dd_tracker_params *params, uint32_t max_tracks, uint32_t max_history,
                                   uint32_t *n_hypotheses, size_t *max_bytes, size_t *device_bytes);
B200DD_API int b200dd_tracker_create(const b200dd_tracker_params *params, uint32_t max_tracks, uint32_t max_history,
                                     int32_t device, b200dd_tracker **out);
B200DD_API void b200dd_tracker_destroy(b200dd_tracker *h);
/* Back to the constructed state: no tracks, timestamp 0, id counter 0, counters 0, not overflowed.  Synchronous. */
B200DD_API int b200dd_tracker_reset(b200dd_tracker *h);
/* The document size bound of the handle's limits. */
B200DD_API size_t b200dd_tracker_max_bytes(const b200dd_tracker *h);
/* Raises the limits of a live handle to max(max_tracks, current) x max(max_history, current) without changing its
 * state: every track, its history, the order of the tracks, the inactivity counters, the id counter and the timestamp
 * carry over, and every later document is the one a handle created at the larger limits gives.  The new limits'
 * arrays are allocated, a kernel on `stream` (NULL = the handle's stream) moves the state into them, and the old
 * arrays are freed (cudaFree waits for the device).  A request that raises neither limit does nothing.
 * B200DD_ERR_ARG, with the handle unchanged, where b200dd_tracker_plan refuses the new limits.  An overflowed handle
 * stays overflowed.  The growth rule belongs to the caller: before a CPI of n detections, live + n * n_hypotheses
 * tracks and longest + 2 history entries cannot overflow (every unassociated detection starts n_hypotheses tracks,
 * and a CPI adds at most the association and the prediction to a history). */
B200DD_API int b200dd_tracker_reserve(b200dd_tracker *h, uint32_t max_tracks, uint32_t max_history, void *stream);
/* The live track count and the longest history among the live tracks, after the work enqueued on `stream`
 * (NULL = the handle's stream).  Synchronises `stream`. */
B200DD_API int b200dd_tracker_usage(b200dd_tracker *h, uint32_t *live_tracks, uint32_t *longest_history,
                                    void *stream);
/* Tracker::process(detection, timestamp) on a device detection list: d_delay (bins), d_doppler (Hz) doubles whose
 * length is the device word *d_count (d_snr is accepted for the Detection's shape; the tracker never reads it).
 * Asynchronous on `stream` (NULL = the handle's stream): no host synchronisation and no count read on the host. */
B200DD_API int b200dd_tracker_process_device(b200dd_tracker *h, const double *d_delay, const double *d_doppler,
                                             const double *d_snr, const uint32_t *d_count, uint64_t timestamp,
                                             void *stream);
/* The same on n HOST detections: copies them to the device and runs the same kernels (asynchronous; the host
 * arrays may be reused on return). */
B200DD_API int b200dd_tracker_process_host(b200dd_tracker *h, const double *delay, const double *doppler,
                                           const double *snr, uint32_t n, uint64_t timestamp, void *stream);
/* Track::to_json(timestamp) of the current tracks into out; *n_bytes = its length.  Synchronises `stream`.  May be
 * called any number of times.  B200DD_ERR_CAPACITY: cap < *n_bytes (nothing written), or the handle overflowed
 * (*n_bytes = 0).  B200DD_ERR_NONFINITE: a value the document holds is not finite (rapidjson's Writer stops there;
 * an association with T = 0 makes one), nothing written; the state has advanced as the reference's does. */
B200DD_API int b200dd_tracker_fetch(b200dd_tracker *h, uint64_t timestamp, char *out, size_t cap, size_t *n_bytes,
                                    void *stream);
/* Host only: the text Writer::Double gives each of n doubles at two decimal places (the track document's numbers),
 * comma-separated, an empty text for a non-finite value.  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_tracker_format_doubles_host(const double *v, uint32_t n, char *out, size_t cap,
                                                  size_t *n_bytes);

/* ------------------------------------------------------------------ whole CPI pipeline
 *
 * One coherent-processing interval through the body of the reference's process thread
 * (src/blah2.cpp:268-287): [WienerHopf::process] -> Ambiguity::process -> Map::set_metrics ->
 * [CfarDetector1D -> Centroid -> Interpolate], with every intermediate (filtered surveillance
 * channel, range matrix, map, detection lists) staying in device memory.  The per-class entry
 * points above remain the drop-in boundary; this is the path a maintainer takes when the caller
 * can hand over a whole CPI at once (INTEGRATION.md "fast path").
 */
typedef struct b200dd_pipeline b200dd_pipeline;

typedef struct {
  b200dd_caf_params caf;
  int32_t clutter_enable;     /* process.clutter.enable   (config/config.yml:28-32) */
  int32_t clutter_delay_min;
  int32_t clutter_delay_max;
  int32_t detection_enable;   /* process.detection.enable (config/config.yml:33-40) */
  b200dd_det_params det;      /* det.resolution_doppler = 1 / tCpi as blah2.cpp:183 passes it */
} b200dd_pipeline_params;

typedef struct {
  int32_t filter_status;   /* B200DD_OK, or B200DD_FILTER_FAILED: the CPI is skipped like blah2.cpp:270-273 --
                              n_detections, noise_power and max_power are then 0 and the map buffer is not a product */
  uint32_t n_detections;
  double noise_power;      /* Map::noisePower */
  double max_power;        /* Map::maxPower   */
} b200dd_cpi_result;

B200DD_API int b200dd_pipeline_create(const b200dd_pipeline_params *params, b200dd_pipeline **out);
B200DD_API void b200dd_pipeline_destroy(b200dd_pipeline *h);
B200DD_API int b200dd_pipeline_get_geometry(const b200dd_pipeline *h, b200dd_caf_geometry *out);
B200DD_API int b200dd_pipeline_get_axes(const b200dd_pipeline *h, int32_t *delay, double *doppler);

/* HOST buffers: x, y = n complex128 samples (n == n_samples when the clutter filter is enabled,
 * >= n_used otherwise).  map_out (nullable) = [nDop][nDel] complex128.  Detections into the three
 * arrays (capacity cap).  Synchronous: returns when the results are in host memory. */
B200DD_API int b200dd_pipeline_process_host(b200dd_pipeline *h, const double *x, const double *y, uint32_t n,
                                            double *map_out, b200dd_cpi_result *result, double *o_delay,
                                            double *o_doppler, double *o_snr, uint32_t cap);

/* Asynchronous form of the host entry: enqueues H2D, all kernels and the D2H of the map on the
 * pipeline's own stream and returns; x, y and map_out must stay valid (pinned memory for true
 * overlap) until b200dd_pipeline_fetch returns.  Two pipelines used alternately overlap the PCIe
 * transfers of one CPI with the kernels of the other. */
B200DD_API int b200dd_pipeline_submit_host(b200dd_pipeline *h, const double *x, const double *y, uint32_t n,
                                           double *map_out);

/* Same, fed with the reference's replay / capture layout: n time instants of little-endian int16
 * I1 Q1 I2 Q2 (src/capture/rspduo/RspDuo.cpp:155-174; channel 1 = reference, channel 2 = surveillance).
 * 8 bytes per instant cross PCIe instead of 32; the de-interleave runs on the device.  int16 is exact
 * in float32, so results equal the complex128 entry point's. */
B200DD_API int b200dd_pipeline_submit_host_rspduo(b200dd_pipeline *h, const int16_t *iq, uint32_t n, double *map_out);

/* Same as b200dd_pipeline_submit_host_rspduo, fed with HackRF's and Kraken's sample format: x_iq (reference) and
 * y_iq (surveillance) are two buffers of n time instants each, every instant an int8 pair I, Q.  HackRF delivers one
 * such buffer per device (src/capture/hackrf/HackRf.cpp:116-128).  Kraken's rtl-sdr bytes are offset binary centred
 * on 127.5, but blah2 reads them as int8_t (src/capture/kraken/Kraken.cpp:97-112), so a byte >= 0x80 is negative
 * here too and no offset is removed.  4 bytes per instant cross PCIe; the conversion to complex64 runs on the
 * device.  int8 is exact in float32, so results equal the int16 entry point's on the same values.  Asynchronous on
 * the pipeline's stream; pair with b200dd_pipeline_fetch.  x_iq, y_iq and map_out (nullable) must stay valid until
 * the fetch returns (pinned memory for overlap).  Errors as b200dd_pipeline_submit_host_rspduo's. */
B200DD_API int b200dd_pipeline_submit_host_ci8(b200dd_pipeline *h, const int8_t *x_iq, const int8_t *y_iq, uint32_t n,
                                               double *map_out);

/* Same, fed with USRP's sample format: x_iq and y_iq are two buffers of n complex float32 samples (I, Q) each, the
 * UHD fc32 host format blah2 receives (src/capture/usrp/Usrp.cpp:54-91).  16 bytes per instant cross PCIe, copied
 * straight into the device chain's complex64 buffers; results equal b200dd_pipeline_submit_device's on the same
 * samples.  Asynchronous, lifetimes and errors as b200dd_pipeline_submit_host_ci8's. */
B200DD_API int b200dd_pipeline_submit_host_cf32(b200dd_pipeline *h, const float *x_iq, const float *y_iq, uint32_t n,
                                                double *map_out);

/* DEVICE buffers (float2), asynchronous on `stream` (NULL = the pipeline's stream).  d_map
 * (nullable) receives the float2 map.  Results stay on the device until b200dd_pipeline_fetch.
 * Ordering: every submit entry (this one, prepare_device, submit_host*, submit_map, submit_record) runs after the
 * pipeline's last CPI, whatever stream either uses: when the last CPI went on another stream and has not been fetched,
 * the new stream waits for it on the device (the host never waits).  On the last CPI's own stream nothing extra is
 * enqueued.  The stream a CPI was submitted on must stay alive until the CPI is fetched. */
B200DD_API int b200dd_pipeline_submit_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n,
                                             void *d_map, void *stream);
/* Plan creation for the device path (optional): records the whole chain for this (d_x, d_y, d_map) triple as a CUDA
 * graph -- it runs the chain once on the buffers' current contents, captures and instantiates it and synchronises
 * the stream -- after which b200dd_pipeline_submit_device on the same triple is ONE cudaGraphLaunch.  Results are
 * identical either way.  Worth it for submit -> fetch -> submit loops over a fixed ring of buffers;
 * with many CPIs enqueued ahead eager launches can be faster, hence opt-in: a triple that was never prepared is
 * enqueued eagerly.  Where the chain cannot be captured, the pipeline stays eager and this call does nothing. */
B200DD_API int b200dd_pipeline_prepare_device(b200dd_pipeline *h, const void *d_x, const void *d_y, uint32_t n,
                                              void *d_map, void *stream);
/* The last CPI's clutter-filter status, set_metrics and detection list into host memory, read on `stream` (NULL =
 * the pipeline's stream) after that CPI, whichever stream it was submitted on; returns when they are there. */
B200DD_API int b200dd_pipeline_fetch(b200dd_pipeline *h, b200dd_cpi_result *result, double *o_delay,
                                     double *o_doppler, double *o_snr, uint32_t cap, void *stream);
B200DD_API void *b200dd_pipeline_stream(b200dd_pipeline *h);

/* Optional first stage of the process thread (src/blah2.cpp:263-265): SpectrumAnalyser(n_samples, bandwidth) on
 * the reference channel of every CPI submitted afterwards, evaluated on the samples already resident on the
 * device (no extra transfer).  *n_spectrum (nullable) receives the number of bins.  The spectrum of the last
 * submitted CPI is read with b200dd_pipeline_fetch_spectrum (call it after b200dd_pipeline_fetch, or it
 * waits for that CPI itself). */
B200DD_API int b200dd_pipeline_enable_spectrum(b200dd_pipeline *h, double bandwidth, uint32_t *n_spectrum);
B200DD_API int b200dd_pipeline_fetch_spectrum(b200dd_pipeline *h, double *spectrum_out, uint32_t cap);

/* Optional last stage (src/blah2.cpp:303-304): renders the map document (see b200dd_mapjson_*) of every CPI
 * submitted afterwards, right after set_metrics, with the noisePower set_metrics left on the device (no host round
 * trip); works in recorded graphs.  Drops the graphs recorded so far.  *max_bytes (nullable) = the document size
 * bound.  b200dd_pipeline_fetch_map_json, called after b200dd_pipeline_fetch, writes the last CPI's document;
 * it returns B200DD_FILTER_FAILED and writes nothing when that CPI's clutter-filter solve failed (the reference
 * skips the CPI and sends no map, blah2.cpp:270-273). */
B200DD_API int b200dd_pipeline_enable_map_json(b200dd_pipeline *h, size_t *max_bytes);
B200DD_API int b200dd_pipeline_fetch_map_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                              size_t *n_bytes);

/* Optional stage after set_metrics: pushes every CPI submitted afterwards into a max-hold window (see
 * b200dd_maxhold_*), with the metrics set_metrics left on the device and the clutter filter's status word (no host
 * round trip); works in recorded graphs.  Independent of the map JSON stage.  Drops the graphs recorded so far.
 * b200dd_pipeline_fetch_maxhold, called after b200dd_pipeline_fetch, writes the /stash/map document after the last
 * CPI; it returns B200DD_FILTER_FAILED, with the window unchanged, when that CPI's solve failed, and
 * B200DD_ERR_ARG when the stage is not enabled or no CPI was accepted yet. */
B200DD_API int b200dd_pipeline_enable_maxhold(b200dd_pipeline *h, size_t *max_bytes);
B200DD_API int b200dd_pipeline_fetch_maxhold(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                             size_t *n_bytes);

/* Optional last stage (src/blah2.cpp:312-317): renders the detection document (see b200dd_detjson_*) of every CPI
 * submitted afterwards from the detection list on the device, and keeps the /stash/detection history of up to
 * max_held detections; works in recorded graphs.  Drops the graphs recorded so far and starts an empty history.
 * *doc_bytes / *stash_bytes (nullable) = the two documents' size bounds.  B200DD_ERR_ARG when the pipeline has no
 * detection stage; B200DD_ERR_GEOMETRY when an Interpolate result on the pipeline's axes (delay within one bin of
 * the delay axis, Doppler within one bin of the Doppler axis) could have hundredths outside int32.  SNR needs no
 * check: from a float map it lies within about +-1700 dB. */
B200DD_API int b200dd_pipeline_enable_detection_json(b200dd_pipeline *h, uint32_t max_held, size_t *doc_bytes,
                                                     size_t *stash_bytes);
/* Called after b200dd_pipeline_fetch: writes the last CPI's detection document (all its detections, whatever cap
 * b200dd_pipeline_fetch was given) and commits it to the history, as b200dd_detjson_fetch.  B200DD_FILTER_FAILED,
 * nothing written or committed, when that CPI's clutter-filter solve failed (blah2.cpp:270-273 skips the CPI);
 * B200DD_ERR_CAPACITY, nothing written or committed, when CFAR found more detections than the list holds. */
B200DD_API int b200dd_pipeline_fetch_detection_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                                    size_t *n_bytes);
/* The /stash/detection document of the pipeline's history (see b200dd_detjson_fetch_stash). */
B200DD_API int b200dd_pipeline_fetch_detection_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes);

/* Optional stage (src/blah2.cpp:291-296, :324-328): a tracker (see b200dd_tracker_*) fed with every CPI's device
 * detection list.  params->cpi and params->fs are replaced by the pipeline's geometry and CAF params.
 * B200DD_ERR_ARG when the pipeline has no detection stage (blah2.cpp:206-209 disables the tracker then).  Starts a
 * fresh tracker; the submitted chain does not change.  *max_bytes (nullable) = the document size bound. */
B200DD_API int b200dd_pipeline_enable_tracker(b200dd_pipeline *h, const b200dd_tracker_params *params,
                                              uint32_t max_tracks, uint32_t max_history, size_t *max_bytes);
/* Called after b200dd_pipeline_fetch: the first call after a submit runs Tracker::process on that CPI's device
 * detection list with `timestamp`; every call then writes the document, as b200dd_tracker_fetch (a call with a
 * too-small cap can be repeated).  B200DD_FILTER_FAILED when the CPI's clutter-filter solve failed (blah2.cpp:270-273
 * skips the CPI) and B200DD_ERR_CAPACITY with *n_bytes = 0 when CFAR found more detections than the list holds:
 * nothing written, the tracker unchanged. */
B200DD_API int b200dd_pipeline_fetch_track_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                                size_t *n_bytes);

/* Optional stage after the spectrum (src/blah2.cpp:299-300): renders the IQ-data document (see b200dd_iqjson_*) of
 * every CPI submitted afterwards from the spectrum stage's device buffer, right after the spectrum kernels, and keeps
 * the /stash/iqdata history; works in recorded graphs.  min, max and mean are the IqData members the document
 * carries.  Drops the graphs recorded so far and starts an empty history.  *doc_bytes / *stash_bytes (nullable) =
 * the two documents' size bounds.  B200DD_ERR_ARG when the spectrum stage is not enabled or a metric is not finite.
 * b200dd_pipeline_enable_spectrum disables this stage (it may change the number of bins): enable it again after. */
B200DD_API int b200dd_pipeline_enable_iqdata_json(b200dd_pipeline *h, double min, double max, double mean,
                                                  size_t *doc_bytes, size_t *stash_bytes);
/* Called after b200dd_pipeline_fetch: writes the last CPI's IQ-data document and commits it to the history, as
 * b200dd_iqjson_fetch.  B200DD_FILTER_FAILED, nothing written or committed, when that CPI's clutter-filter solve
 * failed (blah2.cpp:270-273 skips the CPI). */
B200DD_API int b200dd_pipeline_fetch_iqdata_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                                 size_t *n_bytes);
/* The /stash/iqdata document of the pipeline's history (see b200dd_iqjson_fetch_stash). */
B200DD_API int b200dd_pipeline_fetch_iqdata_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes);

/* Optional stage (src/blah2.cpp:251-345): every CPI submitted afterwards stamps %globaltimer on the device at its
 * stage boundaries, on the submit stream (so recorded graphs stamp too), and its timing document (see
 * b200dd_timing_render_host) is built from those stamps; the API's /stash/timing history is kept.  Timing(t_start):
 * enabling resets nCpi and the history and drops the graphs recorded so far.  Stages, in blah2's order and under
 * blah2's conditions, each the time between two device stamps in ms (ns / 1e6):
 *   extract_buffer        host submits: the H2D copy plus the conversion to complex64 (for b200dd_pipeline_submit_host
 *                         that conversion runs after the filter); device submits: 0
 *   spectrum              the spectrum kernels and the IQ-data render (when the spectrum stage is enabled)
 *   clutter_filter        the WienerHopf kernels (when the clutter filter is enabled)
 *   ambiguity_processing  CAF and set_metrics (after b200dd_pipeline_submit_map: from the clutter boundary to the end
 *                         of set_metrics -- whatever the caller enqueued after that stamp, for SingleCpiPlan the
 *                         distributed CAF and the tile placement, then the spectrum finish, the IQ-data render and
 *                         set_metrics)
 *   detector              CFAR -> Centroid -> Interpolate (when detection is enabled)
 *   tracker               the tracker run at the CPI's first track fetch (when the tracker is enabled; 0 when CFAR
 *                         overflowed and the tracker skipped the CPI)
 *   output_radar_data     the map document, the max-hold push and the detection document enqueued after detection
 *   cpi                   the CPI's first stamp to its last, plus tracker
 * *doc_bytes / *stash_bytes (nullable) = the two documents' size bounds.  With the stage off nothing is stamped. */
B200DD_API int b200dd_pipeline_enable_timing_json(b200dd_pipeline *h, uint64_t t_start, size_t *doc_bytes,
                                                  size_t *stash_bytes);
/* Called after b200dd_pipeline_fetch (and, when the tracker is enabled, after the CPI's track fetch): writes the
 * last CPI's timing document with t_now = timestamp and commits it -- nCpi steps and the history takes it.  Each CPI
 * is committed once.  B200DD_ERR_ARG, nothing written or committed: called too early, or again.
 * B200DD_FILTER_FAILED, nothing written or committed: the CPI's clutter-filter solve failed (blah2.cpp:270-273 skips
 * Timing::update).  A CFAR overflow does not stop the document.  B200DD_ERR_CAPACITY: cap < *n_bytes, nothing
 * written or committed.  The history holds every value as int64 hundredths: a value whose text has more than 15
 * significant digits (a wrapped uptime, a timestamp of 10^15 ms or more) cannot enter it exactly, so the document is
 * written and B200DD_ERR_ARG returned, nothing committed. */
B200DD_API int b200dd_pipeline_fetch_timing_json(b200dd_pipeline *h, uint64_t timestamp, char *out, size_t cap,
                                                 size_t *n_bytes);
/* The /stash/timing document (api/stash/timing.js, api/server.js:105-106): JSON.stringify of an object holding, for
 * every key of the committed documents but "uptime" and "nCpi", the array of its last 20 values (keys in first-seen
 * order, numbers as Number::toString); "{}" before the first document.  B200DD_ERR_CAPACITY: cap < *n_bytes. */
B200DD_API int b200dd_pipeline_fetch_timing_stash(b200dd_pipeline *h, char *out, size_t cap, size_t *n_bytes);
/* Test entry point: the stage names (static strings) and times behind the last timing document written into
 * names[cap] / values[cap]; *count = their number.  B200DD_ERR_ARG: no document yet.  B200DD_ERR_CAPACITY: cap <
 * *count. */
B200DD_API int b200dd_pipeline_debug_timing_values(b200dd_pipeline *h, const char **names, double *values,
                                                   uint32_t cap, uint32_t *count);

/* Share set: makes the stateful stages of n pipelines -- the max-hold window, the detection and IQ-data histories
 * and the tracker -- one object, so that pipelines used alternately (to overlap one CPI's transfers with another's
 * kernels) keep blah2's "last 20 CPIs", "last 300 s" and "the tracker sees every CPI".  The set's CPIs are numbered
 * in submit order across its members.  After every fetch, the /stash/map, /stash/detection, /stash/iqdata and track
 * documents equal those of one unshared pipeline given the same CPIs one after another (fetching every product after
 * every CPI).  Per-CPI products (fetch's results, the spectrum, the map, detection and IQ-data documents) stay per
 * member.
 *  - A member holds at most one unfetched CPI: submit (and prepare_device when it runs the chain, which is a CPI)
 *    returns B200DD_ERR_ARG, nothing enqueued, while its last CPI is not fetched.
 *  - b200dd_pipeline_fetch must follow submit order across the set: B200DD_ERR_ARG, nothing consumed, for any CPI
 *    other than the oldest unfetched one.  A member's CPI enters the max-hold window at that fetch (an unshared
 *    pipeline pushes it at submit): a CPI that is never fetched never enters the window.  Its float2 map buffer must
 *    stay untouched until then.
 *  - The histories take a CPI at its document fetch, the tracker at the first b200dd_pipeline_fetch_track_json after
 *    b200dd_pipeline_fetch.  A product fetch for a CPI older than the one that product took last returns
 *    B200DD_ERR_ARG and commits nothing; so does fetch_maxhold on any CPI but the window's last, and fetch_track_json
 *    before the member's fetch.  B200DD_FILTER_FAILED, B200DD_ERR_NONFINITE and B200DD_ERR_CAPACITY commit nothing.
 *  - The existing fetch entry points of any member read and commit the shared state.
 * B200DD_ERR_ARG, nothing changed, when n is 0, a member is null, given twice or in a set already, the members sit on
 * different devices, or their b200dd_pipeline_params, spectrum stages (enabled, bandwidth) or stateful stages
 * (enabled, IQ-data min / max / mean, max_held, tracker params and limits) differ.  Histories start empty; the
 * members' recorded graphs are dropped.  On a member, enabling a stateful stage returns B200DD_ERR_ARG, and so does
 * b200dd_pipeline_enable_spectrum when the set keeps an IQ-data history (it would disable the member's IQ-data
 * render); the map document and the spectrum stay per member.  Destroying a member leaves the set; the last one
 * frees the shared state.  Every operation on the shared state is ordered after the previous one by a CUDA event,
 * whichever member's stream it runs on; nothing synchronises the host beyond what each call already does.
 * The timing stage, when enabled alike with the same t_start, shares one Timing (nCpi, uptime) and one /stash/timing
 * history; its stamps stay per member, and its documents follow the same commit rule as the histories. */
B200DD_API int b200dd_pipeline_share_history(b200dd_pipeline *const *members, uint32_t n);

/* CPI records: independent CPIs over GPUs with every product on one rank.  A pipeline that computes a CPI exports
 * it as one fixed-size device record holding everything its fetches read besides the map: the clutter-filter status,
 * set_metrics' noisePower and maxPower, CFAR's count, the detection list, the spectrum (spectrum stage) and the
 * timing stamps (timing stage).  Another pipeline, created with the same parameters and spectrum / timing stages,
 * on any GPU, takes the record and the map as if it had run the CPI itself: every fetch, stash, the tracker and the
 * share-set rules apply unchanged.  The record's layout is private to the library; only its size is public.
 *
 * enable_export: from now on every submit (submit_device eager or graph-replayed, submit_host, _rspduo, _ci8,
 * _cf32, and prepare_device's runs) ends its chain with one pack kernel that writes the CPI's record into a device
 * buffer the pipeline owns.  max_detections (1 .. 2^18) detection slots of 24 bytes each bound the record:
 * *record_bytes (nullable) = 64 + 80 with the timing stage + 16 nSpectrum with the spectrum stage + 24
 * max_detections with detection, rounded up to 16.  A CPI with more detections than slots carries the first
 * max_detections and is marked as overflowed.  Enabling the spectrum or timing stage later changes the layout;
 * *record_bytes is then b200dd_pipeline_export_record's buffer size from the next submit on.  Recorded graphs are
 * dropped (prepare_device records them again).  Without this call nothing is enqueued: every submit runs the
 * kernels it ran before.  B200DD_ERR_ARG: max_detections out of range, null handle.
 *
 * export_record: *d_record = the device record of the last submit.  It stays valid until the next submit on this
 * pipeline and is written on the stream that submit ran on (b200dd_pipeline_stream for the host submits).
 * B200DD_ERR_ARG when export is not enabled or nothing was submitted since.
 *
 * submit_record: the importing pipeline takes the CPI of record d_record and float2 map d_map (nDoppler x nDelay,
 * the exporter's map bytes): on b200dd_pipeline_stream(h) it writes the record into its own detection list,
 * metrics and status words, spectrum and stamps, then runs the renders a submit runs after the map -- the map
 * document body on d_map, the IQ-data and detection documents, and the max-hold push (at fetch for a share-set
 * member).  Both buffers must be complete, or ordered before that stream's work, at the call: it reads the record's
 * header synchronously.  d_map must stay untouched until b200dd_pipeline_fetch, as a share-set member's map does.
 * Afterwards b200dd_pipeline_fetch, fetch_spectrum and every fetch_*_json / fetch_*_stash behave as after a submit:
 *  - a failed clutter-filter solve imports as B200DD_FILTER_FAILED: nothing is committed, nCpi does not step;
 *  - a CFAR overflow imports as that overflow;
 *  - a record overflow behaves as a CFAR overflow: fetch and fetch_detection_json return B200DD_ERR_CAPACITY,
 *    nothing enters the detection history and the tracker skips the CPI;
 *  - the timing document's stage times come from the exporter's stamps (differences between stamps of one GPU);
 *    `tracker` is measured here, at the track fetch.
 * Importers may be share-set members (the set's rules apply, the import counts as a submit).  B200DD_ERR_ARG,
 * nothing enqueued: a null argument, not a record of this version, a record from a pipeline whose parameters or
 * spectrum / timing stages differ, a share-set member whose last CPI is not fetched. */
B200DD_API int b200dd_pipeline_enable_export(b200dd_pipeline *h, uint32_t max_detections, size_t *record_bytes);
B200DD_API int b200dd_pipeline_export_record(b200dd_pipeline *h, const void **d_record);
B200DD_API int b200dd_pipeline_submit_record(b200dd_pipeline *h, const void *d_record, const void *d_map);

/* One CPI over GPUs with every product on one rank (blah2_b200.shard.SingleCpiPlan): no GPU holds the whole CPI, so
 * no rank can export a record; the importing pipeline, created with the full parameters, takes the assembled map and
 * runs everything after the CAF itself.
 *
 * submit_map: the pipeline takes a CPI whose float2 map d_map (nDoppler x nDelay) was computed elsewhere, e.g. placed
 * from the tiles of SingleCpiPlan.  d_filter_status: a device int holding the clutter-filter verdict (required iff
 * the clutter filter is enabled; b200dd_wh_device_status of a chunk handle holds the global one, the solve being
 * replicated).  d_spectrum_parts / n_parts: the parts of b200dd_spectrum_fold_slice_device (required iff the spectrum
 * stage is enabled).  On `stream` (NULL = the pipeline's stream), ordered after what is already there, without host
 * synchronisation, it enqueues: the spectrum finish into the pipeline's spectrum buffer and the IQ-data render; a
 * copy of the verdict into the pipeline's clutter-filter status word; set_metrics and the detection stages on d_map;
 * the map document, the max-hold push (at fetch for a share-set member) and the detection document; the detector and
 * output stamps.  d_map must stay untouched until b200dd_pipeline_fetch.  Afterwards every fetch, stash, the tracker
 * and the share-set rules behave as after a submit (path: device); a verdict of B200DD_FILTER_FAILED imports as a
 * failed solve: nothing is committed, nCpi does not step.  No record is packed, and no graph is recorded.
 * B200DD_ERR_ARG, nothing enqueued: a null h or d_map; a status given without the clutter filter or missing with it;
 * parts given without the spectrum stage, missing with it, or n_parts == 0; a share-set member whose last CPI is not
 * fetched.
 *
 * stamp: timing stage, the boundary `slot` (B200DD_STAMP_*) of the CPI about to be submitted with submit_map, on
 * `stream` (NULL = the pipeline's stream).  submit_map stamps at its start every one of the three not stamped since
 * the last submit, so that stages whose work ran elsewhere read 0 ms.  Nothing is enqueued when the timing stage is
 * off.  B200DD_ERR_ARG: a null handle, another slot. */
#define B200DD_STAMP_CHAIN 0     /* the CPI's first stamp: before its spectrum */
#define B200DD_STAMP_SPECTRUM 1  /* after the spectrum fold (the exchange of the parts runs on its own stream) */
#define B200DD_STAMP_CLUTTER 2   /* after the clutter filter */
B200DD_API int b200dd_pipeline_submit_map(b200dd_pipeline *h, const void *d_map, const int *d_filter_status,
                                          const void *d_spectrum_parts, uint32_t n_parts, void *stream);
B200DD_API int b200dd_pipeline_stamp(b200dd_pipeline *h, int slot, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Inter-GPU exchanges (one process per GPU, NCCL over NVLink / NVSwitch).  The reference has no
 * distributed code; these serve the two shardings of SURVEY.md s8(e): independent CPIs round-robin
 * over the GPUs (the only communication: gather of finished maps to one rank) and one large CPI split
 * over the GPUs (all-gather of the range matrix, gather of the delay-column tiles; for the clutter filter
 * an all-reduce of the partial correlations and a halo from the left neighbour).
 * NCCL is resolved with dlopen("libnccl.so.2") at the first call: libb200dd.so has no link-time dependency on it.
 * Every *_async call orders the communicator's own stream after what is enqueued so far on `after` (a CUDA
 * stream, nullable), enqueues the exchange there and returns; b200dd_comm_join makes a compute stream wait for
 * everything enqueued on the communicator so far.  All ranks must issue the same sequence of calls.
 * ------------------------------------------------------------------------------------------------ */
typedef struct b200dd_comm b200dd_comm;
#define B200DD_COMM_ID_BYTES 128

/* rank 0 creates the 128-byte id and hands it to the other ranks by any host-side means */
B200DD_API int b200dd_comm_get_unique_id(uint8_t *id128);
B200DD_API int b200dd_comm_create(int32_t rank, int32_t world, const uint8_t *id128, int32_t device, b200dd_comm **out);
B200DD_API void b200dd_comm_destroy(b200dd_comm *c);
B200DD_API int32_t b200dd_comm_rank(const b200dd_comm *c);
B200DD_API int32_t b200dd_comm_world(const b200dd_comm *c);
B200DD_API void *b200dd_comm_stream(b200dd_comm *c);

/* every rank contributes `bytes` from d_send; rank dst receives rank r's block at d_recv + r * bytes
 * (d_recv may be NULL elsewhere) */
B200DD_API int b200dd_comm_gather_async(b200dd_comm *c, const void *d_send, void *d_recv, size_t bytes, int32_t dst,
                                        void *after);
/* blocks of different sizes: rank r's send_bytes must equal bytes[r]; block r lands at d_recv + offsets[r] */
B200DD_API int b200dd_comm_gatherv_async(b200dd_comm *c, const void *d_send, size_t send_bytes, void *d_recv,
                                         const size_t *bytes, const size_t *offsets, int32_t dst, void *after);
B200DD_API int b200dd_comm_allgatherv_async(b200dd_comm *c, const void *d_send, void *d_recv, const size_t *bytes,
                                            const size_t *offsets, void *after);
/* in-place sum of `count` doubles over the ranks */
B200DD_API int b200dd_comm_allreduce_f64_async(b200dd_comm *c, void *d_buf, size_t count, void *after);
/* one send and / or one receive in one NCCL group (halo exchange): a peer of -1 (or a size of 0) skips that half;
 * the peers' calls must pair up (rank a sends to b <=> rank b receives from a, same size) */
B200DD_API int b200dd_comm_sendrecv_async(b200dd_comm *c, const void *d_send, size_t send_bytes, int32_t send_peer,
                                          void *d_recv, size_t recv_bytes, int32_t recv_peer, void *after);
/* the communicator's stream waits for everything enqueued so far on `stream` (what `after` does inside the *_async
 * calls; call it once per compute stream when an exchange depends on several of them, then pass after = NULL) */
B200DD_API int b200dd_comm_wait_stream(b200dd_comm *c, void *stream);
B200DD_API int b200dd_comm_join(b200dd_comm *c, void *stream);
B200DD_API int b200dd_comm_sync(b200dd_comm *c);

/* Measured FP64 FMA rate of the device (TFLOP/s, 2 flop per FMA): the roofline of the FP64 WienerHopf kernels,
 * which MEASURED_PEAKS.json does not carry.  Takes a few milliseconds. */
B200DD_API int b200dd_ubench_fp64_tflops(int32_t device, double *tflops);

/* Pin the CALLING host thread to the CPUs local to the device's PCIe root (sysfs local_cpulist, intersected with
 * the thread's current affinity mask); call it before allocating pinned staging buffers so that they land on the
 * GPU's NUMA node.  cpulist_out (nullable, `cap` bytes) receives the kernel's list, e.g. "0-31,64-95". */
B200DD_API int b200dd_bind_host_to_device(int32_t device, char *cpulist_out, int32_t cap);

/* Pinned host memory for staging buffers (malloc / free semantics, NULL on failure). */
B200DD_API void *b200dd_host_alloc(size_t bytes);
B200DD_API void b200dd_host_free(void *p);

#ifdef __cplusplus
}
#endif

#endif /* B200DD_H */
