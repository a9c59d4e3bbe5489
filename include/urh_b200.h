/*
 * urh_b200 — C ABI of the H100-native IQ hot path (drop-in for urh.cythonext.* on this path).
 *
 * Every entry point is `extern "C"`, takes plain pointers and sizes, and returns 0 on success or a
 * negative URH_ERR_* code (the ctypes shim maps these onto the Python exceptions the reference raises).
 * Pointers named d_* are DEVICE pointers (from urh_malloc); h_* are HOST pointers.  All work is
 * enqueued on the context's stream; functions that return a count/scalar synchronise that stream.
 *
 * Each function cites the reference interface it replaces (paths relative to the reference root).
 */
#ifndef URH_B200_H
#define URH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct urh_ctx urh_ctx;

/* error codes */
#define URH_OK 0
#define URH_ERR_CUDA (-1)        /* CUDA runtime / cuFFT / NCCL failure -> RuntimeError            */
#define URH_ERR_INVALID (-2)     /* bad argument -> ValueError                                      */
#define URH_ERR_DTYPE (-3)       /* "Unsupported dtype" (signal_functions.pyx:283,354,78)           */
#define URH_ERR_NOMEM (-4)       /* device allocation failed -> MemoryError                         */
#define URH_ERR_MODULATION (-5)  /* unknown modulation (assert at signal_functions.pyx:107,111)     */
#define URH_ERR_NO_DEVICE (-6)   /* no CUDA device: the product has no CPU fallback                 */

/* sample dtypes of the fused `iq` type (util.pxd:1-8) */
#define URH_DT_I8 0
#define URH_DT_U8 1
#define URH_DT_I16 2
#define URH_DT_U16 3
#define URH_DT_F32 4

/* modulation types (Signal.MODULATION_TYPES, Signal.py:26; Modulator.MODULATION_TYPES, Modulator.py:21) */
#define URH_MOD_ASK 0
#define URH_MOD_FSK 1
#define URH_MOD_PSK 2
#define URH_MOD_QAM 3   /* afp_demod leaves zeros for it (signal_functions.pyx:371-376) */
#define URH_MOD_GFSK 4  /* modulator only */
#define URH_MOD_OQPSK 5 /* modulator only; digitizer treats it like PSK (signal_functions.pyx:39) */

/* ---- context, memory, timing ------------------------------------------------------------------ */
int urh_device_count(void);
int urh_ctx_create(int device, urh_ctx** out);
void urh_ctx_destroy(urh_ctx* ctx);
const char* urh_last_error(urh_ctx* ctx);
int urh_sync(urh_ctx* ctx);
int urh_device_info(urh_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem, char* name, int name_cap);
int urh_malloc(urh_ctx* ctx, size_t bytes, void** d_ptr);
int urh_free(urh_ctx* ctx, void* d_ptr);
int urh_memset(urh_ctx* ctx, void* d_ptr, int value, size_t bytes);
int urh_memcpy_h2d(urh_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);   /* async on ctx stream */
int urh_memcpy_d2h(urh_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);   /* synchronises */
int urh_memcpy_d2d(urh_ctx* ctx, void* d_dst, const void* d_src, size_t bytes);
int urh_host_alloc(urh_ctx* ctx, size_t bytes, void** h_ptr);                      /* pinned */
int urh_host_free(urh_ctx* ctx, void* h_ptr);
int urh_timer_start(urh_ctx* ctx);                 /* cudaEventRecord on the ctx stream */
int urh_timer_stop(urh_ctx* ctx, float* ms);       /* records, synchronises, returns elapsed ms */
/* number of kernels this library has launched on this context since creation (bench `gpu_launches`) */
int64_t urh_launch_count(urh_ctx* ctx);

/* ---- demodulation: replaces signal_functions.afp_demod (signal_functions.pyx:333-378) ------------
 * d_iq: (n,2) C-contiguous samples of `dtype`; d_out: float32[n].  mod_type ASK/FSK computed exactly
 * as the reference (float32, glibc atan2f restated); PSK -> Costas loop (signal_functions.pyx:252-330);
 * other -> zeros.  n <= 2 -> zeros (pyx:335). */
int urh_afp_demod(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                  int mod_order, float costas_loop_bandwidth, float* d_out);

/* thresholds: replaces signal_functions.get_center_thresholds (signal_functions.pyx:380-390); host-only */
int urh_get_center_thresholds(float center, float spacing, int modulation_order, float* h_out);

/* ---- digitizer: replaces signal_functions.grab_pulse_lens (signal_functions.pyx:392-495) ----------
 * d_qad float32[n].  Result rows (state, length) int64[k][2] stay in a context-owned device buffer;
 * *k receives the row count; fetch with urh_fetch_pulses.  */
int urh_grab_pulse_lens(urh_ctx* ctx, const float* d_qad, int64_t n, float center, uint16_t tolerance,
                        int mod_type, uint32_t samples_per_symbol, uint8_t bits_per_symbol,
                        float center_spacing, int64_t* k);
/* fused a1+a3: demodulate (writes d_qad_out if non-NULL) and digitize in ONE pass over the IQ data. */
int urh_demod_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                       float center, uint16_t tolerance, uint32_t samples_per_symbol, uint8_t bits_per_symbol,
                       float center_spacing, float* d_qad_out, int64_t* k);
int urh_fetch_pulses(urh_ctx* ctx, int64_t* h_rows, int64_t k);          /* D2H of the last result   */
int urh_pulses_device_ptr(urh_ctx* ctx, const int64_t** d_rows, int64_t* k);

/* ---- auto-interpretation statistics (stats.cu) ------------------------------------------------------- */
/* replaces util.get_magnitudes (util.pyx:128-136): float64[n] */
int urh_get_magnitudes(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, double* d_out);
/* per-chunk (sum, max) of the magnitudes, chunks counted from the END of the capture as
 * AutoInterpretation.detect_noise_level does (AutoInterpretation.py:60-91); h_sum/h_max: host arrays [nchunks] */
int urh_noise_chunk_stats_iq(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int64_t chunksize, int nchunks,
                             double* h_sum, double* h_max);
int urh_noise_chunk_stats(urh_ctx* ctx, const void* d_mags, int is_f64, int64_t n, int64_t chunksize, int nchunks,
                          double* h_sum, double* h_max);
/* AutoInterpretation.detect_center (AutoInterpretation.py:226-277), sample-rate part:
 * stats  -> h_out[7] = {#samples > -4, r0, r1 (rank window after the 5 %/95 % trim and max_size), min, max, mean, var}
 * hist   -> counts of the rank-trimmed samples in the bins hmin + k*hstep, k = 0..nbins (np.histogram semantics) */
int urh_center_stats(urh_ctx* ctx, const float* d_x, int64_t n, int64_t max_size, double* h_out);
int urh_center_histogram(urh_ctx* ctx, const float* d_x, int64_t n, int64_t r0, int64_t r1, double hmin, double hstep,
                         int64_t nbins, int64_t* h_hist);
/* detect_center fused with demodulation (AutoInterpretation.py:183-240 after signal_functions.pyx:282 afp_demod):
 * urh_afp_demod_tiles writes qad AND keeps, from the one pass over the IQ samples, per-tile {count, min, max, sum, sumsq}
 * of the samples detect_center keeps; *h_kept = their number.  The caller forms the rank window [r0, r1) (5 %..95 %,
 * capped by max_size; a shard subtracts its rank offset), urh_center_window_stats returns h_out5 = {count, min, max, sum,
 * sumsq} inside it (a shard all-reduces these), and urh_center_histogram_tiles is then the only extra pass over qad.
 * halo != 0: the previous shard's last sample is stored right before d_iq (as for urh_shard_dense). */
int urh_afp_demod_tiles(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type, float* d_qad_out,
                        int halo, int64_t* h_kept);
int urh_center_window_stats(urh_ctx* ctx, const float* d_qad, int64_t n, int64_t r0, int64_t r1, double* h_out5);
/* {np.mean, np.var} of the same window as numpy computes them for a float32 array — float32 pairwise sums replayed bit for bit
 * (AutoInterpretation.py:240: the histogram's bin width); urh_center_stats uses it unless URH_B200_CENTER_DOUBLE is set. */
int urh_center_window_var(urh_ctx* ctx, const float* d_qad, int64_t n, int64_t r0, int64_t r1, double* h_out2);
int urh_center_histogram_tiles(urh_ctx* ctx, const float* d_qad, int64_t n, int64_t r0, int64_t r1, double hmin, double hstep,
                               int64_t nbins, int64_t* h_hist);
/* replaces auto_interpretation.segment_messages_from_magnitudes (auto_interpretation.pyx:55-111) */
int urh_segment_messages(urh_ctx* ctx, const void* d_mags, int is_f64, int64_t n, float noise_threshold,
                         int64_t* h_segments, int64_t cap, int64_t* k);
/* Sharded captures: urh_segment_shard_pass = the dense pass of one shard's magnitudes (then urh_shard_candidates with the run
 * carry of the preceding shards and urh_fetch_candidates); urh_segments_from_runs = the state machine of
 * auto_interpretation.pyx:69-111 over the concatenated run table of all shards (pure host code). */
int urh_segment_shard_pass(urh_ctx* ctx, const void* d_mags, int is_f64, int64_t n, float noise_threshold, int64_t* h_summary);
int urh_segments_from_runs(const int64_t* h_pos, const int16_t* h_cls, int64_t count, int first_above, int last_cls,
                           int64_t last_len, int64_t n, int64_t* h_segments, int64_t cap, int64_t* k);
int urh_fetch_candidates(urh_ctx* ctx, int64_t* h_pos, int16_t* h_cls, int64_t count);
/* replaces auto_interpretation.get_plateau_lengths (auto_interpretation.pyx:179-208) */
int urh_plateau_lengths(urh_ctx* ctx, const float* d_rect, int64_t n, float center, int percentage, uint64_t* h_out,
                        int64_t cap, int64_t* k);
/* replaces auto_interpretation.median_filter (auto_interpretation.pyx:211-240); k <= 64 */
int urh_median_filter(urh_ctx* ctx, const double* d_x, int64_t n, unsigned int k, float* d_out);
/* replaces util.arr2decibel (util.pyx:38-48): count complex64 values -> float32 dB */
int urh_arr2decibel(urh_ctx* ctx, const float* d_complex, int64_t count, float* d_out);

/* ---- modulator (modulate.cu): replaces signal_functions.modulate_c / __modulate (signal_functions.pyx:56-177),
 * get_gauss_filtered_freqs_phases (:196-226) for a BATCH of messages sharing one parameter set.
 * d_bits: concatenated uint8 bits (OQPSK: already shuffled by get_oqpsk_bits and cut to the original length);
 * h_bit_off[nmsg+1] bit offsets; h_out_off[nmsg+1] output sample offsets (symbols*sps + pause per message);
 * d_out: (h_out_off[nmsg], 2) of out_dtype (URH_DT_I8 / I16 / F32), zero-filled by the call. */
int urh_modulate_batch(urh_ctx* ctx, const uint8_t* d_bits, const int64_t* h_bit_off, const int64_t* h_out_off, int nmsg,
                       uint32_t samples_per_symbol, int mod_type, const float* h_params, int nparams, int bits_per_symbol,
                       float carrier_amplitude, float carrier_frequency, float carrier_phase, float sample_rate,
                       uint32_t start, int out_dtype, const float* h_gauss_fir, int gauss_len, void* d_out);
/* diagnostics: steps of the GFSK phase recurrence taken through an integer prefix sum / one by one since the last call */
int urh_modulate_stats(urh_ctx* ctx, int64_t* h_out2);

/* ---- filters (filter.cu) ----------------------------------------------------------------------------------
 * urh_fir_filter replaces signal_functions.fir_filter (signal_functions.pyx:513-525), exact accumulation order;
 * urh_convolve_c128: y[k] = full_convolution(x, taps)[k + offset], complex128 taps, double accumulation
 *   (Filter.apply_bandpass_filter, Filter.py:84-101); urh_dc_correction: x - mean(x, axis=0) (Filter.py:32-33). */
int urh_fir_filter(urh_ctx* ctx, const float* d_x, int64_t n, const float* d_taps, int m, float* d_y);
int urh_convolve_c128(urh_ctx* ctx, const float* d_x, int64_t n, const double* d_taps, int m, int64_t offset,
                      int64_t out_len, float* d_y);
int urh_dc_correction(urh_ctx* ctx, const float* d_iq, int64_t n, float* d_out, int exact_order);
/* the same for an integer capture: numpy promotes to float64 (exact integer column sums), d_out = double[n][2] */
int urh_dc_correction_int(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, double* d_out);
/* The filters of one shard of a capture cut by contiguous sample range (urh_b200/dist.py).
 * urh_fir_filter_shard: fir_filter (signal_functions.pyx:513-525, Filter.apply_fir_filter Filter.py:35-46) of a shard; has_history != 0
 *   means d_x[-(m-1) .. -1] hold the previous shard's last m-1 samples and y equals urh_fir_filter of the whole capture from d_x[0] on.
 * urh_dc_column_sums / urh_dc_subtract: Filter.dc_correction (Filter.py:31-33) split into per-shard column sums (h_sums: two host
 *   doubles, undivided) and the subtraction of the global mean.  exact_order != 0: numpy's serial float32 chain continued from the two
 *   accumulators h_carry (NULL: 0); otherwise the double sums of urh_dc_correction's reduction.
 * urh_dc_int_column_sums / urh_dc_int_subtract: the same for an integer capture: exact int64 sums, d_out = double[n][2] = x - mean. */
int urh_fir_filter_shard(urh_ctx* ctx, const float* d_x, int64_t n, int has_history, const float* d_taps, int m, float* d_y);
int urh_dc_column_sums(urh_ctx* ctx, const float* d_iq, int64_t n, int exact_order, const float* h_carry, double* h_sums);
int urh_dc_subtract(urh_ctx* ctx, const float* d_iq, int64_t n, float mean_i, float mean_q, float* d_out);
int urh_dc_int_column_sums(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int64_t* h_sums);
int urh_dc_int_subtract(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, double mean_i, double mean_q, double* d_out);

/* ---- spectrogram (spectrogram.cu; cuFFT for the FFT only) -------------------------------------------------
 * urh_stft replaces Spectrogram.stft (Spectrogram.py:94-116): complex128 [num_frames][window_size] = fft(frames*window)/W;
 * urh_spectrogram_db replaces __calculate_spectrogram (:156-162): float32 fliplr(10*log10(|fftshift(stft)|^2)). */
int urh_stft(urh_ctx* ctx, const float* d_x, int64_t n, int window_size, int hop, const double* d_window, int64_t num_frames,
             double* d_out);
int urh_spectrogram_db(urh_ctx* ctx, const float* d_x, int64_t n, int window_size, int hop, const double* d_window,
                       int64_t num_frames, float* d_out);
/* Spectrogram.apply_bgra_lookup (Spectrogram.py:192-206): d_out[cols][rows][4] = colormap[clip(int((entries - 1) * ((data.T - min) /
 * (max - min))))], colormap = entries x 4 bytes (blue, green, red, alpha); normalize = 0: the data are indices already. */
int urh_bgra_lookup(urh_ctx* ctx, const float* d_data, int64_t rows, int64_t cols, const uint8_t* d_colormap, int entries,
                    float data_min, float data_max, int normalize, uint8_t* d_out);
/* Spectrogram.create_spectrogram_image / create_image_segments (Spectrogram.py:164-190) in one launch: the BGRA image
 * apply_bgra_lookup(dB map) of every segment s = d_x[h_seg_start[s] : h_seg_start[s] + h_seg_len[s]] (complex64), each with its own
 * frame count max(1, (len - W) // hop + 1), zero-padded below W samples, written back to back into d_out: transpose = 0 gives
 * [W][frames][4] per segment (Spectrogram.create_image(dB)), transpose = 1 gives [frames][W][4] (create_image(flipud(dB.T))).
 * Bit-identical to urh_spectrogram_db followed by urh_bgra_lookup.  Power-of-two windows 128 .. 4096 with colormaps of up to
 * 65536 entries take the fused kernel; anything else composes those two stages on the device. */
int urh_spectrogram_bgra(urh_ctx* ctx, const float* d_x, int64_t n, int window_size, int hop, const double* d_window,
                         const int64_t* h_seg_start, const int64_t* h_seg_len, int nseg, const uint8_t* d_colormap, int entries,
                         float data_min, float data_max, int transpose, uint8_t* d_out);
/* d_out[i] = d_x[start + i * step], i < count (complex64 samples; a Python slice of a capture of n samples, step may be negative) */
int urh_gather_samples(urh_ctx* ctx, const float* d_x, int64_t n, int64_t start, int64_t step, int64_t count, float* d_out);
/* Spectrogram.export_to_fta (Spectrogram.py:118-154): rows [row0, row0 + nrows) of the record array [W][frames][reps], packed
 * records {f8 f, u4 t, f4 a} (include_amplitude, reps = 3) or {f8 f, u4 t} (reps = 2): f = d_freqs[i], t = int(j * time_width),
 * a = the fftshifted dB map [j][i] (d_db = urh_spectrogram_db's fliplr'ed map).  The caller checks that every t fits a uint32.
 * h_out != NULL: the band is also copied to that (pinned) host buffer, asynchronously; synchronise before reading it. */
int urh_fta_records(urh_ctx* ctx, const float* d_db, int64_t frames, int window_size, int64_t row0, int64_t nrows,
                    const double* d_freqs, double time_width, int include_amplitude, uint8_t* d_out, void* h_out);

/* ---- signal views (path_creator.pyx; view.cu) ---------------------------------------------------------------------------------
 * The source is sample d_src[i * stride], i < n, of dtype URH_DT_*: stride 1 for qad or a 1-D capture, 2 for one column of an
 * (n, 2) capture (d_src then points at that column's first element).  Both need 0 <= start <= end <= n.
 *
 * path_creator.create_path (path_creator.pyx:19-69), spp = samples per pixel > 1: d_values[2k], d_values[2k + 1] = (min, max) of
 * pixel k = samples [start + k * spp, min(start + (k + 1) * spp, end)), k < ceil((end - start) / spp), in the sample dtype, as the
 * reference's walk from the pixel's first sample finds them (:50-59): strict < / > only, so the first of equal values wins, later
 * NaNs are ignored and a NaN first sample is both outputs. */
int urh_path_minmax(urh_ctx* ctx, const void* d_src, int dtype, int64_t stride, int64_t n, int64_t start, int64_t end, int64_t spp,
                    void* d_values);
/* The sub-path loop of create_path (:71-82) and array_to_QPath (:88-120) for every sub-path of one call, in one launch.
 * h_bounds[2s], h_bounds[2s + 1] = the slice [lo, hi) of sub-path s into x / values, both within [0, L] (L = 2 * pixels when
 * spp > 1, else end - start).  Sub-path s is written at d_out + h_offsets[s]: the big-endian stream {i4 n, n x {i4 1, f8 x, f8 y},
 * i4 0, i4 0} with x = x0 + (i >> 1) * spp (or x0 + i when spp <= 1; x0 = start unless d_src holds only the visible range) and y = float64(-value) negated in the sample dtype;
 * y comes from d_values when spp > 1 and straight from the samples otherwise (d_values may then be NULL).  An empty slice writes
 * nothing.  h_offsets[count] = total bytes; with d_out = NULL only h_offsets is filled (no launch). */
int urh_qpath_streams(urh_ctx* ctx, const void* d_src, int dtype, int64_t stride, int64_t n, int64_t start, int64_t end, int64_t spp,
                      int64_t x0, const void* d_values, const int64_t* h_bounds, int count, uint8_t* d_out, int64_t* h_offsets);

/* ---- sharded captures: one contiguous sample range per GPU (digitize.cu, nccl.cu; SURVEY 8e) ----------
 * urh_shard_dense      every rank: demodulate + classify its shard (d_iq[-1] = halo sample when has_halo);
 *                      h_summary = {last_cls, last_len, whole, init_cls}
 * urh_shard_candidates every rank, after exchanging the summaries: candidate table with GLOBAL positions
 * urh_pulses_from_table the gathering rank: concatenated tables -> (state, length) rows of the whole capture */
int urh_shard_dense(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int has_halo, float noise_mag, int mod_type,
                    float center, uint16_t tolerance, uint8_t bits_per_symbol, float center_spacing, float* d_qad_out,
                    int64_t* h_summary);
/* the same step for a shard that is already demodulated (digitizing once a capture-wide center is known) */
int urh_shard_dense_qad(urh_ctx* ctx, const float* d_qad, int64_t n, int mod_type, float center, uint16_t tolerance,
                        uint8_t bits_per_symbol, float center_spacing, int64_t* h_summary);
int urh_shard_candidates(urh_ctx* ctx, int carry_valid, int carry_cls, int64_t carry_len, int64_t global_offset,
                         int64_t* count, const int64_t** d_pos, const int16_t** d_cls, int* last_cand_cls);
/* distributed finish (no gather): every rank keeps its own rows; see urh_b200/dist.py for the two scalars exchanged */
int urh_shard_fire(urh_ctx* ctx, int prev_cls, int64_t* fired, int64_t* last_fired_pos);
int urh_shard_rows(urh_ctx* ctx, int64_t n_total, uint16_t tolerance, int mod_type, uint32_t samples_per_symbol,
                   int64_t prev_fired_pos, int emit_tail, int64_t* k);
/* One-call variants: every stage is enqueued on the context stream, the host synchronises once at the end.
 * urh_demod_center_digitize: afp_demod (ASK/FSK) + AutoInterpretation.detect_center (AutoInterpretation.py:226-277, capture-wide)
 *   + grab_pulse_lens (signal_functions.pyx:392-495, binary symbols) = BASELINE configs[1].  *center_state: 0 no center (None),
 *   1 *center valid and the pulse table is ready (urh_fetch_pulses), 2 the device could not decide (a tie between histogram
 *   peaks whose order np.argsort defines, or > 6000 bins): d_qad_out is valid, finish with the stepwise entry points.
 * urh_shard_*: this rank's shard of a capture spread over the ranks of the context's NCCL communicator (SURVEY 8e); the
 *   exchanges (run carry, candidate class, firing position; kept counts, window partials, histogram) are NCCL calls on the
 *   stream.  Every rank ends with the rows of its own shard. */
int urh_demod_center_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                              uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, float* d_qad_out,
                              double* center, int* center_state, int64_t* k);
/* the same step fed from (pinned) HOST memory: chunked upload on the copy stream overlapped with the demodulation of the chunks
 * that have landed (IQArray.from_file / Signal capture formats into device memory, SURVEY 8f-2); chunk_samples <= 0: 2^24 */
int urh_demod_center_digitize_host(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                                   uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, int64_t chunk_samples,
                                   void* d_iq_scratch, float* d_qad_out, double* center, int* center_state, int64_t* k);
int urh_shard_demod_center_digitize_host(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, int has_halo, float noise_mag,
                                         int mod_type, uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size,
                                         int64_t chunk_samples, void* d_iq_scratch, float* d_qad_out, int64_t global_offset,
                                         int64_t n_total, double* center, int* center_state, int64_t* k);
/* ---- streaming: host captures of any size through a ring of `ring` (2..8) device slots of chunk_samples each (digitize.cu,
 * DESIGN.md §4.11).  chunk_samples <= 0: 2^24; it is rounded down to a multiple of 2048 (at least 2048).  Host buffers may be pinned
 * (urh_host_alloc: copies overlap the kernels) or pageable, e.g. a memory-mapped file (correct, but each copy then blocks the host).
 * Results are bit-identical to the resident entry points named below.  ASK / FSK only; PSK raises URH_ERR_INVALID (PSK has entry
 * points of its own, below).
 * urh_afp_demod_stream: afp_demod (signal_functions.pyx:333-378) from host IQ into host qad h_qad[n].
 * urh_grab_pulse_lens_stream: grab_pulse_lens (signal_functions.pyx:392-495) of qad[n], any bits_per_symbol; qad_on_device != 0: qad
 *   is a device buffer (only the digitizer's work arrays are chunked).  Rows as urh_grab_pulse_lens (urh_fetch_pulses).
 * urh_demod_digitize_stream: afp_demod + grab_pulse_lens for a known center in one pass over the IQ (urh_demod_digitize); h_qad_out
 *   (may be NULL) receives qad.
 * urh_demod_center_digitize_stream: urh_demod_center_digitize (afp_demod + AutoInterpretation.detect_center, AutoInterpretation.py:
 *   226-277, + grab_pulse_lens) with the IQ streamed and qad resident in d_qad_out[n]; h_qad_out (may be NULL) mirrors it to the host.
 *   center_state as urh_demod_center_digitize; on state 2 the tables of urh_center_window_stats / urh_center_histogram_tiles are
 *   left for d_qad_out, and *kept = the number of kept samples (the input of the stepwise detect_center).
 * urh_afp_demod_psk_stream: urh_afp_demod(..., URH_MOD_PSK, mod_order, costas_loop_bandwidth, ...) from host IQ into host qad h_qad[n].
 *   The Costas loop runs chunk by chunk, each chunk continued from the loop state the preceding one left on the device.
 * urh_demod_digitize_psk_stream: urh_demod_digitize for PSK (the Costas loop of order 1 << bits_per_symbol at loop bandwidth 0.1, then
 *   grab_pulse_lens) with the Costas loop streamed as above and the digitizer run on each chunk's qad; h_qad_out (may be NULL)
 *   receives qad.  After either PSK call urh_costas_stats / urh_costas_stitch_stats hold sums over its chunks.
 * urh_stream_footprint: device bytes a call needs, callable without a device.  entry = URH_STREAM_ENTRY_* | URH_STREAM_* flags;
 *   URH_STREAM_RESIDENT gives the resident entry's bytes for the same capture instead.  PSK (AFP_DEMOD and DEMOD_DIGITIZE entries):
 *   URH_STREAM_PSK for a Costas loop of order 2 (also a bound for orders 1 and 3, which run the serial kernel), with
 *   URH_STREAM_PSK4 for order 4 or more.  rows: the pulse-table rows to budget for
 *   (-1: the bound n / (tolerance + 1) + 3 that no capture exceeds; -2: the n / 64 + 1024 rows the resident call reserves up front).
 * urh_stream_schedule: the order in which a call issues its copies and chunk computations, 6 int64 per op {kind (0 upload into
 *   the slot, 1 compute, 2 download from the slot), chunk, slot, first sample, end sample, 1 if the upload carries the halo sample
 *   first - 1}; host only.  flags: URH_STREAM_UPLOAD / DOWNLOAD / HALO.
 * urh_stream_stats: {lowest free device memory seen inside the last streamed call (after each chunk and each chunk's finish and
 *   while the pulse table grows; sampled only with urh_set_profiling on, else -1), chunks of its ring pass, the most bytes of
 *   scratch-arena requests live at once during it}.
 * urh_mem_get_info: cudaMemGetInfo on the context's device. */
#define URH_STREAM_ENTRY_AFP_DEMOD 0
#define URH_STREAM_ENTRY_GRAB_PULSE_LENS 1
#define URH_STREAM_ENTRY_DEMOD_DIGITIZE 2
#define URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE 3
#define URH_STREAM_QAD_OUT 0x10       /* demod_digitize: qad also goes to the host */
#define URH_STREAM_RESIDENT 0x20      /* footprint of the resident entry point */
#define URH_STREAM_QAD_ON_DEVICE 0x40 /* grab_pulse_lens: qad is already on the device */
#define URH_STREAM_PSK 0x80           /* the PSK entry points (Costas loop of order 2) */
#define URH_STREAM_PSK4 0x100         /* with URH_STREAM_PSK: Costas loop of order 4 */
#define URH_STREAM_UPLOAD 1
#define URH_STREAM_DOWNLOAD 2
#define URH_STREAM_HALO 4
int urh_afp_demod_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type, int64_t chunk_samples,
                         int ring, float* h_qad);
int urh_grab_pulse_lens_stream(urh_ctx* ctx, const float* qad, int qad_on_device, int64_t n, float center, uint16_t tolerance,
                               int mod_type, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                               int64_t chunk_samples, int ring, int64_t* k);
int urh_demod_digitize_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type, float center,
                              uint16_t tolerance, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                              int64_t chunk_samples, int ring, float* h_qad_out, int64_t* k);
int urh_demod_center_digitize_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                                     uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, int64_t chunk_samples, int ring,
                                     float* d_qad_out, float* h_qad_out, double* center, int* center_state, int64_t* kept, int64_t* k);
int urh_afp_demod_psk_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_order,
                             float costas_loop_bandwidth, int64_t chunk_samples, int ring, float* h_qad);
int urh_demod_digitize_psk_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, float center, uint16_t tolerance,
                                  uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing, int64_t chunk_samples,
                                  int ring, float* h_qad_out, int64_t* k);
int urh_stream_footprint(int64_t n, int dtype, int tolerance, int64_t chunk_samples, int ring, int entry, int64_t rows, int64_t* bytes);
int urh_stream_schedule(int64_t n, int64_t chunk_samples, int ring, int flags, int64_t* h_ops, int64_t cap, int64_t* count);
int urh_stream_stats(urh_ctx* ctx, int64_t* h_out3);
int urh_mem_get_info(urh_ctx* ctx, size_t* free_bytes, size_t* total_bytes);
int urh_shard_demod_center_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int has_halo, float noise_mag,
                                    int mod_type, uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size,
                                    float* d_qad_out, int64_t global_offset, int64_t n_total, double* center,
                                    int* center_state, int64_t* k);
int urh_shard_digitize(urh_ctx* ctx, const void* d_iq, int dtype, const float* d_qad_in, int64_t n, int has_halo,
                       float noise_mag, int mod_type, float center, uint16_t tolerance, uint32_t samples_per_symbol,
                       uint8_t bits_per_symbol, float center_spacing, float* d_qad_out, int64_t global_offset,
                       int64_t n_total, int64_t* k);
int urh_pulses_from_table(urh_ctx* ctx, const int64_t* d_pos, const int16_t* d_cls, int64_t count, int64_t n_total,
                          uint16_t tolerance, int mod_type, uint32_t samples_per_symbol, int init_cls, int64_t* k);
/* PSK (Costas loop) over shards: speculate concurrently on every rank, then hand the loop state from rank to rank */
int urh_costas_halo_samples(void);
int urh_costas_shard_speculate(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int first_shard, float noise_mag,
                               int loop_order, float bandwidth, float* d_out);
int urh_costas_shard_resolve(urh_ctx* ctx, const float* h_state_in, float* h_state_out);
/* Sharded PSK without the rank-to-rank hand-over: after urh_costas_shard_speculate every later shard hops over its
 * super-chunks under each hypothesis "the shard starts in candidate h's start state" (what a locked loop of the preceding shard
 * ends in, bit for bit); h_out[h] = {start.freq, start.phase, end.freq, end.phase}, *count hypotheses (1 on the first shard).
 * The ranks exchange these few floats, each picks the hypothesis whose start state equals the preceding shard's end state
 * and calls urh_costas_shard_adopt; without a match the serial urh_costas_shard_resolve remains (exact either way). */
int urh_costas_shard_hypotheses(urh_ctx* ctx, float* h_out, int* count);
int urh_costas_shard_adopt(urh_ctx* ctx, int h, float* h_state_out);
/* Signal.estimate_frequency (Signal.py:578-601): arg-max bin of fft(x[0:P]), P = 2^floor(log2 n) (complex64 on the device) */
int urh_fft_argmax(urh_ctx* ctx, const float* d_x, int64_t n, int64_t* h_index, int64_t* h_P);
/* replaces the arithmetic of IQArray.convert_to (IQArray.py:127-200): capture formats cs8/cu8/cs16/cu16/float32 into each
 * other (numpy's integer wrap-around, C truncation for float -> int).  count = number of elements (2 per sample). */
int urh_convert_iq(urh_ctx* ctx, const void* d_in, int in_dtype, void* d_out, int out_dtype, int64_t count);
/* the sample-rate part of AutoInterpretation.detect_modulation (AutoInterpretation.py:151-208) for one message
 * (d_data = complex64[n] on the device): zero removal, normalisation, the two Haar wavelet transforms (cuFFT for the FFTs),
 * variances before/after the median filter and the spectrum features of the FSK test.  h_feat[8] = {n_nonzero, P, L, var_mag,
 * var_norm_mag, var_filtered_mag, var_filtered_norm_mag, |max|}; h_spec[23] = {arg-max bin, value, best bin >= 10 away,
 * value, the 19 values around the arg-max}.  urh_cwt_haar replaces Wavelet.cwt_haar (Wavelet.py:15-43). */
int urh_modulation_features(urh_ctx* ctx, const float* d_data, int64_t n, int wavelet_scale, int median_k, double* h_feat,
                            double* h_spec);
int urh_cwt_haar(urh_ctx* ctx, const void* d_x, int is_c128, int64_t n, int scale, double* d_out, int64_t* out_len);
/* replaces ProtocolAnalyzer._ppseq_to_bits (ProtocolAnalyzer.py:323-414): pulse table -> bits / pauses / bit_sample_pos.
 * d_rows = int64[k,2] on the device, NULL = the table the last digitizer call left in the context.  Results stay in the
 * context until the next call.  Message m = bits[off[m]:off[m+1]]; its sample positions are pos[off[m]+2m : off[m+1]+2m+2]
 * (one entry fewer for a last message that no pause row closes). */
int urh_ppseq_to_bits(urh_ctx* ctx, const int64_t* d_rows, int64_t k, uint32_t samples_per_symbol, uint8_t bits_per_symbol,
                      int pause_threshold, int write_pos, int64_t* n_msgs, int64_t* n_bits, int64_t* n_pos);
int urh_fetch_bits(urh_ctx* ctx, uint8_t* h_bits, int64_t* h_msg_off, int64_t* h_pauses, int64_t* h_pos);
const uint8_t* urh_bits_device_ptr(urh_ctx* ctx);
/* NCCL (dlopen'ed libnccl.so.2): id from rank 0 is distributed by the launcher plumbing */
int urh_nccl_unique_id(char* out128);
int urh_nccl_init(urh_ctx* ctx, const char* id128, int rank, int world);
int urh_nccl_destroy(urh_ctx* ctx);
int urh_nccl_allreduce_f64(urh_ctx* ctx, double* d_buf, int64_t count, int op);   /* op: 0 sum, 1 max, 2 min */
int urh_nccl_allreduce_i64(urh_ctx* ctx, int64_t* d_buf, int64_t count, int op);
int urh_nccl_allgather(urh_ctx* ctx, const void* d_send, void* d_recv, size_t bytes_per_rank);
int urh_nccl_gatherv(urh_ctx* ctx, const void* d_send, void* d_recv, const int64_t* h_bytes, int root);
int urh_nccl_sendrecv(urh_ctx* ctx, const void* d_send, size_t send_bytes, int send_peer, void* d_recv, size_t recv_bytes,
                      int recv_peer);
int urh_nccl_allgather_host(urh_ctx* ctx, const void* h_send, void* h_recv, size_t bytes_per_rank);
int urh_nccl_allreduce_host_i64(urh_ctx* ctx, int64_t* h_buf, int64_t count, int op);
/* the same few-bytes all-gather over NVLink peer memory, one small kernel per rank (p2p.cu): every rank creates a mailbox and
 * hands its 64-byte IPC handle to the launcher plumbing; urh_p2p_open maps the peers' mailboxes (world <= 8, one node). */
int urh_p2p_create(urh_ctx* ctx, char* out_handle64);
int urh_p2p_open(urh_ctx* ctx, const char* handles, int rank, int world);
int urh_p2p_close(urh_ctx* ctx);
int urh_p2p_allgather_host(urh_ctx* ctx, const void* h_send, void* h_recv, size_t bytes_per_rank);
/* The same exchange between DEVICE buffers, enqueued on the context stream with no host synchronisation (what the sharded chains
 * urh_shard_* use between their kernels when the mailboxes are open; NCCL otherwise): all-gather of 8..240 bytes per rank (a multiple
 * of 8); sum over ranks of min(*d_count, max_words) uint64 words (max_words <= 6000, d_out must not alias d_in, d_count a device
 * pointer or NULL).  A peer that does not show up within ~5 s raises a flag instead of hanging the GPU: urh_p2p_check, called after
 * the next synchronisation, returns URH_ERR_CUDA and closes the mailboxes. */
int urh_p2p_allgather_dev(urh_ctx* ctx, const void* d_send, void* d_recv, size_t bytes_per_rank);
int urh_p2p_allreduce_u64_dev(urh_ctx* ctx, const void* d_in, void* d_out, const int64_t* d_count, int max_words);
int urh_p2p_check(urh_ctx* ctx);

/* ---- measurement utilities (not part of the reference's API surface) -------------------------------- */
/* CUDA-event timing of the dominant (dense, sample-rate) kernel of the last demod/digitize call */
int urh_set_profiling(urh_ctx* ctx, int enabled);
/* urh_set_profiling(ctx, 2) also records a stream timeline of the sharded one-call step: CUDA events at the step's start, on
 * either side of every inter-GPU exchange and after the rows are written.  urh_timeline_fetch (after the step's result has been
 * read) returns the milliseconds from the first mark to each mark and the '\n'-separated names; *count = number of marks (<= 32). */
int urh_timeline_fetch(urh_ctx* ctx, float* h_ms, char* h_names, int names_cap, int* count);
int urh_last_dense_ms(urh_ctx* ctx, float* ms);
/* speculative Costas loop diagnostics of the last PSK demodulation: {chunks matched in O(1), chunks walked, samples stepped serially}
 * (after a streamed PSK call: sums over its ring chunks) */
int urh_costas_stats(urh_ctx* ctx, int64_t* h_out3);
/* certificate of the last urh_demod_center_digitize(_host) call: {1 if the fine histogram of the demodulation pass decided the
 * center (no histogram pass over qad) else 0, buckets of that histogram (0: not collected: sharded capture or
 * $URH_B200_CENTER_NO_CERTIFY), U - L summed over the two deciding bins}.  See DESIGN.md §4.4.1. */
int urh_center_certify_stats(urh_ctx* ctx, int64_t* h_out3);
/* speculative digitizing of the last urh_demod_center_digitize call (resident float32 FSK on one GPU): {tiles the demodulation
 * pass digitized at its threshold guess, of those the tiles the qad digitizer did not read again (their margin proved the classes
 * at the detected center, or the tile is silent), tiles it digitized again from qad}.  All zero when nothing was speculated:
 * another dtype, modulation or entry point, or $URH_B200_NO_SPECULATE.  See DESIGN.md §4.4.1. */
int urh_speculate_stats(urh_ctx* ctx, int64_t* h_out3);
int64_t urh_costas_last_redone(urh_ctx* ctx);
/* how the stitch pass of the last PSK demodulation resolved its super-chunks: {adopted from family A, adopted from family B,
 * chained by the stitch warp itself, segments per chunk}; super-chunk 0 of an unsharded capture is not counted.  The serial
 * kernel (captures shorter than 8192 samples) zeroes these and urh_costas_stats and reports segs = 0.  After a streamed PSK call
 * (urh_*_psk_stream) the counters are sums over its ring chunks (each ring chunk's super-chunk 0 not counted; chunks that ran the
 * serial kernel add nothing) and segs is the layout of the first ring chunk that took the speculative path (0: none did).
 * $URH_B200_COSTAS_SEGS = 2, 4, 8 or 16 forces the speculative path's chunk layout (the result does not depend on it). */
int urh_costas_stitch_stats(urh_ctx* ctx, int64_t* h_out4);
/* paired (float2) division used by the FSK fast path vs __fdiv_rn on `count` random operand pairs */
int urh_selftest_packed_div(urh_ctx* ctx, uint64_t seed, int64_t count, int64_t* mismatches, int64_t* tested);
/* synthetic phase-continuous 2-FSK bursts + AWGN + noise-only gaps generated in HBM (SURVEY 8d recipe) */
int urh_synth_fsk(urh_ctx* ctx, float* d_iq, int64_t n, int64_t global_offset, int sps, const int8_t* d_sym_bit,
                  const int32_t* d_sym_sum, double dev_ratio, float amplitude, float sigma, uint64_t seed,
                  int64_t period, int64_t burst, int64_t big_gap_start, int64_t big_gap_end, int64_t tail_start);
int urh_synth_psk(urh_ctx* ctx, float* d_iq, int64_t n, int64_t global_offset, int sps, int order, double carrier_ratio,
                  float amplitude, float sigma, uint64_t seed, int64_t period, int64_t burst, int64_t tail_start);

#ifdef __cplusplus
}
#endif
#endif /* URH_B200_H */
