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
/* speculative Costas loop diagnostics of the last PSK demodulation: {chunks matched in O(1), chunks walked, samples stepped serially} */
int urh_costas_stats(urh_ctx* ctx, int64_t* h_out3);
int64_t urh_costas_last_redone(urh_ctx* ctx);
/* how the stitch pass of the last PSK demodulation resolved its super-chunks: {adopted from family A, adopted from family B,
 * chained by the stitch warp itself, segments per chunk}; super-chunk 0 of an unsharded capture is not counted.  The serial
 * kernel (captures shorter than 8192 samples) zeroes these and urh_costas_stats and reports segs = 0.
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
