/*
 * flac_oracle.h -- TEST INFRASTRUCTURE ONLY. Never imported/linked by the product path
 * (flac_b200/); only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg use it.
 *
 * A plain-C, single-threaded restatement of the reference libFLAC (xiph/flac 1.5.0,
 * /root/reference) per-frame encode pipeline and frame decoder. Every function in
 * flac_oracle.c cites the reference file:line it follows.
 *
 * Floating point semantics = SOURCE ORDER (what the reference computes when its sources
 * are compiled without -fassociative-math: oracle/_ref/libFLAC_ref_strict.so). The
 * shipped-flags build (oracle/_ref/libFLAC_ref.so) lets GCC reassociate the
 * autocorrelation/Levinson sums; tests report parity against both (SURVEY.md §0.3).
 *
 * Parity status: PINNED -- tests/test_oracle_vs_reference.py compares every frame this
 * oracle emits with the frames of the compiled reference on all input families.
 */
#ifndef FLAC_ORACLE_H
#define FLAC_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FO_MAX_CHANNELS 8
#define FO_MAX_LPC_ORDER 32
#define FO_MAX_APODIZATIONS 32
#define FO_MAX_PARTITIONS 256 /* partition order <= 8 */

/* FLAC__ApodizationFunction (src/libFLAC/include/protected/stream_encoder.h:45-65), oracle numbering */
enum {
	FO_APOD_TUKEY = 0, FO_APOD_SUBDIVIDE_TUKEY = 1, FO_APOD_BARTLETT = 2, FO_APOD_BARTLETT_HANN = 3, FO_APOD_BLACKMAN = 4,
	FO_APOD_BLACKMAN_HARRIS = 5, FO_APOD_CONNES = 6, FO_APOD_FLATTOP = 7, FO_APOD_GAUSS = 8, FO_APOD_HAMMING = 9, FO_APOD_HANN = 10,
	FO_APOD_KAISER_BESSEL = 11, FO_APOD_NUTTALL = 12, FO_APOD_RECTANGLE = 13, FO_APOD_TRIANGLE = 14, FO_APOD_PARTIAL_TUKEY = 15,
	FO_APOD_PUNCHOUT_TUKEY = 16, FO_APOD_WELCH = 17
};

typedef struct {
	int32_t type;   /* FO_APOD_* */
	float p;        /* tukey p (for subdivide: already divided by parts); gauss stddev */
	int32_t parts;  /* subdivide_tukey parts */
	float start, end; /* partial_/punchout_tukey extents (fractions of the block) */
} fo_apodization;

typedef struct {
	uint32_t channels, bits_per_sample, sample_rate, blocksize;
	int32_t do_mid_side, loose_mid_side;
	uint32_t max_lpc_order;
	uint32_t qlp_coeff_precision; /* 0 = choose like the reference */
	int32_t do_qlp_coeff_prec_search;
	int32_t do_exhaustive_model_search;
	uint32_t min_residual_partition_order, max_residual_partition_order;
	uint32_t num_apodizations;
	fo_apodization apodizations[FO_MAX_APODIZATIONS];
	int32_t disable_constant_subframes, disable_fixed_subframes, disable_verbatim_subframes;
	int32_t limit_min_bitrate;
	/* 0: the reference's C routines (default; what the CUDA engine follows). 1: restate the x86 AVX2 dispatch of the fixed-order
	 * guess, which leaves the last (blocksize - 4) % 4 samples out of its error sums (fixed_intrin_avx2.c:138) -- only a short last
	 * block can tell the difference. */
	int32_t x86_avx2_fixed_guess;
} fo_config;

/* What the search decided for one subframe (debug/stage-level comparison with the CUDA path). */
typedef struct {
	int32_t type;            /* 0 constant, 1 verbatim, 2 fixed, 3 lpc */
	int32_t order;
	int32_t wasted_bits;
	int32_t subframe_bps;
	int32_t qlp_precision, qlp_shift;
	int32_t qlp_negative_shift; /* lpc: quantised through the divide branch (computed shift < 0, coded as 0) */
	int32_t qlp_coeff[FO_MAX_LPC_ORDER];
	int32_t rice_method;     /* 0 RICE, 1 RICE2 */
	int32_t partition_order;
	int32_t rice_params[FO_MAX_PARTITIONS];
	uint32_t estimate_bits;
} fo_subframe_plan;

typedef struct {
	int32_t channel_assignment;  /* 0 independent, 1 left/side, 2 right/side, 3 mid/side */
	fo_subframe_plan sub[FO_MAX_CHANNELS];
	/* all four candidates of a stereo frame: L, R, M, S (valid when mid-side evaluated) */
	fo_subframe_plan cand[4];
	uint32_t cand_valid[4];
} fo_frame_plan;

typedef struct fo_encoder fo_encoder;

/* Fill cfg with the reference's preset `level` (0..8) (stream_encoder.c:117-140, 1873-1904). */
void fo_config_preset(fo_config *cfg, uint32_t channels, uint32_t bps, uint32_t sample_rate, uint32_t level, uint32_t blocksize);

/* Resolves blocksize / qlp precision defaults like init_stream_internal_ (stream_encoder.c:742-830).
 * Returns NULL when the configuration is outside what this oracle restates (bps > 24, bad sizes ...). */
fo_encoder *fo_encoder_new(const fo_config *cfg);
void fo_encoder_delete(fo_encoder *e);
const fo_config *fo_encoder_config(const fo_encoder *e);

/* Encode one frame of `blocksize` (<= cfg.blocksize) samples of interleaved int32 PCM.
 * Returns the frame length in bytes, 0 on error. plan may be NULL. */
size_t fo_encode_frame(fo_encoder *e, const int32_t *interleaved, uint32_t blocksize, uint32_t frame_number,
                       uint8_t *out, size_t out_cap, fo_frame_plan *plan);

/* Encode a whole PCM buffer as consecutive frames (last one short), frame numbers from 0. */
int fo_encode_stream(fo_encoder *e, const int32_t *interleaved, uint64_t samples_per_channel,
                     uint8_t *out, size_t out_cap, size_t *out_len,
                     uint32_t *frame_sizes, size_t max_frames, size_t *nframes);

/* Stage-level entry points (same arithmetic the frame encoder uses). */
void fo_window_tukey(float *window, int32_t L, float p);
int fo_window(const fo_apodization *a, float *window, int32_t L);     /* any FO_APOD_* ; 0 on unknown type */
void fo_config_set_apodization(fo_config *cfg, const char *spec);     /* FLAC__stream_encoder_set_apodization */
void fo_autocorrelation(const float *data, uint32_t data_len, uint32_t lag, double *autoc);
void fo_window_data(const int32_t *in, const float *window, float *out, uint32_t data_len);  /* lpc.c:68-74 */
void fo_window_data_partial(const int32_t *in, const float *window, float *out, uint32_t data_len, uint32_t part_size,
                            uint32_t data_shift);                                            /* lpc.c:82-94 */
void fo_lp_coefficients(const double *autoc, uint32_t *max_order, float lp_coeff[][FO_MAX_LPC_ORDER], double *error);
uint32_t fo_best_order(const double *lpc_error, uint32_t max_order, uint32_t total_samples, uint32_t overhead_bits_per_order);
int fo_quantize_coefficients(const float *lp_coeff, uint32_t order, uint32_t precision, int32_t *qlp_coeff, int *shift);
uint8_t fo_crc8(const uint8_t *data, size_t len);
uint16_t fo_crc16(const uint8_t *data, size_t len);
/* lpc.c:942-968 FLAC__lpc_max_prediction_value_before_shift / FLAC__lpc_max_residual_bps */
uint64_t fo_max_prediction_value_before_shift(uint32_t subframe_bps, const int32_t *qlp, uint32_t order);
uint32_t fo_max_residual_bps(uint32_t subframe_bps, const int32_t *qlp, uint32_t order, int lp_quantization);
uint32_t fo_silog2(int64_t v);

/* What the CUDA encoder's stage A must produce for nblocks whole blocks of cfg.blocksize samples (interleaved int32 PCM), per
 * (block, signal) item -- signals are the channels, then mid and side when the configuration codes mid-side, formed as
 * stream_encoder.c:3777-3867 forms them:
 *   meta[2 * item], meta[2 * item + 1]: wasted bits and subframe bps; both 0 for the pair a loose mid-side block does not code;
 *   sigor[item]: the OR of the signal's samples before its wasted bits are shifted out (0 for an uncoded pair);
 *   rows[(sec * nitems + item) * lag_stride + l], l < lags: the autocorrelation of every section apply_apodization_ computes
 *   (:4318-4392), in the order it computes them; punch-out differences are not sections. unshifted = 1: rows of the signal
 *   before its wasted bits are shifted out. An uncoded pair's rows are 0.
 * lags may exceed max_lpc_order + 1 (the kernels compute a fixed number of lags): every lag is the same ascending sum.
 * Returns the number of sections, -1 on bad arguments or when rows_cap (doubles) is too small. */
int fo_stage_a(fo_encoder *e, const int32_t *interleaved, uint32_t nblocks, uint32_t lags, uint32_t lag_stride, int unshifted,
               double *rows, size_t rows_cap, int32_t *meta, uint32_t *sigor);

/* One LPC candidate of one apodization, in the order process_subframe_ evaluates them (stream_encoder.c:4220-4260, 4591-4599). */
enum { FO_LPC_QUANTIZED = 0, FO_LPC_SHIFT_TOO_SMALL = 1, FO_LPC_CMAX_ZERO = 2, FO_LPC_DONT_EVEN_TRY = 3 };
typedef struct {
	int32_t status;          /* FO_LPC_*: 1 and 2 are quantize_coefficients' return codes; 3 skips the whole order */
	int32_t order;
	int32_t precision_tried; /* the precision the search asked for */
	int32_t precision;       /* after the <= 17-bit cap */
	int32_t shift;
	int32_t negative_shift;  /* quantised through the divide branch: the computed shift was negative, the coded one is 0 */
	int32_t qlp[FO_MAX_LPC_ORDER];
} fo_lpc_cand;
#define FO_MAX_LPC_CANDIDATES (FO_MAX_LPC_ORDER * (15 - 5 + 1))

/* Levinson-Durbin on autoc[0 .. max_order], the order guess (or every order with do_exhaustive_model_search) and every
 * precision the configuration tries (cfg: do_qlp_coeff_prec_search, qlp_coeff_precision, do_exhaustive_model_search).
 * Returns the number of candidates written to out (at most FO_MAX_LPC_CANDIDATES); 0 when autoc[0] == 0. The frame encoder
 * evaluates exactly these. */
size_t fo_lpc_candidates(const double *autoc, uint32_t max_order, uint32_t subframe_bps, uint32_t blocksize, const fo_config *cfg,
                         fo_lpc_cand *out);

/* evaluate_lpc_subframe_ from the residual on (stream_encoder.c:4600-4666) for one quantised candidate on one subframe, with
 * the encoder's Rice parameter limit and the given partition orders: the estimate, 0 when a checked residual leaves int32. */
uint32_t fo_lpc_estimate(fo_encoder *e, const int32_t *signal, uint32_t blocksize, uint32_t subframe_bps, uint32_t wasted,
                         const fo_lpc_cand *c, uint32_t min_po, uint32_t max_po);

/* How often the encoder took each rarely reached branch of its LPC stage, summed over every call in the process since the
 * last reset. The counters are one process-wide static that every encode increments without synchronisation: encodes run
 * concurrently from several threads race on them (their frames stay correct, the counts do not), so read them only from
 * single-threaded tests. */
typedef struct {
	uint64_t shift_clamped;     /* quantize: shift above 15 clamped to 15 */
	uint64_t negative_shift;    /* quantize: divide branch, shift set to 0 */
	uint64_t shift_too_small;   /* quantize: shift below -16, candidate dropped (return 1) */
	uint64_t cmax_zero;         /* quantize: every coefficient 0, candidate dropped (return 2) */
	uint64_t coef_clipped;      /* quantize: a coefficient clipped to qmin / qmax */
	uint64_t round_half;        /* quantize: lround of an accumulated error of exactly +-.5 */
	uint64_t precision_capped;  /* subframe bps <= 17: the precision lowered to 32 - bps - ilog2(order) */
	uint64_t order_skipped;     /* "don't even try": expected bits >= subframe bps */
	uint64_t levinson_early;    /* Levinson's error reached 0.0 before max_order */
	uint64_t wide;              /* evaluated: prediction before shift > 32 bits, or limit */
	uint64_t limit;             /* evaluated: max residual bps > 32 */
	uint64_t limit_rejected;    /* evaluated with limit: a residual left (INT32_MIN, INT32_MAX], candidate dropped */
	uint64_t narrow_wrapped;    /* a partition sum the 32-bit accumulator wrapped */
} fo_lpc_counters;
void fo_lpc_counters_get(fo_lpc_counters *out, int reset);

/* ---- decode ---- */
typedef struct {
	uint32_t channels, bits_per_sample, sample_rate; /* from STREAMINFO, used when the header says "get from STREAMINFO" */
} fo_streaminfo;

/* Decode one frame starting at data[0]. Writes interleaved int32 PCM. Returns bytes consumed,
 * 0 on error (bad sync, CRC mismatch, unsupported). */
size_t fo_decode_frame(const uint8_t *data, size_t len, const fo_streaminfo *si,
                       int32_t *out_interleaved, size_t out_cap_samples_per_channel,
                       uint32_t *blocksize, uint32_t *channels, uint32_t *bps, uint64_t *frame_or_sample_number);

#ifdef __cplusplus
}
#endif
#endif
