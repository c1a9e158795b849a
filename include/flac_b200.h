/*
 * flac_b200.h -- C ABI of the H100-native FLAC block engine (libflac_b200.so).
 *
 * Plain pointers and sizes only. This is the boundary the reference's per-frame hot path
 * is replaced at: everything libFLAC does between "a blocksize worth of samples is
 * buffered" and "the frame bytes are handed to the write callback"
 *   reference: process_frame_ -> process_subframes_ -> add_subframe_ -> CRC-16
 *              (src/libFLAC/stream_encoder.c:3435-3480, 3747-4043)
 * and, for decode, between "frame bytes located" and "PCM handed to the write callback"
 *   reference: read_frame_ (src/libFLAC/stream_decoder.c:2373-2622).
 *
 * The FLAC__stream_encoder_* / FLAC__stream_decoder_* object API (include/flac_b200_stream.h)
 * is implemented in host C++ on top of these entry points.
 *
 * All functions return 0 on success or a negative FB200_ERR_* code; there is no CPU
 * fallback: without a CUDA device every compute entry point fails with FB200_ERR_CUDA.
 */
#ifndef FLAC_B200_H
#define FLAC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FB200_MAX_CHANNELS 8
#define FB200_MAX_LPC_ORDER 32
#define FB200_MAX_APODIZATIONS 32

enum {
	FB200_OK = 0,
	FB200_ERR_CUDA = -1,          /* no device / CUDA runtime failure (see fb200_last_error) */
	FB200_ERR_UNSUPPORTED = -2,   /* legal FLAC setting outside this engine's scope; fails loudly, no fallback */
	FB200_ERR_INVALID = -3,       /* illegal argument (mirrors FLAC__StreamEncoderInitStatus rejections) */
	FB200_ERR_OUTPUT_TOO_SMALL = -4,
	FB200_ERR_BAD_STREAM = -5,    /* decoder: sync/CRC/parse error in a frame */
	FB200_ERR_ALLOC = -6
};

/* Apodization functions (reference: FLAC__stream_encoder_set_apodization,
 * src/libFLAC/stream_encoder.c:1939-2065; window generators src/libFLAC/window.c:50-302).
 * Every function the reference's specification string knows is here; the window tables are
 * generated on the host once per blocksize (flac_b200/csrc/windows.h). */
enum {
	FB200_APOD_TUKEY = 0,            /* tukey(P) */
	FB200_APOD_SUBDIVIDE_TUKEY = 1,  /* subdivide_tukey(N[/P]) */
	FB200_APOD_BARTLETT = 2,
	FB200_APOD_BARTLETT_HANN = 3,
	FB200_APOD_BLACKMAN = 4,
	FB200_APOD_BLACKMAN_HARRIS_4TERM_92DB_SIDELOBE = 5,
	FB200_APOD_CONNES = 6,
	FB200_APOD_FLATTOP = 7,
	FB200_APOD_GAUSS = 8,            /* gauss(STDDEV): stddev in .p */
	FB200_APOD_HAMMING = 9,
	FB200_APOD_HANN = 10,
	FB200_APOD_KAISER_BESSEL = 11,
	FB200_APOD_NUTTALL = 12,
	FB200_APOD_RECTANGLE = 13,
	FB200_APOD_TRIANGLE = 14,
	FB200_APOD_PARTIAL_TUKEY = 15,   /* one window of partial_tukey(N[/OV[/P]]): .p .start .end */
	FB200_APOD_PUNCHOUT_TUKEY = 16,  /* one window of punchout_tukey(N[/OV[/P]]): .p .start .end */
	FB200_APOD_WELCH = 17
};

typedef struct {
	int32_t type;   /* FB200_APOD_* */
	float p;        /* tukey(p) / gauss(stddev); for subdivide_tukey(n/p) this is p/n as the reference stores it (:2045) */
	int32_t parts;  /* subdivide_tukey parts */
	float start;    /* partial_/punchout_tukey: window start as a fraction of the block (:2008, :2029) */
	float end;      /* partial_/punchout_tukey: window end as a fraction of the block (:2009, :2030) */
} fb200_apodization;

/* One field per FLAC__stream_encoder_set_* knob that reaches the per-frame path
 * (include/FLAC/stream_encoder.h:738-1289; defaults src/libFLAC/stream_encoder.c:2630-2660). */
typedef struct {
	uint32_t channels;                      /* set_channels           1..8 */
	uint32_t bits_per_sample;               /* set_bits_per_sample    4..24 (25..32 -> FB200_ERR_UNSUPPORTED) */
	uint32_t sample_rate;                   /* set_sample_rate */
	uint32_t blocksize;                     /* set_blocksize          0 = reference default (1152 / 4096) */
	int32_t do_mid_side_stereo;             /* set_do_mid_side_stereo */
	int32_t loose_mid_side_stereo;          /* set_loose_mid_side_stereo */
	uint32_t max_lpc_order;                 /* set_max_lpc_order      0..32 */
	uint32_t qlp_coeff_precision;           /* set_qlp_coeff_precision 0 = reference default */
	int32_t do_qlp_coeff_prec_search;       /* set_do_qlp_coeff_prec_search (flac -p; stream_encoder.c:4230-4243) */
	int32_t do_exhaustive_model_search;     /* set_do_exhaustive_model_search */
	uint32_t min_residual_partition_order;  /* set_min_residual_partition_order */
	uint32_t max_residual_partition_order;  /* set_max_residual_partition_order (<= 8) */
	uint32_t num_apodizations;
	fb200_apodization apodizations[FB200_MAX_APODIZATIONS];
	int32_t disable_constant_subframes;     /* FLAC__stream_encoder_disable_constant_subframes (share/private.h:41) */
	int32_t disable_fixed_subframes;        /* ..._disable_fixed_subframes */
	int32_t disable_verbatim_subframes;     /* ..._disable_verbatim_subframes */
	int32_t limit_min_bitrate;              /* set_limit_min_bitrate (stream_encoder.c:3874) */
} fb200_encoder_config;

typedef struct fb200_encoder fb200_encoder;
typedef struct fb200_decoder fb200_decoder;

/* ---- library ---- */
const char *fb200_version(void);
const char *fb200_last_error(void);          /* thread-local description of the last failure */
int fb200_device_count(void);                /* <0: FB200_ERR_CUDA */

/* ---- encoder ----
 * fb200_encoder_config_preset == FLAC__stream_encoder_set_compression_level
 * (stream_encoder.c:117-140, 1873-1904) plus set_channels/bits_per_sample/sample_rate/blocksize. */
int fb200_encoder_config_preset(fb200_encoder_config *cfg, uint32_t channels, uint32_t bits_per_sample,
                                uint32_t sample_rate, uint32_t compression_level, uint32_t blocksize);

/* FLAC__stream_encoder_set_apodization (stream_encoder.c:1940-2065): parse a ';'-separated
 * specification ("tukey(0.5);partial_tukey(2);gauss(0.2);hann" ...) into cfg->apodizations. */
int fb200_encoder_config_set_apodization(fb200_encoder_config *cfg, const char *specification);
/* The window table the encoder uploads for one apodization at block length `length`
 * (FLAC__window_* of src/libFLAC/window.c); host-side, needs no GPU. */
int fb200_window(const fb200_apodization *apodization, int32_t length, float *out);

/* Validates like init_stream_internal_ (stream_encoder.c:725-830), resolves blocksize and
 * qlp precision defaults, uploads window tables, sizes device workspaces for up to
 * max_blocks_per_launch blocks (0 = default). */
int fb200_encoder_create(const fb200_encoder_config *cfg, int device, uint32_t max_blocks_per_launch, fb200_encoder **out);
void fb200_encoder_destroy(fb200_encoder *enc);
int fb200_encoder_get_config(const fb200_encoder *enc, fb200_encoder_config *resolved);
/* Upper bound for one frame in bytes (verbatim worst case), for sizing output buffers. */
size_t fb200_encoder_max_frame_bytes(const fb200_encoder *enc);

/*
 * Encode `samples` samples per channel of interleaved, sign-extended int32 PCM
 * (the layout of FLAC__stream_encoder_process_interleaved, include/FLAC/stream_encoder.h:1896)
 * as consecutive frames of `blocksize` samples, the last one short, numbered from
 * first_frame_number. Frames are written back to back into `out`; frame i occupies
 * [frame_offsets[i], frame_offsets[i+1]) and *nframes = ceil(samples / blocksize).
 * frame_offsets must hold *nframes + 1 entries.
 *
 * _host:   pcm/out/frame_offsets are HOST pointers; H2D and D2H copies happen inside.
 * _device: pcm/out/frame_offsets are DEVICE pointers on the encoder's device; kernels are
 *          enqueued on `cuda_stream` (a cudaStream_t, may be NULL) and the call returns after
 *          enqueueing unless `sync` is non-zero. total_bytes (host, optional) needs sync.
 */
int fb200_encode_host(fb200_encoder *enc, const int32_t *pcm_interleaved, uint64_t samples,
                      uint32_t first_frame_number, uint8_t *out, size_t out_capacity,
                      uint64_t *frame_offsets, uint32_t *nframes);

/* The same for packed little-endian signed PCM, bytes_per_sample = 2 (bits_per_sample <= 16), 3 (<= 24) or 4
 * (== fb200_encode_host): the bytes a WAV/AIFF reader holds before the reference's client widens them to int32
 * (src/flac/encode.c:2352 format_input, feed loop :1199-1309). Half (or 3/4) of the host->device traffic of the
 * int32 layout; one device kernel widens it. A sample outside bits_per_sample fails with FB200_ERR_INVALID
 * (the reference's process() range check, stream_encoder.c:2543-2548). */
int fb200_encode_host_packed(fb200_encoder *enc, const void *pcm_interleaved, uint32_t bytes_per_sample, uint64_t samples,
                             uint32_t first_frame_number, uint8_t *out, size_t out_capacity,
                             uint64_t *frame_offsets, uint32_t *nframes);

/* Many-file batches: frame numbers restart at first_frame_number every blocks_per_file blocks, i.e. the call
 * encodes consecutive files of blocks_per_file full blocks each, every one numbered like its own stream
 * (stream_encoder.c:3772: frame_number = current_frame_number of that encoder). 0 = one stream (default). */
int fb200_encoder_set_file_blocks(fb200_encoder *enc, uint32_t blocks_per_file);

int fb200_encode_device(fb200_encoder *enc, const int32_t *d_pcm_interleaved, uint64_t samples,
                        uint32_t first_frame_number, uint8_t *d_out, size_t out_capacity,
                        uint64_t *d_frame_offsets, uint32_t *nframes, uint64_t *total_bytes,
                        void *cuda_stream, int sync);

/* Number of kernel launches issued by this encoder so far (bench.py's gpu_launches). */
uint64_t fb200_encoder_launch_count(const fb200_encoder *enc);

/* Measurement support: per-kernel device time from CUDA events recorded on the launching
 * stream between the kernels of every launch (off by default). Index = FB200_PROF_*. */
enum { FB200_PROF_PREP = 0, FB200_PROF_AUTOC, FB200_PROF_LPC, FB200_PROF_SEARCH, FB200_PROF_EMIT,
       FB200_PROF_SCAN, FB200_PROF_GATHER, FB200_PROF_KERNELS };
int fb200_encoder_set_profiling(fb200_encoder *enc, int on);
int fb200_encoder_get_profile(fb200_encoder *enc, double ms[FB200_PROF_KERNELS], uint64_t launches[FB200_PROF_KERNELS], int reset);

/* Stage-level debug access used by the parity tests: the per-signal decisions (fb200::SubframePlan,
 * flac_b200/csrc/fb200_internal.h) and channel assignments of the most recent launch. */
int fb200_debug_copy_plans(fb200_encoder *enc, uint32_t nblocks, void *host_plans, size_t plan_bytes, uint32_t *host_chan_assign);
/* y[i] = the engine's device restatement of the host libm's log(x[i]) (reference: lpc.c:1594, fixed.c:284). */
int fb200_debug_log(const double *x, double *y, uint32_t n, int device);

/* ---- decoder ----
 * Batch frame decode (read_frame_ for many frames). The caller supplies frame boundaries
 * (frames carry no length field; SURVEY.md §3.3) and the STREAMINFO facts. Every frame must
 * have `blocksize` samples except the last, which may be shorter. Output is interleaved
 * int32 PCM, frame i at sample offset i*blocksize. */
typedef struct {
	uint32_t channels, bits_per_sample, sample_rate, blocksize;
} fb200_decoder_config;

int fb200_decoder_create(const fb200_decoder_config *cfg, int device, uint32_t max_frames_per_launch, fb200_decoder **out);
void fb200_decoder_destroy(fb200_decoder *dec);

int fb200_decode_host(fb200_decoder *dec, const uint8_t *frames, const uint64_t *frame_offsets, uint32_t nframes,
                      int32_t *pcm_interleaved, uint64_t pcm_capacity_samples, uint64_t *samples_decoded,
                      uint32_t *bad_frames);

/* The same with the samples narrowed on the device to packed little-endian PCM (bytes_per_sample 2 or 3; 4 = int32): what
 * a WAV writer stores, and the smaller device-to-host copy -- the end-to-end bound of a decoder. */
int fb200_decode_host_packed(fb200_decoder *dec, const uint8_t *frames, const uint64_t *frame_offsets, uint32_t nframes,
                             void *pcm_interleaved, uint32_t bytes_per_sample, uint64_t pcm_capacity_samples, uint64_t *samples_decoded,
                             uint32_t *bad_frames);

/* _device: d_frames must be readable 8 bytes past the last frame (the bit reader fetches whole
 * aligned words); d_frame_status[i] = status (low byte, 0 = ok) | decoded blocksize << 8. */
int fb200_decode_device(fb200_decoder *dec, const uint8_t *d_frames, const uint64_t *d_frame_offsets, uint32_t nframes,
                        int32_t *d_pcm_interleaved, uint64_t pcm_capacity_samples, uint32_t *d_frame_status,
                        void *cuda_stream, int sync);

uint64_t fb200_decoder_launch_count(const fb200_decoder *dec);

/* Per-frame status words of the last fb200_decode_host / fb200_decode_indexed_host call: low byte 0 = ok, else
 * 1 sync, 2 header, 3 CRC-8, 4 unsupported, 5 parse / sample out of range, 6 length, 7 CRC-16, 8 STREAMINFO mismatch;
 * upper 24 bits: the frame's blocksize. (The reference reports these per frame through its error callback and does not
 * deliver the frame: stream_decoder.c:2443-2590.) */
int fb200_decoder_get_frame_status(const fb200_decoder *dec, uint32_t *status, uint32_t nframes);

/* What the reference hands a client in FLAC__Frame.subframes[] (include/FLAC/format.h:211-484; consumer: src/flac/analyze.c),
 * collected by the decode kernels when enabled: one record per (frame, channel) of the last decode call. */
typedef struct {
	uint8_t type;       /* 0 constant, 1 verbatim, 2 fixed, 3 lpc */
	uint8_t order;
	uint8_t wasted_bits;
	uint8_t qlp_coeff_precision;
	int8_t quantization_level;
	uint8_t entropy_method;   /* 0 PARTITIONED_RICE, 1 PARTITIONED_RICE2 */
	uint8_t partition_order;
	uint8_t reserved;
	int32_t qlp_coeff[FB200_MAX_LPC_ORDER];
	int32_t warmup[FB200_MAX_LPC_ORDER];  /* constant subframes: warmup[0] is the value */
} fb200_subframe_info;
int fb200_decoder_enable_subframe_info(fb200_decoder *dec, int on);
int fb200_decoder_get_subframe_info(fb200_decoder *dec, fb200_subframe_info *info, uint32_t nframes);

/* Stream-level front end: fb200_decoder_index_host copies `stream` (frames only or a whole .flac file) to the device and
 * returns, ascending, every byte offset that carries a sync code and a self-consistent frame header (frame_sync_ +
 * read_frame_header_ incl. CRC-8, stream_decoder.c:2321-2371, 2624-2947, for all positions at once). The stream stays
 * resident; fb200_decode_indexed_host decodes the frames STARTING at begins[i], each bounded by max_frame_bytes: the parse
 * finds the frame's true length (frame_bytes[i]) and the CRC-16 is checked over exactly that, so junk between or after frames
 * (ID3v1 / APE tags, padding) costs nothing. A false candidate fails its parse or CRC-16 (frame_status[i] != 0). */
int fb200_decoder_index_host(fb200_decoder *dec, const uint8_t *stream, uint64_t nbytes, uint64_t *candidates, uint32_t capacity, uint32_t *ncandidates);
int fb200_decode_indexed_host(fb200_decoder *dec, const uint64_t *begins, uint32_t nframes, uint32_t max_frame_bytes, uint64_t stream_bytes,
                              int32_t *pcm_interleaved, uint64_t pcm_capacity_samples, uint32_t *frame_status, uint32_t *frame_bytes);

enum { FB200_DPROF_WALK = 0, FB200_DPROF_CRC, FB200_DPROF_FRAMES, FB200_DPROF_KERNELS };  /* k_dec_walk, k_dec_crc, k_dec_frames */
int fb200_decoder_set_profiling(fb200_decoder *dec, int on);
int fb200_decoder_get_profile(fb200_decoder *dec, double ms[FB200_DPROF_KERNELS], uint64_t launches[FB200_DPROF_KERNELS], int reset);

#ifdef __cplusplus
}
#endif
#endif /* FLAC_B200_H */
