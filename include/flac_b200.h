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
	FB200_ERR_ALLOC = -6,
	FB200_ERR_VERIFY = -7         /* encoder verify: a file of the call failed verification (fb200_encoder_get_verify) */
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
	/* Which fixed-order guess the encoder reproduces. libFLAC picks the fixed predictor order it tries from the abs sums of
	 * each difference order. On x86-64 hosts with AVX2 it computes those sums for "wide" subframes (subframe bps < 28 and
	 * bps + ilog2((blocksize - 4) * 17) >= 32, stream_encoder.c:4098-4103) with FLAC__fixed_compute_best_predictor_wide_intrin_avx2
	 * (fixed_intrin_avx2.c:57-138) instead of its C routine. That routine splits the block into four lanes that skip up to 3
	 * samples and read a few samples of history from the wrong place whenever blocksize - 4 is not a multiple of 4 (short last
	 * blocks, odd blocksizes), so it can guess another order there, and the frames the flac tool writes on such a host differ.
	 * 0 (default, written by fb200_encoder_config_preset): the C routine, what libFLAC computes everywhere else.
	 * 1: the AVX2 routine for wide subframes, as libFLAC on an AVX2 host. fb200_host_x86_avx2_fixed_guess() tells which one the
	 *    flac tool on this host uses. Full blocks of the standard blocksizes are identical in both modes.
	 * Any other value fails fb200_encoder_create with FB200_ERR_INVALID. */
	int32_t x86_avx2_fixed_guess;
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

/* 1 when libFLAC on this host would take its x86 AVX2 fixed-order guess (cpu.c:151-200: CPUID leaf 1 ECX has AVX and OSXSAVE,
 * XGETBV(0) & 6 == 6, the maximum CPUID leaf is at least 7 and leaf 7 EBX has AVX2), else 0; always 0 on builds for other
 * CPUs. Set fb200_encoder_config.x86_avx2_fixed_guess from it for the frames the flac tool writes on this host. Needs no GPU. */
int fb200_host_x86_avx2_fixed_guess(void);

/* FLAC__stream_encoder_set_apodization (stream_encoder.c:1940-2065): parse a ';'-separated
 * specification ("tukey(0.5);partial_tukey(2);gauss(0.2);hann" ...) into cfg->apodizations. */
int fb200_encoder_config_set_apodization(fb200_encoder_config *cfg, const char *specification);
/* The window table the encoder uploads for one apodization at block length `length`
 * (FLAC__window_* of src/libFLAC/window.c); host-side, needs no GPU. */
int fb200_window(const fb200_apodization *apodization, int32_t length, float *out);

/* Validates like init_stream_internal_ (stream_encoder.c:725-830), resolves blocksize and
 * qlp precision defaults, uploads window tables, sizes device workspaces for up to
 * max_blocks_per_launch blocks (0 = default: 4096 blocks).
 *
 * Blocks whose signal or frame does not fit one CTA's shared memory (e.g. 24-bit stereo at
 * 16384, 24-bit 5.1 at 8192, any channel count at 32768 and up) are encoded by the tiled
 * kernels. For such a configuration the default capacity is FB200_TILED_SAMPLE_BUDGET
 * samples: budget / (blocksize * channels) blocks, at least 1 and at most 4096 (1024 blocks of
 * 16384 x 2, 64 of 65535 x 8; the workspaces take at most about 25 bytes per sample of
 * capacity, so the default stays under 1 GB). The FLAC__stream_encoder_* shell bounds its
 * batch by the same budget for these configurations only. */
#define FB200_TILED_SAMPLE_BUDGET (1u << 25)
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

/* ---- batches of whole files ----
 * nfiles files of file_samples[f] samples per channel each, back to back in pcm_interleaved, all with the encoder's
 * configuration, each encoded as its own stream: frames numbered from 0 (stream_encoder.c:3772), the short last block as its
 * last frame (:1703-1711), byte-identical to encoding that file alone. The output is file-major: file f's frames are
 * frame_offsets[files[f].first_frame ... + files[f].nframes] (frame i occupies [frame_offsets[i], frame_offsets[i+1])),
 * *nframes is the total and frame_offsets must hold *nframes + 1 entries (at most sum of ceil(file_samples / blocksize) + 1).
 * With do_md5 the MD5 of each file's samples (as little-endian integers of (bits_per_sample + 7) / 8 bytes, md5.c:280-521)
 * is computed on the device; without, the STREAMINFO MD5 is all zero.
 * A file of 0 samples, nfiles == 0, or a sample outside bits_per_sample fails with FB200_ERR_INVALID, a short `out` with
 * FB200_ERR_OUTPUT_TOO_SMALL. fb200_encoder_set_file_blocks does not apply to these entry points.
 *
 * _host:   bytes_per_sample 2, 3 or 4 (packed little-endian signed PCM, as fb200_encode_host_packed); host pointers.
 * _device: int32 PCM, out and frame_offsets on the device, file_samples and files on the host; enqueued on cuda_stream,
 *          returns after completion. */
typedef struct {
	uint64_t first_frame;     /* index into frame_offsets of this file's first frame */
	uint32_t nframes;         /* ceil(samples / blocksize) */
	uint8_t  streaminfo[34];  /* STREAMINFO body as update_metadata_ leaves it (format.c:65-73): min/max blocksize = the
	                             configured blocksize (stream_encoder.c:1358-1359), min/max frame size over all of the file's
	                             frames (:3031-3032), rate / channels / bps, total samples, MD5 (all zero when do_md5 == 0) */
} fb200_file_info;

int fb200_encode_files_host(fb200_encoder *enc, const void *pcm_interleaved, uint32_t bytes_per_sample,
                            const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                            uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                            fb200_file_info *files);
int fb200_encode_files_device(fb200_encoder *enc, const int32_t *d_pcm_interleaved,
                              const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                              uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes,
                              fb200_file_info *files, void *cuda_stream);

/* ---- batches of complete .flac files ----
 * The same encode, each file written as the whole stream libFLAC's encoder writes when given that file's
 * FLAC__stream_encoder_set_metadata blocks and a seek callback (init_stream + process + finish, stream_encoder.c:1336-1430,
 * write_frame_ :3065-3103, update_metadata_ :3139-3300). File f is out[files[f].offset, + files[f].bytes), the files back to back:
 *   "fLaC"; STREAMINFO (not last) as fb200_file_info carries it; an empty VORBIS_COMMENT unless the file's blocks hold one (last
 *   when there are no client blocks); the client blocks in their order, the last one flagged last; the frames, byte for byte
 *   those of fb200_encode_files_* for the same call.
 * File f's client blocks are metadata[metadata_offsets[f], metadata_offsets[f + 1]) (both NULL: none for any file): metadata
 * blocks in stream syntax, back to back, each a 4-byte header (last flag, 7-bit type, 24-bit length) and its body, so a block
 * lifted from a .flac can be passed as it is. They are written as FLAC__add_metadata_block writes them
 * (stream_encoder_framing.c:47-243): a VORBIS_COMMENT gets this library's FLAC__VENDOR_STRING and its length adjusted, a PADDING
 * body is zeros, the reserved fields of a CUESHEET are zeros, and every other block keeps its bytes. A SEEKTABLE body is a
 * template of 18-byte big-endian points: a point t below the file's length L becomes {first sample of the frame holding t, that
 * frame's offset from the first frame, its samples (the tail length for the short last frame)}, a point t > L a placeholder that
 * keeps its other fields, t == L stays as given; then the table is sorted, uniquified and filled up with placeholders
 * (format.c:281-314), so points that land on one frame collapse into one.
 *
 * Rejected with FB200_ERR_INVALID before any device work (fb200_last_error names the file, the block and the rule): every list
 * init_stream_internal_ rejects with INVALID_METADATA (stream_encoder.c:869-920) -- a STREAMINFO, a second SEEKTABLE or
 * VORBIS_COMMENT, a seek table not ascending up to its placeholders, a CUESHEET or PICTURE that FLAC__format_*_is_legal rejects
 * (the CD-DA rules when is_cd is set), a second picture of type 1 or 2, a type-1 picture that is not a 32x32 PNG -- and what only
 * a byte blob can get wrong: a block running past its file's slice, type 127, a SEEKTABLE length not a multiple of 18, a
 * VORBIS_COMMENT, CUESHEET or PICTURE whose fields disagree with its block length, a NUL in a PICTURE's MIME type or
 * description, an APPLICATION block shorter than 4 bytes. A short `out` gives FB200_ERR_OUTPUT_TOO_SMALL; verify works and
 * fails as with fb200_encode_files_*. frame_offsets (may be NULL) receives the absolute start of every frame in `out`, entry
 * nframes being the end of the last file. Unlike with fb200_encode_files_*, frame_offsets[i + 1] - frame_offsets[i] is not the
 * size of a file's last frame (except the last file's): the next entry is the next file's first frame, which follows that file's
 * header. A file's last frame ends at files[f].offset + files[f].bytes.
 *
 * _host: one device-to-host copy of all the files. _device: as fb200_encode_files_device; metadata, metadata_offsets and files
 * are host memory. */
typedef struct {
	uint64_t offset;          /* the file's first byte ("fLaC") in out */
	uint64_t bytes;           /* the file's length: offset[f + 1] == offset[f] + bytes[f] */
	uint64_t audio_offset;    /* the file's first frame, from the file's start (what seek point stream_offset is relative to) */
	uint64_t first_frame;     /* index into frame_offsets of this file's first frame */
	uint32_t nframes;
	uint32_t seek_points;     /* points in the written SEEKTABLE, 0 = none */
	uint8_t  streaminfo[34];  /* as fb200_file_info */
	uint8_t  reserved[6];
} fb200_flac_file_info;

int fb200_encode_flac_files_host(fb200_encoder *enc, const void *pcm_interleaved, uint32_t bytes_per_sample,
                                 const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                                 const uint8_t *metadata, const uint64_t *metadata_offsets,
                                 uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                                 fb200_flac_file_info *files);
int fb200_encode_flac_files_device(fb200_encoder *enc, const int32_t *d_pcm_interleaved,
                                   const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                                   const uint8_t *metadata, const uint64_t *metadata_offsets,
                                   uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes,
                                   fb200_flac_file_info *files, void *cuda_stream);

/* ---- batches of WAV / RF64 / Wave64 / AIFF / AIFF-C files (flac *.wav) ----
 * fb200_pcm_files_probe parses each container file data[file_offsets[f], file_offsets[f + 1]) as the flac tool 1.5.0 does
 * (src/flac/main.c:1510-1556 picks the kind from the first 12 bytes; get_sample_info_wave / _aiff, encode.c:192-803; the
 * checks of flac__encode_file, :934-946), skipping the chunks it skips with the same padding rules. It never fails the call
 * for one file: each file gets a status, and a file the tool rejects gets FB200_PCM_MALFORMED with the tool's rule in `error`.
 * A file the tool encodes but this engine cannot gets FB200_PCM_UNSUPPORTED: 32 significant bits, or no sample present.
 *
 * `declared` is the data chunk's sample count (what the tool sizes the padding and the seek table template from); `samples`
 * the count present in the slice when the data chunk is cut short (the tool encodes those, "unexpected EOF"). A data region
 * whose present bytes do not make whole samples is MALFORMED ("got partial sample"), as the tool fails then. */
enum { FB200_PCM_OK = 0, FB200_PCM_NOT_CONTAINER = 1, FB200_PCM_MALFORMED = 2, FB200_PCM_UNSUPPORTED = 3 };
enum { FB200_PCM_WAVE = 1, FB200_PCM_RF64 = 2, FB200_PCM_WAVE64 = 3, FB200_PCM_AIFF = 4, FB200_PCM_AIFF_C = 5 };
typedef struct {
	uint32_t status;              /* FB200_PCM_* */
	uint32_t kind;                /* FB200_PCM_WAVE .. FB200_PCM_AIFF_C, 0 for NOT_CONTAINER */
	uint32_t channels;
	uint32_t container_bits;      /* 8, 16, 24 or 32: the bits each sample occupies in the data chunk */
	uint32_t shift;               /* padding bits below the sample; bits_per_sample = container_bits - shift */
	uint32_t bits_per_sample;
	uint32_t sample_rate;
	uint32_t is_unsigned;         /* 8-bit WAVE data (0x80 is zero) */
	uint32_t is_big_endian;       /* AIFF and AIFF-C NONE */
	uint32_t channel_mask;        /* WAVEFORMATEXTENSIBLE dwChannelMask, 0 when none */
	uint64_t data_offset;         /* the data region's first byte, an offset into `data` as file_offsets are */
	uint64_t declared;            /* samples per channel the data chunk declares */
	uint64_t samples;             /* samples per channel present in the slice (<= declared) */
	char     error[96];           /* the rule, NUL-terminated, when status is not OK */
} fb200_pcm_file_info;
int fb200_pcm_files_probe(const uint8_t *data, uint64_t nbytes, const uint64_t *file_offsets, uint32_t nfiles,
                          fb200_pcm_file_info *info);

/* fb200_encode_pcm_files_host / _device: the probed files encoded in one call, each written as the .flac file the flac tool
 * writes for it (EncoderSession_init_encoder's metadata for a non-FLAC input, encode.c:1945-2020), by the machinery of
 * fb200_encode_flac_files_*: a SEEKTABLE from "<seek_spacing_s>s;" over the declared sample count
 * (convert_to_seek_table_template, :2207-2255; none when seek_spacing_s is 0 or no point results), a VORBIS_COMMENT of the
 * file's tags plus WAVEFORMATEXTENSIBLE_CHANNEL_MASK=0x%04X when the mask is not 0 (flac__utils_set_channel_mask_tag,
 * src/flac/utils.c:458, replacing a tag of that name), and a PADDING (:2004-2017). Frames, MD5, verify, out, frame_offsets and
 * files[] are as fb200_encode_flac_files_*.
 *
 * k_pcm_unpack widens every file's data region (1-4 byte containers, either byte order, unsigned 8-bit) to the encoder's int32
 * input in one launch, as format_input (:2352-2505) does. A sample whose `shift` low bits are not zero fails the call with
 * FB200_ERR_INVALID, fb200_last_error naming the first such (file, sample, channel); it takes the place of the out-of-range
 * check of fb200_encode_files_*. FB200_ERR_INVALID before any device work: a file not probed OK, or whose channels, bits per
 * sample or rate differ from the encoder's; info[] from another batch; a tag list whose lengths disagree.
 *
 * tags / tag_offsets (both NULL: none): file f's -T entries are tags[tag_offsets[f], tag_offsets[f + 1]), "NAME=value"
 * strings each ending in a NUL, written in that order.
 * _host: one host-to-device copy of the container bytes, one device-to-host copy of the files. _device: data is device memory
 * (only [file_offsets[0], file_offsets[nfiles]) is read); out and frame_offsets as fb200_encode_flac_files_device; file_offsets,
 * info, opt, tags and files are host memory. */
/* replay_gain (flac --replay-gain; src/flac/main.c, encode.c, share/grabbag/replaygain.c): the call is one album, as one
 * invocation of the tool is. Every file must be mono or stereo at a rate fb200_replaygain_device accepts, else
 * FB200_ERR_INVALID before any device work, naming the file. A PADDING block (padding not 0) grows by 190 bytes at encode
 * time (still at most 2^24 - 1). Each file's VORBIS_COMMENT then takes the tool's three edits, in order: reference loudness,
 * track gain and peak, album gain and peak. Each edit removes the entries of its names (the field name before the first '='
 * compared without ASCII case), appends "REPLAYGAIN_REFERENCE_LOUDNESS=89.0 dB", "..._GAIN=%+2.2f dB", "..._PEAK=%1.8f" (C
 * locale), and lays the metadata out again as a metadata chain write with padding does: a shrunk block list extends its last
 * PADDING or gains a new one (from 4 bytes shrunk on), a grown one uses up or trims the last PADDING when that is large enough,
 * and otherwise the metadata grows. files[], audio offsets and frame offsets describe the final files; capacity needs at most
 * 190 more bytes per file than without ReplayGain. The analysis runs on the device concurrently with the encode. */
typedef struct {
	int32_t  seek_spacing_s;  /* -S <n>s: 10 is the tool's default, 0 = -S- (no SEEKTABLE) */
	int32_t  padding;         /* -P: -1 = the tool's default (8192, 65536 from 20 minutes on), 0 = --no-padding */
	uint32_t md5;             /* 0: STREAMINFO MD5 left zero */
	uint32_t replay_gain;     /* non-zero: --replay-gain. 0 is the only value callers before this field existed passed */
} fb200_pcm_encode_options;
int fb200_encode_pcm_files_host(fb200_encoder *enc, const uint8_t *data, const uint64_t *file_offsets, uint32_t nfiles,
                                const fb200_pcm_file_info *info, const fb200_pcm_encode_options *opt,
                                const uint8_t *tags, const uint64_t *tag_offsets,
                                uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                                fb200_flac_file_info *files);
int fb200_encode_pcm_files_device(fb200_encoder *enc, const uint8_t *d_data, const uint64_t *file_offsets, uint32_t nfiles,
                                  const fb200_pcm_file_info *info, const fb200_pcm_encode_options *opt,
                                  const uint8_t *tags, const uint64_t *tag_offsets,
                                  uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes,
                                  fb200_flac_file_info *files, void *cuda_stream);

/* A sample range of one file of a batch: samples [first_sample, first_sample + samples) per channel (the ranged decode
 * fb200_decode_files_ranges_* and the ranged encodes below). */
typedef struct {
	uint32_t file;            /* index into the batch (the indexed batch for .flac input, file_offsets' files for containers) */
	uint32_t reserved;        /* 0 */
	uint64_t first_sample;    /* per channel, from the file's start */
	uint64_t samples;         /* per channel, >= 1 */
} fb200_sample_range;

/* ---- sample ranges of container files (flac [--skip] [--until] *.wav) ----
 * fb200_encode_pcm_files_ranges_host / _device write one .flac per range of the probed files, in request order: range r's output is what flac --skip=<first_sample> --until=<first_sample + samples> writes for file
 * ranges[r].file with the same options, and files[r] describes it (nranges records). A range may name any file any number of
 * times, in any order, and ranges may overlap: k_pcm_unpack widens each range from its own first value, so every range gets its
 * own copy. Everything else is as fb200_encode_pcm_files_*, with the range in place of the file:
 *  - the SEEKTABLE template and the default padding's 20-minute threshold come from the range's length, not the declared count
 *    (total_samples_to_encode, encode.c:2010, 2226);
 *  - the channel-mask tag, MD5 (over the range's samples) and verify work per range; fb200_encoder_get_verify takes nranges
 *    records; fb200_last_error counts ranges where it names a file of the encode;
 *  - tags / tag_offsets hold nranges + 1 offsets: the -T entries are per range;
 *  - with replay_gain the ranges are one album, as one tool invocation with one --skip / --until over several files.
 * FB200_ERR_INVALID before any device work, naming the range and its file: the rules of fb200_encode_pcm_files_* for every file a
 * range names (files no range names are not checked beyond their offsets); ranges NULL, nranges 0 or >= 2^31, a file index >= nfiles,
 * samples 0, first_sample + samples overflowing; a range that starts past `declared` ("value of --skip exceeds input size") or ends
 * past it ("--until value is after end of input").
 * A data chunk cut short (samples < declared) follows the whole-file rule: the samples of the range that are present are encoded
 * and the metadata is sized from the requested length. Known difference: a range that starts at or past the last sample present
 * is FB200_ERR_INVALID, where the tool writes a stream without frames. */
int fb200_encode_pcm_files_ranges_host(fb200_encoder *enc, const uint8_t *data, const uint64_t *file_offsets, uint32_t nfiles,
                                       const fb200_pcm_file_info *info, const fb200_pcm_encode_options *opt,
                                       const fb200_sample_range *ranges, uint32_t nranges, const uint8_t *tags, const uint64_t *tag_offsets,
                                       uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes, fb200_flac_file_info *files);
int fb200_encode_pcm_files_ranges_device(fb200_encoder *enc, const uint8_t *d_data, const uint64_t *file_offsets, uint32_t nfiles,
                                         const fb200_pcm_file_info *info, const fb200_pcm_encode_options *opt,
                                         const fb200_sample_range *ranges, uint32_t nranges, const uint8_t *tags, const uint64_t *tag_offsets,
                                         uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes,
                                         fb200_flac_file_info *files, void *cuda_stream);

/* The flac tool's --skip / --until arithmetic, device-free (flac__utils_parse_skip_until_specification and
 * flac__utils_canonicalize_skip_until_specification, utils.c:78-107, 326-398; main.c:1659-1670; encode.c:1003-1081, 2257-2303):
 * skip NULL is no --skip, until NULL no --until (the tool's "-0"). Both take a sample count or [m]m:ss[.,]sss; seconds become
 * samples as (int64_t)(seconds * sample_rate). skip may not be relative; until may: +N counts from skip, -N from the end, and any
 * relative value that comes to 0 samples (+0, -0, -0:00.1 at a low rate) is the end of the stream. total_samples is the container's
 * declared count or STREAMINFO total_samples; when it is 0 any until but the end is an error. Gives the range
 * [*first_sample, *first_sample + *samples). Every case the tool rejects (a usage error or exit 1) is FB200_ERR_INVALID with the
 * tool's message in fb200_last_error. Known difference: a range of 0 samples (skip equal to the length) is FB200_ERR_INVALID; the
 * tool writes a stream without frames. */
int fb200_skip_until(const char *skip, const char *until, uint32_t sample_rate, uint64_t total_samples, uint64_t *first_sample, uint64_t *samples);

/* ---- re-encoding .flac files (flac -f [-S ..] [-P ..] [-T ..] [--replay-gain] *.flac) ----
 * fb200_reencode_flac_files_host / _device re-encode files[0 .. nfiles) of the batch left resident on `dec` by
 * fb200_decode_files_index into the .flac files the flac tool 1.5.0 writes from FLAC input, back to back in list order. Each listed
 * file must be a distinct index; every one whose index status is FB200_FILE_OK must match the encoder's channels, bits per sample
 * and sample rate (one encoder per format group), and the encoder and decoder must share a device.
 *
 * Per file, as the tool does (src/flac/encode.c: get_sample_info_flac :805-857, EncoderSession_init_encoder :1710-1939):
 *  - A file the index did not pass, or one that starts with an ID3v2 tag, fails (INPUT).
 *  - STREAMINFO total_samples 0 fails the file (NO_TOTAL); so does any decode error (DAMAGED: a damaged stretch or a sample no
 *    accepted frame covers), and, when the input's STREAMINFO MD5 is not all zero, a different MD5 of the decoded samples
 *    (MD5_MISMATCH). MD5 is always computed: it is the output's STREAMINFO MD5 too.
 *  - The metadata list is the input's blocks after STREAMINFO in file order, unknown types included, then: with tags, every input
 *    VORBIS_COMMENT goes (its WAVEFORMATEXTENSIBLE_CHANNEL_MASK tag carries over); with tags or without an input VORBIS_COMMENT, a
 *    new one of the tags goes first, else the input's stays where it was (the encoder writes its own vendor string in either case).
 *    A CUESHEET whose lead-out is not total_samples goes. seek_spacing_s 0 drops every SEEKTABLE, n > 0 replaces them with the
 *    "<n>s" template, first; -1 keeps the input's, or puts the "10s" template first when there is none. A kept table is a template
 *    as fb200_encode_flac_files_* take one: its points are moved to the new frames. Every PADDING block goes, and one PADDING
 *    block ends the list: the sum of the input's, or `padding` when > 0, or the tool's default (8192; 65536 from 20 minutes on)
 *    when the input had none; none when padding is 0 or the size is 0; + 190 with replay_gain; at most 2^24 - 1.
 *  - A list fb200_encode_flac_files_* would reject fails the file (METADATA, `error` naming block and rule).
 * replay_gain: the listed files are one album, as with fb200_encode_pcm_files_*; the analysis sees the decoded samples. Album tags
 * are written only when every listed file succeeds (the tool writes none after a failure). A file that fails gets its status, no
 * bytes, and the call goes on; the output, frame_offsets, *nframes and info[].file describe the files that succeed.
 *
 * FB200_ERR_INVALID before any device work: no resident batch, an index out of range or listed twice, a format mismatch, encoder
 * and decoder on different devices, a tag list whose lengths disagree, and with replay_gain a file that is not mono or stereo, a
 * rate the analysis does not cover, or, above 48 kHz, STREAMINFO blocksizes that are not one fixed multiple of the decimation
 * factor (the tool analyses frame by frame; the values then would depend on the input's frame boundaries).
 *
 * Samples never leave the device: the decoder writes every frame straight into the encoder's input, and that copy is the only
 * one. Known differences from the tool:
 *  - a truncated input whose STREAMINFO MD5 is all zero is DAMAGED (the tool writes a shorter file and exits 0);
 *  - on an MD5 mismatch nothing is written (the tool writes the file and exits 1);
 *  - a 25-32-bit input is INPUT (index status FB200_FILE_UNSUPPORTED);
 *  - junk between frames that carries no frame header is never seen (the files index holds frame headers only, as for
 *    fb200_decode_pcm_files_*), so such a file re-encodes OK where the tool reports lost sync and exits 1;
 *  - a VORBIS_COMMENT with bytes left after its last entry, or whose fields disagree with its length, and a CUESHEET or PICTURE
 *    whose body is not exactly its fields, fail the file with METADATA: the blocks are checked as fb200_encode_flac_files_*
 *    checks client blocks, while the tool's decoder reads what fits, skips the rest and re-encodes the fields it read. Verify (fb200_encoder_set_verify) works and fails as with the other files entry points;
 * fb200_encoder_get_verify then takes nfiles records, OK for a file that was not encoded.
 *
 * _host: out and frame_offsets (may be NULL) are host memory, one device-to-host copy of the files. _device: both on the
 * encoder's device, enqueued on cuda_stream; returns after completion. tags / tag_offsets as fb200_encode_pcm_files_*. */
typedef struct {
	int32_t  seek_spacing_s;  /* -1: no -S (keep the input's SEEKTABLE, else "10s"); 0: -S-; n > 0: -S <n>s */
	int32_t  padding;         /* -1: no -P (the input's PADDING merged, else the tool's default); 0: --no-padding; n > 0: -P n */
	uint32_t replay_gain;     /* non-zero: --replay-gain, the listed files are one album */
	uint32_t reserved;        /* must be 0 (FB200_ERR_INVALID otherwise) */
} fb200_flac_reencode_options;
enum { FB200_REENCODE_OK = 0, FB200_REENCODE_INPUT = 1 /* index status not FB200_FILE_OK, or an ID3v2 tag in front (the tool
                                                             refuses such input, main.c:1524); `error` names it */,
       FB200_REENCODE_NO_TOTAL = 2, FB200_REENCODE_DAMAGED = 3, FB200_REENCODE_MD5_MISMATCH = 4,
       FB200_REENCODE_METADATA = 5 /* the encoder would reject the block list; `error` names block and rule */ };
typedef struct {
	uint32_t status;              /* FB200_REENCODE_* */
	char     error[92];
	fb200_flac_file_info file;    /* as fb200_encode_flac_files_*; bytes == 0 when status != OK */
} fb200_flac_reencode_info;
int fb200_reencode_flac_files_host(fb200_encoder *enc, fb200_decoder *dec, const uint32_t *files, uint32_t nfiles,
                                   const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets,
                                   uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                                   fb200_flac_reencode_info *info);
int fb200_reencode_flac_files_device(fb200_encoder *enc, fb200_decoder *dec, const uint32_t *files, uint32_t nfiles,
                                     const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets,
                                     uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes,
                                     fb200_flac_reencode_info *info, void *cuda_stream);

/* fb200_reencode_flac_files_ranges_host / _device: flac -f --skip=<first_sample> --until=<first_sample + samples> over sample ranges
 * of the resident batch, one .flac per range in request order, info[r] (a FB200_REENCODE_* status) per range. A range may name any
 * file any number of times, in any order, and ranges may overlap. The rules of fb200_reencode_flac_files_* hold per range, with the
 * tool's changes for --skip / --until (encode.c:1003-1130, 1772-1930):
 *  - MD5: the input's STREAMINFO MD5 is never compared (the tool zeroes it whenever --skip or --until is given), so MD5_MISMATCH
 *    does not occur; the output's MD5 covers the range's samples.
 *  - SEEKTABLE: the input's is kept (a template moved to the new frames) only when the range is the whole file (first_sample 0,
 *    samples == total_samples) and seek_spacing_s is -1; otherwise it goes, and with -1 the "10s" template over the range's length
 *    goes first.
 *  - CUESHEET: kept when its lead-out equals the range's length, else dropped; track offsets are not moved (the tool's rule as
 *    written).
 *  - PADDING: the default's 20-minute threshold uses the range's length.
 *  - STREAMINFO total_samples 0 gives NO_TOTAL for every range of that file.
 *  - DAMAGED: a range with a damaged stretch among its candidate frames, or a sample no accepted frame covers, gets no bytes; frames
 *    are accepted as fb200_decode_files_ranges_* accepts them, range_sees_its_frames included.
 * FB200_ERR_INVALID before any device work: the call's checks of fb200_reencode_flac_files_* (a file listed twice excepted), ranges
 * NULL, nranges 0 or >= 2^31, a file index out of range, samples 0, first_sample + samples overflowing, and a range past
 * total_samples of a file whose index status is OK. The decoder's ranged path places every cropped frame straight into the
 * encoder's input; samples never leave the device, and launches do not grow with nranges. Verify gives nranges records. */
int fb200_reencode_flac_files_ranges_host(fb200_encoder *enc, fb200_decoder *dec, const fb200_sample_range *ranges, uint32_t nranges,
                                          const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets,
                                          uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                                          fb200_flac_reencode_info *info);
int fb200_reencode_flac_files_ranges_device(fb200_encoder *enc, fb200_decoder *dec, const fb200_sample_range *ranges, uint32_t nranges,
                                            const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets,
                                            uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes,
                                            fb200_flac_reencode_info *info, void *cuda_stream);

/* ---- ReplayGain analysis of device PCM (the values flac --replay-gain and metaflac --add-replay-gain compute) ----
 * fb200_replaygain_device analyses int32 samples in device memory, in the layout fb200_decode_files_device writes: file f's
 * `samples` x `channels` values interleaved from d_pcm[first_value] on. ReplayGain 1.0 (replaygain_analysis.c): a rate above
 * 48000 is halved until it is a filter rate (8000 ... 48000), every ds-th sample (ds = 2^halvings) goes through the 10th-order
 * Yule-Walker and 2nd-order Butterworth filters, the mean square is taken over 50 ms windows, and the 95th percentile of the
 * windows' loudness gives the gain; peak = max |sample| / 2^(bits_per_sample - 1). Files with the same `album` id form one album
 * (the album gain over all their windows, the album peak over all their samples); they must share a sample rate. Samples must
 * fit bits_per_sample. The values are bit for bit those the flac tool writes for a file it encodes, and those metaflac writes
 * for a .flac file whose frame blocksizes are multiples of ds. track_gain is -24601 for a file shorter than one window.
 *
 * FB200_ERR_INVALID before any launch, naming the file: channels not 1 or 2, bits_per_sample outside 4-24, a rate the filters
 * do not cover, an album whose files differ in sample rate, a file that runs past pcm_values. Returns after completion. */
typedef struct {
	uint64_t first_value;    /* the file's first value in d_pcm */
	uint64_t samples;        /* per channel */
	uint32_t channels;       /* 1 or 2 */
	uint32_t bits_per_sample;
	uint32_t sample_rate;
	uint32_t album;          /* album id: files with the same id form one album */
} fb200_replaygain_file;
typedef struct {
	float track_gain, track_peak, album_gain, album_peak;  /* what the REPLAYGAIN_* tags print */
	uint64_t windows;                                      /* the file's complete 50 ms windows */
} fb200_replaygain_info;
int fb200_replaygain_device(int device, const int32_t *d_pcm, uint64_t pcm_values, const fb200_replaygain_file *files, uint32_t nfiles,
                            fb200_replaygain_info *info, void *cuda_stream);
/* Test hook: the same analysis; every window's mean square v = (left + right sum) / W * 0.5 + 1e-37 (mono: left twice), file
 * after file, into host windows[0 .. *nwindows) (FB200_ERR_OUTPUT_TOO_SMALL when more than capacity, *nwindows still set). */
int fb200_debug_replaygain_windows(int device, const int32_t *d_pcm, uint64_t pcm_values, const fb200_replaygain_file *files, uint32_t nfiles,
                                   double *windows, uint64_t capacity, uint64_t *nwindows, void *cuda_stream);

/* ---- ReplayGain tags on existing .flac files (metaflac --add-replay-gain / --scan-replay-gain) ----
 * fb200_add_replaygain_flac_files_host / _device tag files[0 .. nfiles) of the batch left resident on `dec` by
 * fb200_decode_files_index as metaflac 1.5.0 does (src/metaflac/operations.c:557-650, share/grabbag/replaygain.c). The audio frames
 * are not touched. albums[i] (NULL: all one album) is file i's album id; each album is one metaflac invocation, and albums fail
 * independently of each other. Per album, in list order:
 *  1. Pre-checks: a file the index did not pass is INPUT; a file whose rate, bits or channels differ from the album's first file's,
 *     or whose rate the filters do not cover, or that has 3 or more channels, is FORMAT. Either fails the album.
 *  2. Analysis: every file is decoded with MD5 checking off. Any decode error fails the album with DECODE: a damaged or missing
 *     frame (a gap in the sample numbers between two frames included, where libFLAC reports MISSING_FRAME), a frame whose header codes a sample rate other than STREAMINFO's, and any byte of the audio region that no accepted
 *     frame covers (the frames must tile [audio_offset_in, end of file) exactly: junk between or after the frames, a truncated last
 *     frame). The analysis feeds the filters frame by frame in calls of at most 2048 samples, as grabbag__replaygain_analyze does
 *     (each call decimates from its own start and drops its remainder; after a call of m < 10 decimated samples the filter's input
 *     history takes the call's first m undecimated samples, replaygain_analysis.c:502-506). Values are bit for bit metaflac's for
 *     every blocksize and rate.
 *  3. Writes (not with scan_only): per file, the metaflac chain rules: the first VORBIS_COMMENT, or a new one with this library's
 *     vendor string appended after the last block; the reference loudness, track and album edits (the entries of each name go,
 *     compared without ASCII case, then "REPLAYGAIN_REFERENCE_LOUDNESS=89.0 dB", "..._GAIN=%+2.2f dB", "..._PEAK=%1.8f" are
 *     appended); every PADDING block moved to the end and merged (FLAC__metadata_chain_sort_padding); then one chain write with
 *     padding (a grown list uses up or trims the last PADDING when that is large enough, a shrunk one extends it or gains a new
 *     PADDING from 4 bytes on). A file whose new blocks do not fit a block length fails that chain write: METADATA, its
 *     album's earlier files are written, its later ones are NOT_WRITTEN.
 * Before step 1, as metaflac reads every file's metadata chain first, a file the chain read refuses (a block running past the file,
 * a SEEKTABLE whose length is not a multiple of 18, a VORBIS_COMMENT whose fields run past the block, ...) is METADATA and fails
 * its album, in scan_only too.
 * A failed album's other files are ALBUM, `error` naming the failing file by its place in files[].
 *
 * New file = head + input[audio_offset_in ..]: the bytes before the first block (an ID3v2 tag, "fLaC"), the new blocks, then the
 * input's bytes after its metadata. in_place: the metadata length is unchanged (metaflac rewrites the head only).
 * whole_files 0: out gets each written file's head, back to back in list order; 1: the complete files. Files not written get
 * 0 bytes. info[i].rg holds the values the tags print for every file of an album that passed steps 1 and 2.
 *
 * FB200_ERR_INVALID before any launch: no resident batch, an index out of range or listed twice, a non-zero reserved, NULL
 * pointers. FB200_ERR_OUTPUT_TOO_SMALL before any launch when out_capacity is below the sum over the listed files the index passed
 * of their input bytes (whole_files) or their bytes before the first frame (heads), plus FB200_ADD_REPLAYGAIN_GROWTH each; 0 is
 * enough with scan_only.
 * Known differences from metaflac:
 *  - a 25-32-bit input is INPUT (the decoder stops at 24 bits);
 *  - a frame that runs past STREAMINFO's total_samples is DECODE;
 *  - a frame whose blocksize exceeds STREAMINFO's max_blocksize is not indexed, so its file is DECODE (its bytes are not
 *    covered), where libFLAC decodes it;
 *  - the frame decoder accepts some tiny frames libFLAC reports as lost sync (seen with a 2-sample variable-blocksize frame of
 *    FIXED and LPC order-1 subframes at partition order 1), so such a file is tagged where metaflac refuses it;
 *  - a CUESHEET or PICTURE whose body is not exactly its fields is METADATA (metaflac's reader reads the fields and goes on
 *    from there).
 * _host: one device-to-host copy of out. _device: out is device memory on the decoder's device, enqueued on cuda_stream; returns
 * after completion. The launch count does not depend on the number of files. */
#define FB200_ADD_REPLAYGAIN_GROWTH 256u  /* >= a new VORBIS_COMMENT: 4 + 4 + vendor (47) + 4 + the five longest entries (189) */
typedef struct {
	uint32_t scan_only;    /* non-zero: --scan-replay-gain, values only, nothing written */
	uint32_t whole_files;  /* non-zero: out gets the complete files, else the heads */
	uint32_t reserved;     /* must be 0 */
} fb200_add_replaygain_options;
enum { FB200_ADD_RG_OK = 0, FB200_ADD_RG_INPUT = 1, FB200_ADD_RG_FORMAT = 2, FB200_ADD_RG_DECODE = 3, FB200_ADD_RG_ALBUM = 4,
       FB200_ADD_RG_METADATA = 5, FB200_ADD_RG_NOT_WRITTEN = 6 };
typedef struct {
	uint32_t status;              /* FB200_ADD_RG_* */
	uint32_t album;
	char     error[88];
	fb200_replaygain_info rg;
	uint64_t offset, bytes;       /* in out */
	uint64_t head_bytes;          /* prefix + "fLaC" + blocks of the new file */
	uint64_t audio_offset_in;     /* the input's first byte after its metadata */
	uint32_t in_place, pad;
} fb200_add_replaygain_info;
int fb200_add_replaygain_flac_files_host(fb200_decoder *dec, const uint32_t *files, const uint32_t *albums, uint32_t nfiles,
                                         const fb200_add_replaygain_options *opt, uint8_t *out, size_t out_capacity,
                                         fb200_add_replaygain_info *info);
int fb200_add_replaygain_flac_files_device(fb200_decoder *dec, const uint32_t *files, const uint32_t *albums, uint32_t nfiles,
                                           const fb200_add_replaygain_options *opt, uint8_t *d_out, size_t out_capacity,
                                           fb200_add_replaygain_info *info, void *cuda_stream);
/* The host half, device-free: the new head of one .flac file (file[0 .. nbytes), at least its metadata) with these four values, as
 * step 3 above writes it. FB200_ERR_INVALID with fb200_last_error when metaflac's chain read or write would refuse the file;
 * FB200_ERR_OUTPUT_TOO_SMALL when the head is longer than head_capacity (*head_bytes still set). */
int fb200_replaygain_rewrite_head(const uint8_t *file, uint64_t nbytes, float track_gain, float track_peak, float album_gain, float album_peak,
                                  uint8_t *head, uint64_t head_capacity, uint64_t *head_bytes, uint64_t *audio_offset_in, uint32_t *in_place);
/* Test hook: every window's mean square of the listed files' analysis (as fb200_debug_replaygain_windows gives them), album by
 * album in ascending id, file after file in list order within one, for the albums that pass steps 1 and 2. */
int fb200_debug_add_replaygain_windows(fb200_decoder *dec, const uint32_t *files, const uint32_t *albums, uint32_t nfiles,
                                       double *windows, uint64_t capacity, uint64_t *nwindows);

/* ---- verify (flac -V, FLAC__stream_encoder_set_verify, stream_encoder.c:5186-5231) ----
 * With verify on, fb200_encode_files_host / _device decode every frame they encode on the device, from the frame bytes alone
 * (none of the encoder's decisions are used), and compare it with the input. A frame passes when it decodes with exact frame
 * bounds, CRC-8 and CRC-16 are good, its header agrees with the encoder's channels, bits per sample and sample rate, its coded
 * frame number is its index in its file, its blocksize is the block's length (the configured blocksize, or the file's tail
 * length), and every decoded sample equals the input value at its place. The input compared against is the engine's widened,
 * range-checked int32 copy of the caller's samples (the values the encode and the MD5 read), not the caller's packed bytes.
 *
 * Output, frame offsets, *nframes and files[] are filled exactly as with verify off. If any file fails, the call returns
 * FB200_ERR_VERIFY after filling all of them. FB200_ERR_INVALID and FB200_ERR_OUTPUT_TOO_SMALL keep their meaning and
 * precedence; such a call produces no verify records. With verify on, the block entry points (fb200_encode_host,
 * fb200_encode_host_packed, fb200_encode_device) fail with FB200_ERR_UNSUPPORTED: they never return frames that were not checked.
 *
 * One record per file describes its first failing frame in file order, the frame the reference's verify stops at: a decode or
 * header failure gives DECODER_ERROR (it wins over a sample mismatch in the same frame); otherwise MISMATCH reports the
 * lowest channel with a mismatch and that channel's first mismatching sample (channel first, as stream_encoder.c:5203-5212),
 * with absolute_sample / frame_number / expected / got as FLAC__stream_encoder_get_verify_decoder_error_stats (:2334). */
enum { FB200_VERIFY_OK = 0, FB200_VERIFY_DECODER_ERROR = 1, FB200_VERIFY_MISMATCH = 2 };
/* frame_status of a DECODER_ERROR beyond the fb200_decoder_get_frame_status codes (1-8): the coded frame number or blocksize
 * is not this frame's */
#define FB200_VERIFY_WRONG_FRAME 10
typedef struct {
	uint32_t status;           /* FB200_VERIFY_* */
	uint32_t frame_number;     /* first failing frame: its number in the file */
	uint32_t frame_status;     /* DECODER_ERROR: fb200_decoder_get_frame_status low-byte code, or FB200_VERIFY_WRONG_FRAME */
	uint32_t channel, sample;  /* MISMATCH: channel, sample within the frame */
	uint32_t reserved;
	uint64_t absolute_sample;  /* MISMATCH: frame_number * blocksize + sample, from the file's start */
	int32_t  expected, got;    /* MISMATCH: input value, decoded value */
} fb200_file_verify_info;
int fb200_encoder_set_verify(fb200_encoder *enc, int on);  /* default off */
/* The per-file records of the last fb200_encode_files_* call. FB200_ERR_INVALID if that call did not verify (verify off, or it
 * failed before verifying) or nfiles differs from its file count. */
int fb200_encoder_get_verify(const fb200_encoder *enc, fb200_file_verify_info *info, uint32_t nfiles);

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
/* Stage A (the windowed FP64 autocorrelation) of the most recent encode call's first nblocks blocks, all of the configured
 * blocksize, for tests that compare the kernels' sums with the reference's. The call's blocks must have fitted one workspace set
 * (at most max_blocks_per_launch frames) and its full blocks must have taken one route; otherwise FB200_ERR_INVALID. info gets
 * the section count, the LPC lag count, the lags the kernel computes and writes (kernel_lags), the record stride and the route
 * (FB200_STAGE_A_*). With autoc == NULL nothing else is read. Otherwise, with item = block * nsig + signal:
 *   autoc[(sec * nitems + item) * lag_stride + l], l < kernel_lags: the records as written -- on the fused route the sums of the
 *     signal before its wasted bits are shifted out, on the others after; records of items with subframe bps 0 (the pair a loose
 *     mid-side block does not code) are not written;
 *   meta[2 * item], meta[2 * item + 1]: wasted bits and subframe bps;
 *   sigor[item]: the OR of the signal's samples (fused route only; left untouched on the others);
 *   sections[5 * sec ..]: window offset, partial, data_len, part_size and data_shift of each section (fb200::DevSection).
 * The encode itself records only the route and block range of each chunk on the host for this: no launch, synchronisation or
 * device allocation. */
enum { FB200_STAGE_A_FUSED = 0, FB200_STAGE_A_META = 1, FB200_STAGE_A_PLANAR = 2 };
typedef struct {
	uint32_t nsec, lags, kernel_lags, lag_stride;
	int32_t route;
} fb200_debug_autoc_info;
int fb200_debug_copy_autoc(fb200_encoder *enc, uint32_t nblocks, double *autoc, size_t autoc_doubles, int32_t *meta, uint32_t *sigor,
                           int32_t *sections, uint32_t max_sections, fb200_debug_autoc_info *info);
/* Verify tests: for the next fb200_encode_files_* call only, XOR xor_mask into a buffer the engine owns after the frames are
 * encoded and before they are verified. what = 0: byte b of frame a of file `file` in the encode scratch (the output is not
 * touched; a byte past the frame is left alone); what = 1: the value (sample a, channel b) of that file's int32 copy of the
 * input. Several calls queue several flips. That next call fails with FB200_ERR_INVALID if a flip names a file, frame or
 * sample it does not have, or if it computes MD5 (the MD5 reads the same copy concurrently). */
int fb200_debug_perturb_verify(fb200_encoder *enc, uint32_t file, uint32_t what, uint32_t a, uint32_t b, uint32_t xor_mask);
/* y[i] = the engine's device restatement of the host libm's log(x[i]) (reference: lpc.c:1594, fixed.c:284). */
int fb200_debug_log(const double *x, double *y, uint32_t n, int device);
/* The encoder's LPC analysis kernel (Levinson-Durbin, order guess, precision loop, quantisation, residual-width flags) on
 * caller-supplied autocorrelations, with the kernel instantiation the encoder takes for max_order (8, 12 or 32).
 * autoc: nsec x nitems records of lag_stride doubles, record (sec, item) at (sec * nitems + item) * lag_stride, entries
 * [0 .. max_order] used. meta: per item (wasted bits, subframe bps). cands: per window (kind, sec, root); kind 1 is a punch-out
 * window, autoc[sec, root][l] - autoc[sec][l] for l < max_order. autoc_unshifted: the records are of the signal before its
 * wasted bits were shifted out. out: nitems x *nslots_out records of cand_bytes (fb200::CandDesc,
 * flac_b200/csrc/fb200_internal.h), window w's slots from w * (*nslots_out / nwin). */
/* The general search kernel's evaluation of one LPC candidate (residual -- 32-bit, 64-bit or checked as its wide / limit flags
 * say --, partition sums, Rice parameters, bit estimate) on each of n signals of blocksize samples: signal i is
 * signals[i * blocksize ..], meta[i] its (wasted bits, subframe bps), cands[i] an fb200::CandDesc (cand_bytes each). est[i] is
 * the estimate, 0xffffffff when the candidate is rejected (a checked residual outside int32). */
int fb200_debug_evaluate_lpc(int device, const int32_t *signals, const int32_t *meta, const void *cands, size_t cand_bytes, uint32_t n,
                             uint32_t blocksize, uint32_t min_po, uint32_t max_po, uint32_t rice_limit, uint32_t *est);
int fb200_debug_lpc(int device, const double *autoc, uint32_t nsec, uint32_t lag_stride, const int32_t *meta, const int32_t *cands,
                    uint32_t nwin, uint32_t nitems, uint32_t max_order, uint32_t qlp_precision, int prec_search, int exhaustive,
                    uint32_t blocksize, int autoc_unshifted, void *out, size_t cand_bytes, uint32_t *nslots_out);

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

/* ---- batches of whole .flac files ----
 * fb200_decode_files_index parses nfiles .flac files, file f = data[file_offsets[f], file_offsets[f + 1]), copies the batch to
 * the device once and indexes every file's frames; the batch stays resident for any number of decode calls until the next
 * index call. Files may mix channel counts (1-8), bit depths (4-24) and sample rates; the decoder's fb200_decoder_config is
 * not consulted, only its device and max_frames_per_launch. A file that cannot be decoded never fails the call: it gets a
 * status, 0 samples, and is skipped.
 *
 * Frames of a file: the headers found in its audio that agree with its STREAMINFO (channels, bits per sample, blocksize <=
 * max_blocksize), each bounded by its own file's end. A frame is accepted when it decodes (CRC-16 included) and begins at or
 * after the end of the file's previous accepted frame; a failed frame past that point starts a damaged stretch (`errors`
 * counts stretches). A frame's first sample is frame number x blocksize when STREAMINFO min == max blocksize, else the coded
 * sample number; a frame-number-coded frame with min != max is not accepted. An accepted frame whose samples overlap the
 * previous placed frame's counts as an error and is not placed.
 *
 * Output: the files back to back in file order, each interleaved with its own channel count and `samples` long (STREAMINFO's
 * total_samples; when that is 0, the end of the file's last frame header found). Frames are cut at `samples`; samples that no
 * accepted frame covers are zero. A lost frame in the middle of a file is therefore silence, as the reference delivers it
 * (stream_decoder.c:2483-2554), with one difference: the reference writes at most 50 of the previous frame's blocks or 5
 * seconds of silence, whichever is less, and then the next frame early, while here every frame stays at its sample number, so
 * a longer gap is all zeros and the file keeps its length. A lost first or last frame keeps the file's length, where the
 * reference delivers a shorter stream. Other known differences from libFLAC on damaged files:
 *  - header_disagrees: a frame whose channels, bits per sample or blocksize disagree with STREAMINFO is not indexed, so its
 *    samples are lost; libFLAC decodes and writes it.
 *  - overlap: a frame that starts before the end of the frame placed before it (a repeated or reordered frame) is not
 *    placed, its samples are zeros unless another frame covers them, and it counts as an error; libFLAC writes every frame in
 *    stream order.
 *  - lost_without_candidate: `errors` counts damaged stretches the index found a candidate in; a frame lost with its header
 *    (a damaged header, or frames cut out) shows only in samples_missing, where libFLAC reports lost sync, a bad header or a
 *    missing frame.
 *  - trailing_junk: the drop-in decoder reports nothing for bytes after the last frame (an ID3v1 or APE tag); libFLAC
 *    reports them as lost sync.
 *  - junk: junk that carries no frame header (and ID3v1 / APE tags) is never seen by the index; libFLAC reports it as lost
 *    sync.
 * With do_md5, each decoded file's MD5 (its samples as (bps + 7) / 8-byte little-endian integers, md5.c:280-521) is
 * computed on the device and compared with STREAMINFO's; an all-zero STREAMINFO MD5 is not checked.
 *
 * Candidates are decoded into a scratch of at most FB200_DECODE_FILES_SAMPLE_BUDGET samples (all channels, int32) per launch
 * set, so device memory beyond the batch, the index and the output does not grow with the batch. The per-frame status of
 * fb200_decoder_get_frame_status is left as the last frame-level call set it. */
#define FB200_DECODE_FILES_SAMPLE_BUDGET (1u << 27)
enum {
	FB200_FILE_OK = 0,
	FB200_FILE_NOT_FLAC = 1,          /* no "fLaC" after an optional ID3v2 tag, or metadata that runs past the file */
	FB200_FILE_NO_STREAMINFO = 2,
	FB200_FILE_BAD_STREAMINFO = 3,    /* length != 34, blocksizes < 16 or min > max, sample rate 0, bits per sample < 4 */
	FB200_FILE_UNSUPPORTED = 4,       /* bits_per_sample > 24 */
	FB200_FILE_WIDTH = 5,             /* bits_per_sample does not fit the host call's bytes_per_sample (decode call) */
	FB200_FILE_TOO_BIG = 6,           /* fb200_decode_pcm_files_*: the flac tool refuses this container kind for this length */
	FB200_FILE_NO_TOTAL = 7           /* fb200_decode_pcm_files_* with ranges: STREAMINFO total_samples is 0 (no --skip / --until) */
};
typedef struct {
	uint32_t status;          /* FB200_FILE_* */
	uint32_t channels, bits_per_sample, sample_rate, min_blocksize, max_blocksize;  /* from STREAMINFO */
	uint64_t total_samples;   /* STREAMINFO's value (0 = unknown) */
	uint64_t samples;         /* samples per channel this file occupies in the output */
	uint64_t first_value;     /* index of the file's first value in the output (sum of samples * channels of the files before) */
	uint32_t nframes;         /* frames accepted (decode call) */
	uint32_t errors;          /* damaged stretches + overlapping frames (decode call) */
	uint64_t samples_missing; /* samples of [0, samples) that no accepted frame covered; left zero (decode call) */
	int32_t  md5_state;       /* 0 not checked (off, or STREAMINFO MD5 all zero), 1 matches, 2 differs (decode call) */
	uint8_t  md5[16];         /* computed over the output as placed, when checked */
} fb200_file_decode_info;

/* files[nfiles] receives the STREAMINFO facts, status, samples and first_value; *total_values = the output's length in values. */
int fb200_decode_files_index(fb200_decoder *dec, const uint8_t *data, uint64_t nbytes, const uint64_t *file_offsets, uint32_t nfiles,
                             fb200_file_decode_info *files, uint64_t *total_values);
/* Decodes the resident batch into host memory as packed little-endian PCM of bytes_per_sample 2, 3 or 4 bytes (a file deeper
 * than that gets FB200_FILE_WIDTH and zeros). The batch is decoded, then narrowed and copied back; copies do not overlap
 * compute. files[nfiles] is filled completely. pcm_capacity_values < total_values fails with FB200_ERR_OUTPUT_TOO_SMALL
 * before anything is written; without a resident index the call fails with FB200_ERR_INVALID. */
int fb200_decode_files_host(fb200_decoder *dec, void *pcm, uint32_t bytes_per_sample, uint64_t pcm_capacity_values, int do_md5,
                            fb200_file_decode_info *files);
/* The same into int32 device memory on the decoder's device, enqueued on cuda_stream; returns after completion. */
int fb200_decode_files_device(fb200_decoder *dec, int32_t *d_pcm, uint64_t pcm_capacity_values, int do_md5, fb200_file_decode_info *files,
                              void *cuda_stream);

/* ---- sample ranges of the indexed batch (flac -d --skip / --until over many files; random crops for a data loader) ----
 * fb200_decode_files_ranges_* decode samples [first_sample, first_sample + samples) per channel of files of the batch left
 * resident by fb200_decode_files_index, without decoding the rest of each file. The ranges go to the output back to back in
 * request order, each interleaved with its file's channel count. A range may name any file any number of times; ranges may
 * overlap and come in any order (each decodes its own frames: frames shared by overlapping ranges are decoded once per range).
 *
 * The whole call fails with FB200_ERR_INVALID, before any work, without a resident index, for nranges 0 or >= 2^31, a file
 * index >= nfiles, samples 0, first_sample + samples overflowing, or -- for a file with status FB200_FILE_OK -- a range that
 * runs past the file's `samples` (as with flac --until, that is an error, not a clamp). A range over a file whose status is not
 * OK gets that status and 0 values, and the call goes on; with _host, so does a file deeper than 8 * bytes_per_sample
 * (FB200_FILE_WIDTH). *total_values and info[r]'s status, channels, bits_per_sample, first_value and values are filled before
 * the capacity check: pcm_capacity_values < *total_values fails with FB200_ERR_OUTPUT_TOO_SMALL and writes nothing, so a call
 * with capacity 0 (pcm may then be NULL) sizes the output.
 *
 * Frames of a range: the candidates of its file (see the frame rules above) whose samples [first, first + blocksize) meet the
 * range, walked in byte order. One is accepted when it decodes and begins at or after the end of the range's previous accepted
 * candidate; an accepted frame overlapping the previous placed one is not placed; the part of each placed frame inside the
 * range is copied, and samples no accepted frame covers are zero (samples_missing). So a range's output equals the same slice
 * of fb200_decode_files_* output whenever no false header candidate passes CRC-16, and a lost frame inside a range is silence.
 * Known divergence (range_sees_its_frames): a range walks only the frames that meet it, so a frame the whole-file decode drops
 * because an earlier frame in the file ends past its first sample (swapped or moved frames) is placed by a range that does not
 * meet that earlier frame.
 * No MD5 is computed (the reference turns MD5 checking off after a seek). The resident index is not changed: decode_files_*
 * afterwards returns what it returned before; the next index call replaces the batch for both. The per-frame status of
 * fb200_decoder_get_frame_status is left untouched. */
typedef struct {
	uint32_t status;          /* FB200_FILE_* of the range's file; FB200_FILE_WIDTH as in fb200_decode_files_host */
	uint32_t channels, bits_per_sample;
	uint32_t nframes;         /* frames accepted for this range (each placed samples into it unless it overlapped the previous) */
	uint64_t first_value;     /* where the range starts in the output */
	uint64_t values;          /* samples * channels; 0 when status != FB200_FILE_OK */
	uint64_t samples_missing; /* samples of the range that no accepted frame covered (left zero) */
	uint64_t candidates;      /* candidate frames decoded for this range (>= nframes; diagnostic) */
} fb200_range_decode_info;
/* Packed little-endian PCM of bytes_per_sample 2, 3 or 4 bytes into host memory; decoded, narrowed and copied back. */
int fb200_decode_files_ranges_host(fb200_decoder *dec, const fb200_sample_range *ranges, uint32_t nranges,
                                   void *pcm, uint32_t bytes_per_sample, uint64_t pcm_capacity_values,
                                   uint64_t *total_values, fb200_range_decode_info *info);
/* int32 into device memory on the decoder's device, enqueued on cuda_stream; returns after completion. */
int fb200_decode_files_ranges_device(fb200_decoder *dec, const fb200_sample_range *ranges, uint32_t nranges,
                                     int32_t *d_pcm, uint64_t pcm_capacity_values,
                                     uint64_t *total_values, fb200_range_decode_info *info, void *cuda_stream);

/* ---- the indexed batch as WAV / RF64 / Wave64 / AIFF / AIFF-C files (flac -d *.flac) ----
 * fb200_decode_pcm_files_* decode the batch left resident by fb200_decode_files_index into the container files the flac tool
 * 1.5.0 writes (src/flac/decode.c): the header of write_iff_headers (:718-989), the samples as write_callback stores them
 * (:1245-1632: shifted left into (bps + 7) / 8 bytes, unsigned 8-bit and little-endian for WAVE / RF64 / Wave64, signed and
 * big-endian for AIFF and AIFF-C NONE, little-endian for AIFF-C sowt) and the pad byte(s) after the data (:551-574). Each file
 * comes out at its own width and in its own layout; the containers go to the output back to back.
 *
 * ranges == NULL: one container per indexed file, in file order (flac -d). Otherwise one per range, in request order (flac -d
 * --skip=first_sample --until=first_sample+samples), validated as fb200_decode_files_ranges_* validate them; a range over a file
 * whose STREAMINFO total_samples is 0 gets FB200_FILE_NO_TOTAL (the tool refuses --skip / --until there). A container's sample
 * count is the file's `samples` (fb200_file_decode_info) or the range's. When total_samples is 0 the tool writes the header
 * after decoding, with the decoded count, and writes no pad byte (it sizes the pad from total_samples); so does this call.
 *
 * The channel mask: the value of the first WAVEFORMATEXTENSIBLE_CHANNEL_MASK entry (name matched case-insensitively) of a
 * VORBIS_COMMENT block, when it is at least 4 bytes longer than the name and its value starts with "0x" (either case) that
 * sscanf("%x") reads (flac__utils_get_channel_mask_tag, utils.c:474-493); a later block with such a tag overrides an earlier
 * one. Without one, the tool's default for the channel count (decode.c:429-454); channel_map_none: 0 (the tool then reads no
 * VORBIS_COMMENT). EXTENSIBLE is written when forced, or for WAVE / RF64 / Wave64 unless legacy is forced when the mask is not
 * 0, 3 or 4, bps is not 8 or 16, or there are more than 2 channels.
 *
 * Every container's length is known before any device work: *total_bytes and every info[] field but nframes, errors,
 * samples_missing, md5_state, md5 and tool_ok are filled before the capacity check, and out_capacity < *total_bytes fails with
 * FB200_ERR_OUTPUT_TOO_SMALL having written nothing, so a call with capacity 0 (out may be NULL) sizes the output. A file that
 * is not OK (FB200_FILE_* of the index call), 32-bit, or too big for the kind (FB200_FILE_TOO_BIG: RIFF / FORM size >=
 * 0xFFFFFFF4 for WAVE, AIFF and AIFF-C, where the tool stops with "stream is too big") gets 0 bytes, and the call goes on.
 *
 * tool_ok is 1 when the tool would exit 0 and keep the file: no damaged stretch (errors 0), no sample missing, and (with md5,
 * whole files only) no MD5 mismatch; without -F the tool deletes the file on any decoder error. The bytes are written either way,
 * a lost frame as silence. Known divergence: junk that carries no frame header is never seen by the engine, while the tool
 * reports it as lost sync and refuses the file.
 *
 * Samples are decoded into the decoder's int32 scratch by the paths of fb200_decode_files_* and fb200_decode_files_ranges_*,
 * then one k_pcm_pack launch writes every container (headers, data and pad bytes) whatever the kinds and widths; launches do not
 * grow with the number of files. _host: packed on the device, then one device-to-host copy. _device: d_out is device memory on
 * the decoder's device, any alignment; ranges, info and total_bytes are host memory. Both return after completion. */
enum { FB200_PCM_SUB_AUTO = 0, FB200_PCM_SUB_WAVE_PCM = 1, FB200_PCM_SUB_WAVE_EXTENSIBLE = 2,
       FB200_PCM_SUB_AIFF_C_NONE = 3, FB200_PCM_SUB_AIFF_C_SOWT = 4 };
typedef struct {
	uint32_t kind;              /* FB200_PCM_WAVE .. FB200_PCM_AIFF_C (the probe's enum) */
	uint32_t subformat;         /* FB200_PCM_SUB_*: WAVE takes AUTO, WAVE_PCM (--force-legacy-wave-format) or WAVE_EXTENSIBLE
	                               (--force-extensible-wave-format); AIFF_C needs AIFF_C_NONE or AIFF_C_SOWT; the other kinds AUTO.
	                               A mismatched pair is FB200_ERR_INVALID */
	uint32_t md5;               /* check each whole file's MD5 (the tool always does); ignored for ranges */
	uint32_t channel_map_none;  /* --channel-map=none */
} fb200_pcm_decode_options;
typedef struct {
	uint32_t status;            /* FB200_FILE_* of the source file, or FB200_FILE_TOO_BIG / FB200_FILE_NO_TOTAL */
	uint32_t tool_ok;           /* 1 when the flac tool would exit 0 and keep this file (see above) */
	uint32_t channels, bits_per_sample, container_bits, sample_rate;
	uint32_t channel_mask;      /* the mask the header carries (tag, default or 0) */
	uint32_t extensible;        /* 1: WAVE_FORMAT_EXTENSIBLE */
	uint32_t header_bytes;      /* where the data begins in the container */
	uint32_t reserved;
	uint64_t offset, bytes;     /* where this container starts in the output, and its length (0 when status != OK) */
	uint64_t samples;           /* samples per channel in the container */
	uint64_t samples_missing;   /* of those, samples no accepted frame covered (written as zeros) */
	uint32_t nframes, errors;   /* frames accepted; damaged stretches + overlapping frames */
	int32_t  md5_state;         /* as fb200_file_decode_info (0 for ranges) */
	uint8_t  md5[16];
} fb200_pcm_decode_info;
int fb200_decode_pcm_files_host(fb200_decoder *dec, const fb200_pcm_decode_options *opt,
                                const fb200_sample_range *ranges, uint32_t nranges,
                                uint8_t *out, uint64_t out_capacity, uint64_t *total_bytes, fb200_pcm_decode_info *info);
int fb200_decode_pcm_files_device(fb200_decoder *dec, const fb200_pcm_decode_options *opt,
                                  const fb200_sample_range *ranges, uint32_t nranges,
                                  uint8_t *d_out, uint64_t out_capacity, uint64_t *total_bytes, fb200_pcm_decode_info *info,
                                  void *cuda_stream);
/* ---- the same containers with ReplayGain applied (flac -d --apply-replaygain-which-is-not-lossless[=SPEC]) ----
 * fb200_decode_pcm_files_replaygain_* write what fb200_decode_pcm_files_* write (same lengths, headers, pad bytes, statuses,
 * tool_ok and MD5 of the decoded samples before gain), except that the samples of each container the tool applies gain to are
 * those of FLAC__replaygain_synthesis__apply_gain (src/share/replaygain_synthesis/replaygain_synthesis.c): scaled, optionally
 * hard-limited (glibc tanh restated bit for bit), re-quantised to the container's width, with noise-shaped triangular dither
 * for noise_shaping 1-3. The decision per file follows the tool's metadata callback (decode.c:1775-1820,
 * grabbag/replaygain.c:582-669): names matched without case, values read by strtod in the C locale from the first
 * min(31, length - 1) characters after '=' (parse_double_'s safe_strncpy drops the last one), a negative peak fails the pair, a
 * failed pair retries the other mode, and the last VORBIS_COMMENT block decides. Then bits per sample outside 4-24 is BPS,
 * |gain| > 90 is GAIN, no usable pair is NO_TAGS, and the container is decoded plainly.
 *
 * The dither generator of the tool (random_int_) is process-global: its state runs on from file to file of one invocation.
 * Whole files with per_file 0 reproduce one invocation over the listed files in order; per_file 1 and every range reproduce one
 * invocation per container. A file draws 2 x channels numbers per sample the tool writes before its first decode error (the
 * write callback aborts there); rginfo[i].first_draw / draws say where each container's draws lie. The engine still writes a
 * damaged file in full with tool_ok 0, its samples after the error dithered with draws that follow on. Known difference: the
 * first error is taken to be the first sample no accepted frame covers, so a damaged stretch that loses no samples (junk
 * between frames) does not end a file's draws as it ends the tool's. */
enum { FB200_RGS_LIMIT_NONE = 0, FB200_RGS_LIMIT_PEAK = 1, FB200_RGS_LIMIT_HARD = 2 };
typedef struct {
	double   preamp;         /* dB */
	uint32_t album;          /* 1: album gain and peak (falls back to track); 0: track (falls back to album) */
	uint32_t limiter;        /* FB200_RGS_LIMIT_* */
	uint32_t noise_shaping;  /* 0: no dither; 1-3: low / medium / high (triangular dither, 16-tap shaping filter) */
	uint32_t per_file;       /* whole files: 0 = the list is one invocation, 1 = one invocation per file; ranges: always per range */
} fb200_replaygain_synthesis;
/* The tool's parse of SPEC (main.c:767-790); spec NULL: the option without '=' (album, hard limiter, low shaping, preamp 0).
 * FB200_ERR_INVALID where the tool prints a usage error. per_file is set to 0. */
int fb200_replaygain_synthesis_parse(const char *spec, fb200_replaygain_synthesis *rg);
enum { FB200_RGS_APPLIED = 0, FB200_RGS_NO_TAGS = 1, FB200_RGS_BPS = 2, FB200_RGS_GAIN = 3, FB200_RGS_NOT_DECODED = 4 };
typedef struct {
	uint32_t status;                 /* FB200_RGS_*: the tool's decision; not APPLIED = the plain decode's bytes */
	uint32_t album_used;             /* which tag pair gave gain and peak after the fallback */
	double   reference, gain, peak;  /* as parsed */
	double   scale;                  /* grabbag__replaygain_compute_scale_factor */
	uint64_t first_draw, draws;      /* the generator's position at the container's first sample, and the draws the tool makes for it */
} fb200_replaygain_synthesis_info;
/* Device-free: the decision and the scale for one .flac from its metadata; first_draw and draws are left 0. */
int fb200_replaygain_synthesis_file(const uint8_t *file, uint64_t nbytes, const fb200_replaygain_synthesis *rg,
                                    fb200_replaygain_synthesis_info *info);
/* As fb200_decode_pcm_files_host / _device, with rginfo[n] (one per container) filled before the capacity check. Containers
 * that are not decoded get FB200_RGS_NOT_DECODED. One k_rg_synth launch per call (two when both shaping 0 and 1-3 would run,
 * which one spec never asks for), whatever the number of files. */
int fb200_decode_pcm_files_replaygain_host(fb200_decoder *dec, const fb200_pcm_decode_options *opt, const fb200_replaygain_synthesis *rg,
                                           const fb200_sample_range *ranges, uint32_t nranges, uint8_t *out, uint64_t out_capacity,
                                           uint64_t *total_bytes, fb200_pcm_decode_info *info, fb200_replaygain_synthesis_info *rginfo);
int fb200_decode_pcm_files_replaygain_device(fb200_decoder *dec, const fb200_pcm_decode_options *opt, const fb200_replaygain_synthesis *rg,
                                             const fb200_sample_range *ranges, uint32_t nranges, uint8_t *d_out, uint64_t out_capacity,
                                             uint64_t *total_bytes, fb200_pcm_decode_info *info, fb200_replaygain_synthesis_info *rginfo,
                                             void *cuda_stream);
/* Debug: y[i] = the device restatement of the host libm's tanh(x[i]) (the hard limiter's). */
int fb200_debug_tanh(const double *x, double *y, uint32_t n, int device);
/* Debug: apply_gain on constructed input. `in`: channels x samples int32 values, interleaved; `blocks`: nblocks lengths summing to
 * samples, the lengths the write callback would receive; the generator starts at draw first_draw. bps 4-24 is the source
 * width; the target is the container's, 8 x ((bps + 7) / 8). scale, limiter (hard or not) and noise_shaping as the tool uses them.
 * out: the val32 of every value (interleaved), before byte packing. */
int fb200_debug_replaygain_synthesis(int device, const int32_t *in, uint32_t channels, uint64_t samples, const uint32_t *blocks, uint32_t nblocks,
                                     uint32_t bps, double scale, uint32_t hard_limit, uint32_t noise_shaping, uint64_t first_draw, int32_t *out);

/* Device-free: the header the tool writes for these facts into out[0 .. *length), *length being where the data begins.
 * channel_mask: the tag's value (0: none; the default for the channel count then applies), ignored with channel_map_none.
 * channels 1-8, bits_per_sample 4-32, else FB200_ERR_INVALID; FB200_ERR_UNSUPPORTED (*length 0) where the tool refuses the
 * kind for this length; FB200_ERR_OUTPUT_TOO_SMALL (*length set) when capacity < *length. 128 bytes always suffice. */
int fb200_pcm_header(const fb200_pcm_decode_options *opt, uint32_t channels, uint32_t bits_per_sample, uint32_t sample_rate,
                     uint32_t channel_mask, uint64_t samples, uint8_t *out, uint32_t capacity, uint32_t *length);

enum { FB200_DPROF_WALK = 0, FB200_DPROF_CRC, FB200_DPROF_FRAMES, FB200_DPROF_KERNELS };  /* k_dec_walk, k_dec_crc, k_dec_frames */
int fb200_decoder_set_profiling(fb200_decoder *dec, int on);
int fb200_decoder_get_profile(fb200_decoder *dec, double ms[FB200_DPROF_KERNELS], uint64_t launches[FB200_DPROF_KERNELS], int reset);

#ifdef __cplusplus
}
#endif
#endif /* FLAC_B200_H */
