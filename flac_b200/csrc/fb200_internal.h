// fb200_internal.h -- shared declarations for the libflac_b200.so translation units.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "../../include/flac_b200.h"

namespace fb200 {

void set_error(const char *fmt, ...);
const char *get_error();

#define FB_CUDA(call)                                                                              \
	do {                                                                                           \
		cudaError_t e_ = (call);                                                                   \
		if(e_ != cudaSuccess) {                                                                    \
			fb200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
			return FB200_ERR_CUDA;                                                                 \
		}                                                                                          \
	} while(0)

// ---- FLAC bitstream constants (reference src/libFLAC/format.c:117-154) ----
constexpr uint32_t kSubframeHeaderBits = 8;  // zero pad 1 + type 6 + wasted flag 1
constexpr uint32_t kQlpPrecisionLen = 4, kQlpShiftLen = 5;
constexpr uint32_t kEntropyTypeLen = 2, kRiceOrderLen = 4;
constexpr uint32_t kRiceParamLen = 4, kRice2ParamLen = 5;
constexpr uint32_t kRiceEscape = 15, kRice2Escape = 31;
constexpr uint32_t kMaxFixedOrder = 4;
constexpr uint32_t kMinQlpPrecision = 5, kMaxQlpPrecision = 15;
constexpr int kQlpPrecisionSteps = 11;  // precisions a precision search tries per order: 5 .. 15
constexpr uint32_t kMaxExtraResidualBps = 4;  // private/stream_encoder.h:44
constexpr int kMaxPartitionOrder = 8;         // engine scope (-0..-8 use <= 6)
constexpr int kMaxPartitions = 1 << kMaxPartitionOrder;

// subframe types as stored in plans
enum : int { SF_CONSTANT = 0, SF_VERBATIM = 1, SF_FIXED = 2, SF_LPC = 3 };

// One autocorrelation "section" of a block: a full window or a partial (subdivide_tukey) window.
struct DevSection {
	int win_off;     // offset of the window table (floats) for this apodization
	int partial;     // 0: out[i]=x[i]*w[i], i<bs.  1: partial window (lpc.c:82-94)
	int data_len;    // samples the autocorrelation runs over
	int part_size;   // partial: half length
	int data_shift;  // partial: first sample
};

// One LPC candidate in evaluation order (stream_encoder.c:4318-4392).
struct DevCand {
	int kind;  // 0: autoc = section[sec]; 1: punch-out: autoc[i<max] = section[root][i]-section[sec][i], autoc[max] = section[sec][max]
	int sec;
	int root;
};

struct SigMeta {
	int wasted;
	int bps;  // subframe bps (after wasted bits, +1 for side)
};

// Output of the LPC analysis kernel for one candidate slot.
struct CandDesc {
	int valid;
	int order;
	int precision;
	int shift;
	int wide;   // needs 64-bit accumulation (FLAC__lpc_max_prediction_before_shift_bps > 32)
	int limit;  // residual range must be checked (FLAC__lpc_max_residual_bps > 32)
	int pad0, pad1;
	int qlp[FB200_MAX_LPC_ORDER];
};

// What the search kernel decides for one signal of one block.
struct SubframePlan {
	int type, order, wasted, bps;
	int precision, shift, method, porder;
	uint32_t est_bits;
	int wide;
	int pad0, pad1;
	int qlp[FB200_MAX_LPC_ORDER];
	uint8_t params[kMaxPartitions];
};

// Per-launch constants (passed by value to every kernel).
struct EncK {
	int channels, bps, sample_rate;
	int bs, bs_stride, nsig;
	int do_ms, loose_ms;
	int max_order;       // min(cfg.max_lpc_order, bs-1)
	int lags;            // max_order + 1
	int lag_stride;      // doubles per (section,item) autocorrelation record
	int qlp_precision, exhaustive;
	int prec_search;     // do_qlp_coeff_prec_search: every order is tried at precisions 5 .. 15 (stream_encoder.c:4230-4243)
	int min_po, max_po;  // resolved for this blocksize (stream_encoder.c:3759-3761)
	int rice_limit;      // 15 (stream bps <= 16) or 31 (stream_encoder.c:4076)
	int dis_const, dis_fixed, dis_verb;
	int nsec, nwin, nslots;
	int slot_stride;     // bytes per frame slot in the staging buffer (multiple of 16)
	int slot_words;
	int emit3_words;     // word-buffer capacity of k_emit3: the largest frame the search can produce (tighter than slot_words)
	uint32_t first_frame;  // frame number of the call's first block
	uint32_t blk0;         // index (inside the call) of this launch's first block
	int file_blocks;     // > 0: frame numbers restart every file_blocks blocks (many-file batches: one stream per file, stream_encoder.c:3772)
	const uint32_t *frame_no;  // non-null: block blk0 + i of the call is frame frame_no[blk0 + i] (fb200_encode_files_*); overrides the two above
	int limit_min_bitrate;  // stream_encoder.c:3874: a frame must not consist of constant subframes only
	int sig_group;       // k_search5: signals per CTA when a block's signals are split over several CTAs (0: one CTA per block)
	const int *redo;     // search kernels, second pass of limit_min_bitrate: only blocks with redo[blk] != 0, only signals >= channels - 1
	int x86_avx2_fixed_guess;  // fb200_encoder_config's: the general and tiled searches guess wide subframes' fixed order as x86 AVX2 libFLAC does
};

// ---- row layout shared by k_search5 and k_emit3: a signal lives in rows of R_T samples with a 36-word stride and one
// zero row in front (the history of row 0)
constexpr int kSearch4ZeroRow = 36;

// ---- k_emit3 (emit_kernel.cuh)
// device table of k_emit3's CRC-16 pass (uint16 entries): 4 x 256 slicing tables, combine multipliers x^(32 Lw 2^s) for odd
// Lw < 64 and s < 9, and their nibble-product tables
constexpr int kCrcLwRows = 32;
constexpr int kCrcMulBase = 1024 + kCrcLwRows * 9 + 32;
constexpr int kCrcTabEntries = kCrcMulBase + kCrcLwRows * 9 * 64;
constexpr unsigned kLbEpochMask = 0x3fffffu;  // decoupled look-back status word: value << 24 | epoch (22 bits) << 2 | flag
// Per-launch arguments of k_emit3 beyond EncK.
struct Emit3Args {
	const int32_t *pcm;                  // interleaved int32, block b at pcm + b * bs * channels
	const SigMeta *meta;                 // [nb * nsig]
	const int *blkflags;                 // [nb]
	const SubframePlan *plans;           // [nb * nsig]
	const uint16_t *crc_tab;             // 4 x 256
	uint8_t *out;
	unsigned long long out_cap;
	unsigned long long *offsets;         // offsets[0 .. nb] of this launch
	const unsigned long long *running_in;  // bytes emitted by earlier launches of the same call
	unsigned long long *running_out;
	unsigned long long *lookback;        // [>= nb] status words
	unsigned *ticket;                    // monotonically increasing across launches
	unsigned ticket_base;                // value of *ticket when this launch starts
	unsigned epoch;
	int nb;
	uint32_t *chan_assign_out;           // may be null
	int *err;
	// more than two channels: k_emit3<PAIR> packs channel pairs into staging regions, k_join splices them into frames
	uint32_t *stage;                     // [nb][npairs][pair_words]
	uint32_t *stage_bits;                // [nb][npairs] bits of each region (0xffffffff: the pair overflowed its region)
	int pair_words, join_words;
};

// Fixed-size shared state of one k_emit3 CTA (in front of the signal / word buffers).
struct Emit3Shared {
	unsigned long long mbar;
	unsigned long long off;      // this frame's byte offset in the output stream
	uint32_t scan[16];           // per-warp totals of the run scan
	uint32_t mlev[16];           // CRC combine multipliers x^(32 Lw 2^s)
	uint32_t part[16];           // per-warp CRC partials
	uint32_t hdr[4];             // frame header bytes (big-endian words, left aligned)
	int blk, zero_words, pad0, pad1;
	int warm[2][FB200_MAX_LPC_ORDER];  // the first 32 samples of each channel (warm-up samples / constant value)
};

__host__ __device__ inline size_t emit3_sig_bytes(int bs, int R_T, int nch)
{
	const size_t planar = (size_t)nch * (size_t)(kSearch4ZeroRow + (bs / R_T) * 36) * 4;
	const size_t raw = (size_t)bs * nch * 4;
	return ((planar > raw ? planar : raw) + 15) / 16 * 16;
}
__host__ __device__ inline size_t emit3_smem_bytes(int bs, int R_T, int nch, int slot_words)
{
	return (sizeof(Emit3Shared) + 15) / 16 * 16 + emit3_sig_bytes(bs, R_T, nch) + (size_t)(slot_words + 8) * 4;
}


// ---- launchers (one translation unit per kernel family; encoder.cu holds no device code)
// general_kernels.cu
void launch_unpack(const void *packed, int bytes_per_sample, int32_t *pcm, unsigned long long n, int bps, int *err, cudaStream_t st);
void launch_meta(const EncK &k, const int32_t *pcm, SigMeta *meta, int *blkflags, int nb, cudaStream_t st);
void launch_prep(const EncK &k, const int32_t *pcm, int32_t *sig, SigMeta *meta, int *blkflags, int nb, cudaStream_t st);
void launch_minbr_flags(const EncK &k, const SubframePlan *plans, const int *blkflags, int nb, int *flags, cudaStream_t st);
void launch_debug_evaluate(const EncK &k, const int32_t *sig, const SigMeta *meta, const CandDesc *cands, uint32_t *absr, uint32_t *est, int n);
void launch_lpc(const EncK &k, const double *autoc, const DevCand *cands, SigMeta *meta, const uint32_t *sigor, CandDesc *cdesc, int nitems, int autoc_unshifted, cudaStream_t st);
void launch_search_general(const EncK &k, size_t smem, const int32_t *sig, const SigMeta *meta, const CandDesc *cdesc, SubframePlan *plans, int nitems, cudaStream_t st);
void launch_emit_general(const EncK &k, size_t smem, const int32_t *sig, const int *blkflags, const SubframePlan *plans, uint8_t *slots, uint32_t *frame_bytes, uint32_t *chan_assign, int nb, cudaStream_t st);
void launch_scan(const uint32_t *bytes, int n, unsigned long long *offsets, unsigned long long *running, cudaStream_t st);
void launch_gather(const EncK &k, const uint8_t *slots, const uint32_t *bytes, const unsigned long long *offsets, uint8_t *out, unsigned long long capacity, int *err, int nb, cudaStream_t st);
void launch_debug_log(const double *dx, double *dy, int n);
void general_kernels_init(int device);  // raises the dynamic shared-memory limits once per device (never lowers them)
// autoc_kernel.cu
int autoc_kernel_lags(int lags);  // the LAGS instantiation k_autoc3 / k_autoc4 run for k.lags: values each record receives
void launch_autoc3(const EncK &k, const int32_t *sig, const SigMeta *meta, const float *windows, const DevSection *secs, double *autoc, int nitems, cudaStream_t st);
void autoc3_init(int device);
void launch_autoc4(const EncK &k, const int32_t *pcm, const SigMeta *meta, const float *secwin, int secwin_stride, const DevSection *secs, double *autoc, int nitems, uint32_t *sigor, int or_sec, cudaStream_t st);
void autoc4_init(int device);
constexpr int kSecwinSlack = 160;  // zero floats behind every per-section weight table (>= the largest autocorrelation tile)
// search_kernel.cu
void launch_search5(const EncK &k, int rt, int maxord_t, int wps, size_t smem, const int32_t *pcm, const SigMeta *meta, const CandDesc *cdesc, SubframePlan *plans, int nb, cudaStream_t st);
size_t search5_smem(int bs, int rt, int nsig, int wps, int max_po, bool wide);  // wide: more than 16 bits per sample
void search5_init(int device);
// emit_kernel.cu
void launch_emit3_pairs(const EncK &k, int rt, int maxord_t, size_t pair_smem, size_t join_smem, const Emit3Args &a, int nb, cudaStream_t st);
size_t join_smem(int join_words);
void launch_emit3(const EncK &k, int rt, int maxord_t, size_t smem, const Emit3Args &a, int nb, cudaStream_t st);
void launch_crc16_tables(uint16_t *tab, cudaStream_t st);
void emit3_init(int device);
// tiled_kernels.cu: stage B for frames that do not fit one CTA's shared memory
size_t search_tiled_smem();
void launch_search_tiled(const EncK &k, const int32_t *sig, const SigMeta *meta, const CandDesc *cdesc, SubframePlan *plans, int nitems, cudaStream_t st);
// k_emit_tiled (subframes into stage[nb * channels][sub_words], bit counts into stage_bits) + k_join_tiled (frames into slots)
void launch_emit_tiled(const EncK &k, const int32_t *sig, const int *blkflags, const SubframePlan *plans, uint32_t *stage, uint32_t *stage_bits,
                       int sub_words, uint32_t cap_bits, uint8_t *slots, uint32_t *frame_bytes, uint32_t *chan_assign, int *err, int nb, cudaStream_t st);
void tiled_init(int device);

// ---- fb200_encode_files_* (files_kernels.cu, md5_kernel.cu)
// One run of a file's samples, in int32 elements: `src` in the caller's back-to-back input, `dst` in the compacted layout (every
// file's full blocks block-major, then the tails grouped by length), `item0` its first k_unpack_files work item. A batch has two
// per file, its full blocks at [2f] and its tail at [2f + 1]; either may be empty.
struct FileSeg { unsigned long long src, dst, n, item0; };
// A file's frames in encode order: `nfull` full-block frames from `first` on, then its tail frame `tail` (~0u: none).
struct FileFrames { uint32_t first, nfull, tail; };
constexpr int kUnpackFilesItem = 4096;  // samples per k_unpack_files CTA
void launch_unpack_files(const void *in, int bytes_per_sample, const FileSeg *segs, int nsegs, unsigned long long items, int32_t *pcm, int bps, int *err,
                         cudaStream_t st);
// fb200_encode_pcm_files_* (pcm_container.cu): one file's data region in the container bytes. elem0 is its first value in the
// back-to-back numbering of every file's values (FileSeg::src), data its first byte from the start of the call's input, bytes
// 1-4 per value; big / is_unsigned / shift as format_input takes them.
struct PcmFileDev { unsigned long long elem0, data; uint32_t bytes, big, is_unsigned, shift; };

// ---- ReplayGain (replaygain_kernel.cu)
// One file of a k_replaygain launch: its samples are `n` per channel, interleaved int32, the first `na` of them from value `a`
// on and the rest from value `b` on; its windows go to v[win ..]. ds, W and filt are those of replaygain_rate.
struct RgFileDev { unsigned long long a, na, b, n, win; uint32_t channels, bps, ds, W, filt, pad; };
// The analysis rate of sample_rate: false when the ReplayGain filters cover neither it nor any of its halvings. Else
// *ds = the decimation factor, *W = samples per 50 ms window after decimation, *filt = the filter's row.
bool replaygain_rate(uint32_t sample_rate, uint32_t *ds, uint32_t *W, uint32_t *filt);
// k_replaygain, one launch for every file: every window's v and each file's max |sample| (peak[f], uint32).
void launch_replaygain(const int32_t *pcm, const RgFileDev *files, int nfiles, double *v, uint32_t *peak, cudaStream_t st);
// The host half: per-file and per-album gains and peaks from the windows and peaks (album[f]: the file's album id).
// nwin (null: n / ds / W each): file f's window count
void replaygain_results(const std::vector<RgFileDev> &files, const uint32_t *album, const double *v, const uint32_t *peak, fb200_replaygain_info *info,
                        const uint64_t *nwin = nullptr);
// fb200_encode_pcm_files_* with replay_gain: the analysis runs on the encoder's int32 copy; after it, rebuild() gives every file's
// final metadata blocks from the results (it returns FB200_OK or an error already set).
struct ReplayGainJob {
	uint32_t ds, W, filt;
	std::vector<uint32_t> bps;  // per file: the bits the tool scales by, the container's (info.bits_per_sample, shift included)
	int (*rebuild)(void *ctx, const fb200_replaygain_info *info, std::vector<uint8_t> *meta, std::vector<uint64_t> *moffs);
	void *ctx;
};
struct PcmSource {
	const uint8_t *data;  // host or device: the input's first byte
	unsigned long long bytes;
	std::vector<PcmFileDev> files;
	const ReplayGainJob *rg = nullptr;  // null: no ReplayGain
	// fb200_reencode_flac_files_*: fill() decodes every file straight into the compacted input (pcm, `values` int32, at the places
	// of d_segs) in place of k_pcm_unpack; the MD5 then runs on the call's stream before the encode, and check() (one synchronise)
	// reads the decode's verdicts and the digests d_md5 (16 per file) and sets keep[f] = 0 for each file the output leaves out.
	// A left-out file is still encoded with the rest (its blocks sit among the others'); the gather and the headers skip it.
	int (*fill)(void *ctx, int32_t *pcm, unsigned long long values, const FileSeg *d_segs, cudaStream_t st) = nullptr;
	int (*check)(void *ctx, const uint8_t *d_md5, cudaStream_t st, std::vector<uint8_t> *keep) = nullptr;
	void *ctx = nullptr;
};
// k_pcm_unpack over the segments of k_unpack_files: widens every file's values into pcm; *first_bad (start at ~0) = the lowest
// back-to-back value index whose shift bits are not zero. Reads only words that hold a byte of in[0, in_bytes).
void launch_pcm_unpack(const uint8_t *in, unsigned long long in_bytes, const PcmFileDev *files, const FileSeg *segs, int nsegs, unsigned long long items,
                       int32_t *pcm, unsigned long long *first_bad, cudaStream_t st);
// fb200_encode_flac_files_* with src's container bytes as input (encoder.cu); file_samples are the values present per channel
int encode_pcm_files_impl(fb200_encoder *e, const PcmSource &src, bool device, const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                          const uint8_t *metadata, const uint64_t *metadata_offsets, uint8_t *out, size_t out_capacity, uint64_t *frame_offsets,
                          uint64_t *nframes, fb200_flac_file_info *files, void *cuda_stream);
// One file's header of fb200_encode_flac_files_* (planned by flac_metadata.cu, written by k_flac_file_headers): `bytes` bytes
// (the file's audio offset) at `blob` in the call's header blob, "fLaC" + STREAMINFO + the other blocks, the STREAMINFO body
// and the SEEKTABLE body (at st_body, 0: none) left to the device; its seek table template is pts[pts .. pts + npts).
struct FlacHead { unsigned long long blob, pts; uint32_t bytes, st_body, npts, pad; };
struct SeekPt { unsigned long long sample, offset; uint32_t frame_samples, pad; };
struct FlacHeaderPlan {
	std::vector<FlacHead> heads;
	std::vector<uint8_t> blob;
	std::vector<SeekPt> pts;
};
// k_files_scan + k_files_gather: frames[o] = (frame in encode order, file) of output frame o; writes offsets[0 .. nframes].
// src holds src_cap bytes of frames (+ 4 readable bytes); frames the encode could not store there are not copied. heads
// (null: none) leaves each file's header room before its frames, fbase[f] being where the file's first frame goes, and copies
// each file's header from blob (readable 4 bytes past its end) there, nfiles CTAs more in the same launch.
void launch_files_gather(const uint8_t *src, unsigned long long src_cap, const unsigned long long *voff, const FileFrames *files, int nfiles, const uint2 *frames,
                         unsigned long long nframes, const FlacHead *heads, const uint8_t *blob, unsigned long long *fbase, uint8_t *out,
                         unsigned long long cap, unsigned long long *offsets, int *err, cudaStream_t st);
// k_flac_file_headers, one warp per file after the gather and the MD5: si[34 f ..] = file f's STREAMINFO body (min/max frame size
// over its frames, total samples, md5 + 16 f or zeros when md5 is null). With heads, also the parts of each file's header (copied
// before fbase[f] by k_files_gather) that depend on the frames: that STREAMINFO, and the seek table marked from the template,
// sorted, uniquified and padded with placeholders (stream_encoder.c:3070-3103, 3250-3261; format.c:281-314). Nothing is
// written at or past cap.
void launch_flac_file_headers(const unsigned long long *voff, const FileFrames *files, const FileSeg *segs, int nfiles, uint32_t blocksize, uint32_t channels,
                              uint32_t bits_per_sample, uint32_t sample_rate, const uint8_t *md5, uint8_t *si, const FlacHead *heads, const SeekPt *pts,
                              const unsigned long long *fbase, uint8_t *out, unsigned long long cap, cudaStream_t st);
void launch_md5_files(const int32_t *pcm, const FileSeg *segs, int nfiles, int bytes, uint8_t *digests, cudaStream_t st);  // digests[16 * nfiles]
// k_files_perturb (fb200_debug_perturb_verify): frames != null: frames[voff[v] + byte] ^= mask if that byte lies inside frame v
// and below cap; else pcm[elem] ^= mask
void launch_files_perturb(uint8_t *frames, const unsigned long long *voff, unsigned long long cap, unsigned long long v, uint32_t byte, int32_t *pcm,
                          unsigned long long elem, uint32_t mask, cudaStream_t st);
// k_files_tail_slots: every file's tail input (segs[2f + 1]) to out + (files[f].tail - first_tail) * slot, so that all tails, whatever
// their lengths, are verified by one launch set with the configured blocksize as the slot stride
void launch_files_tail_slots(const int32_t *pcm, const FileSeg *segs, const FileFrames *files, int nfiles, uint32_t first_tail, unsigned long long slot,
                             int32_t *out, cudaStream_t st);

// ---- verify of fb200_encode_files_* (decoder.cu: the frame decoder in compare mode)
// a frame's verdict: its lowest channel with a decoded sample != the input, and that channel's first one (channel ~0u: none)
struct DecVerdict { uint32_t channel, sample; int32_t expected, got; };
size_t verify_meta_bytes();  // the decoder's per-frame record, one per verified frame
constexpr size_t kVerifyCrcTabBytes = (1024 + 1024 * 5) * sizeof(uint16_t);  // k_dec_crc's table (decode_kernels.cuh, kDecCrcTabEntries)
void launch_verify_crc_tables(uint16_t *tab, cudaStream_t st);
// vb[i] = min(voff[i], cap) for i <= nframes
void launch_verify_bounds(const unsigned long long *voff, unsigned long long nframes, unsigned long long cap, unsigned long long *vb, cudaStream_t st);
// k_dec_walk + k_dec_frames<12 / 32, compare> + k_dec_crc over frames [vb[i], vb[i + 1]) of `frames`, i < nframes, every one of
// `blocksize` samples: frame i is compared with pcm[i * blocksize * channels ...]. Four launches.
void launch_verify_chunk(int channels, int bps, int sample_rate, int blocksize, const uint8_t *frames, const unsigned long long *vb, int nframes,
                         void *meta, DecVerdict *verdict, int32_t *pcm, const uint16_t *crc_tab, cudaStream_t st);
// k_verify_files: one record per file from the meta / verdicts of every frame of the call (indexed in encode order)
void launch_verify_files(const void *meta, const DecVerdict *verdict, const FileFrames *files, const FileSeg *segs, int nfiles, uint32_t channels,
                         uint32_t blocksize, uint32_t sample_rate, fb200_file_verify_info *info, cudaStream_t st);

// ---- fb200_decode_files_* (files_decode_kernels.cu)
// A candidate frame of a file: its first sample (~0: never accepted, e.g. a frame-number-coded frame in a stream whose
// STREAMINFO blocksizes differ), its header's blocksize, and whether its header codes a sample rate other than STREAMINFO's.
struct FileDecCand { unsigned long long first_sample; uint32_t blocksize, rate_differs; };
// One decode state, carried across the chunks of a call: a whole file (first_sample 0, end_sample its length) or a sample range
// of one (fb200_decode_files_ranges_*). Its candidates are [cand0, cand0 + ncand) of the arrays the call decodes.
struct FileDecState {
	unsigned long long cand0, ncand;
	unsigned long long first_value;           // where sample first_sample goes in the output
	unsigned long long first_sample, end_sample;  // the samples per channel placed: [first_sample, end_sample)
	unsigned long long accepted_end;          // byte end of the last accepted frame
	unsigned long long placed_end;            // sample end of the last placed frame
	unsigned long long covered;               // samples placed
	uint32_t channels, nframes, errors, damaged;  // damaged: inside a damaged stretch
};
// Where a candidate's slot goes: n values (0: nowhere) from slot value `off` on, to output value dst.
struct FilePlace { unsigned long long dst; uint32_t n, off; };
// k_files_accept over files[0 .. nfiles) for the chunk of candidates [c0, c1) (status / frame_bytes / place indexed from c0)
void launch_files_accept(FileDecState *files, int nfiles, const unsigned long long *begins, const FileDecCand *cands, const uint32_t *status,
                         const uint32_t *frame_bytes, unsigned long long c0, unsigned long long c1, FilePlace *place, cudaStream_t st);
// k_files_place: slot i (slot_values int32 each) to place[i], i < n. With segs (nsegs of them, a batch's FileSeg pairs), place[i].dst
// is a value index in the back-to-back numbering of FileSeg::src, and each value goes to the compacted layout the segments give.
void launch_files_place(const int32_t *slots, unsigned long long slot_values, const FilePlace *place, unsigned n, int32_t *out, const FileSeg *segs,
                        int nsegs, cudaStream_t st);
// A sample range's selection: the candidates [src0, src0 + nsrc) of the resident index that belong to its file, and the
// range [start, end) per channel.
struct RangeSel { unsigned long long src0, nsrc, start, end; };
// k_ranges_count: count[r] = candidates of range r whose samples meet it (first_sample != ~0, first_sample < end,
// first_sample + blocksize > start).
void launch_ranges_count(const RangeSel *sel, int nranges, const FileDecCand *cands, uint32_t *count, cudaStream_t st);
// k_ranges_select: those candidates, in index order, to out_*[dst0[r] ...]
void launch_ranges_select(const RangeSel *sel, int nranges, const unsigned long long *begins, const unsigned long long *ends, const FileDecCand *cands,
                          const unsigned long long *dst0, unsigned long long *out_begins, unsigned long long *out_ends, FileDecCand *out_cands,
                          cudaStream_t st);

// ---- fb200_decode_pcm_files_* (pcm_container.cu)
// The container header the flac tool writes (write_iff_headers, decode.c:718-989) for one file or range. mask: the resolved
// channel mask (tag, default or 0); too_big: the tool refuses the kind for this length (then nothing else is meaningful).
struct PcmHeader {
	uint8_t bytes[128];
	uint32_t length, container_bits, extensible, mask;
	uint64_t data_bytes;  // samples x channels x container bytes
	uint64_t pad;         // zero bytes after the data (decode.c:551-574)
	bool too_big;
};
// tag_mask: the WAVEFORMATEXTENSIBLE_CHANNEL_MASK tag's value (0: none); opt is valid (pcm_decode_options_ok)
void pcm_header_build(const fb200_pcm_decode_options &opt, uint32_t channels, uint32_t bps, uint32_t rate, uint32_t tag_mask, uint64_t samples, PcmHeader *h);
bool pcm_decode_options_ok(const fb200_pcm_decode_options *opt);  // sets the error when not
// One container of a k_pcm_pack launch: `out` its first byte in the output, the header's `hlen` bytes at `blob` of the header
// blob, then the data region (`data` bytes: FileSeg::n values from FileSeg::src of the int32 input, `bytes` 1-4 each, shifted
// left by `shift`, big-endian or not, +0x80 when unsigned), then `pad` zero bytes.
struct PcmPackDev { unsigned long long out, blob, data; uint32_t hlen, pad, bytes, big, is_unsigned, shift; };
// k_pcm_pack: segs[i] (dst = the data region's first output byte) describe the data regions of the containers that have values,
// seg_cont[i] their container; items = the data items of those segments; ncont extra CTAs write the headers and pad bytes.
void launch_pcm_pack(const int32_t *pcm, const FileSeg *segs, const uint32_t *seg_cont, int nsegs, unsigned long long items, const PcmPackDev *conts,
                     int ncont, const uint8_t *blob, uint8_t *out, cudaStream_t st);

// STREAMINFO body, 34 bytes (format.c:65-73; stream_encoder_framing.c:62-95): what the object-API shell writes (the batch entry
// points build theirs on the device, k_flac_file_headers)
void put_streaminfo(uint8_t body[34], uint32_t min_blocksize, uint32_t max_blocksize, uint32_t min_framesize, uint32_t max_framesize,
                    uint32_t sample_rate, uint32_t channels, uint32_t bits_per_sample, uint64_t total_samples, const uint8_t md5[16]);

// ---- fb200_reencode_flac_files_* (reencode.cu)
// decoder.cu: the facts a re-encode reads of the batch fb200_decode_files_index left resident (false without one): each file's
// index record, its bytes [start, audio) (the ID3v2 tag and metadata, from the resident copy), its STREAMINFO MD5 and its channel
// mask tag (channel_mask_tag)
bool decoder_files(const fb200_decoder *d, uint32_t *nfiles, int *device);
const fb200_file_decode_info &decoder_file_info(const fb200_decoder *d, uint32_t f);
int decoder_file_metadata(fb200_decoder *d, uint32_t f, std::vector<uint8_t> *bytes);
const uint8_t *decoder_file_md5(const fb200_decoder *d, uint32_t f);
uint32_t decoder_file_mask(const fb200_decoder *d, uint32_t f);
// decoder.cu: the whole-file decode of files[0 .. n) of the resident batch, file files[i]'s samples to the back-to-back value
// first_value[i] on, placed through d_segs into pcm (zeroed first, `values` long). Enqueued on st.
// keep_place / keep_bytes (null: not kept): one entry per candidate of the index, where every decoded candidate's FilePlace and
// frame byte count stay (a listed file's accepted frames are its candidates with place n > 0, in file order).
int decoder_decode_into(fb200_decoder *d, const uint32_t *files, const uint64_t *first_value, uint32_t n, int32_t *pcm, unsigned long long values,
                        const FileSeg *d_segs, int nsegs, cudaStream_t st, FilePlace *keep_place = nullptr, uint32_t *keep_bytes = nullptr);
// decoder.cu: the ranged decode (fb200_decode_files_ranges_*) of ranges[0 .. n) of the resident batch, each over a file whose index
// status is OK and within its samples, range i's samples to the back-to-back value first_value[i] on, placed through d_segs into pcm
// (zeroed first, `values` long). Returns after completion with each range's damaged stretches + overlapping frames (errors) and
// samples no accepted frame covered (missing).
int decoder_decode_ranges_into(fb200_decoder *d, const fb200_sample_range *ranges, const uint64_t *first_value, uint32_t n, int32_t *pcm,
                               unsigned long long values, const FileSeg *d_segs, int nsegs, cudaStream_t st, uint32_t *errors, uint64_t *missing);
// per listed file, after decoder_decode_into and a synchronise: damaged stretches and samples no accepted frame covered
int decoder_decode_verdicts(fb200_decoder *d, const uint32_t *files, uint32_t n, cudaStream_t st, uint32_t *errors, uint64_t *missing);
// ---- fb200_add_replaygain_flac_files_* (add_replaygain.cu): the resident index on the device, and one file's place in it: bytes
// [start, audio) are its metadata, [audio, end) its audio region; its candidates are [cand0, cand0 + ncand), its state states[state]
struct DecoderFilesView {
	const uint8_t *data;
	const unsigned long long *begins;
	const FileDecCand *cands;
	const FileDecState *states;
	uint64_t ncand;
};
struct DecoderFileSpan { uint64_t start, audio, end, cand0, ncand; uint32_t state; };
DecoderFilesView decoder_files_view(const fb200_decoder *d);
DecoderFileSpan decoder_file_span(const fb200_decoder *d, uint32_t f);  // f must have index status FB200_FILE_OK
void decoder_count_launches(fb200_decoder *d, uint64_t n);
// k_replaygain_frames (replaygain_kernel.cu): one file of a launch. Its accepted frames are its candidates [cand0, cand0 + ncand)
// with place[i].n > 0; they must tile [audio, end) (begins[i], bytes[i]) and the file's decode state must hold no error. win: its
// first window in v, at most nwin_cap of them. ds, W, filt as replaygain_rate.
struct RgFramesFileDev { unsigned long long cand0, ncand, audio, end, win, nwin_cap; uint32_t state, channels, bps, ds, W, filt; };
// per file: the windows written, max |sample|, and 1 when the frames passed the checks
struct RgFramesOut { unsigned long long nwin; uint32_t peak, ok; };
void launch_replaygain_frames(const int32_t *pcm, const RgFramesFileDev *files, int nfiles, const FilePlace *place, const unsigned long long *begins,
                              const uint32_t *bytes, const FileDecCand *cands, const FileDecState *states, double *v, RgFramesOut *out, cudaStream_t st);

// ---- ReplayGain synthesis (replaygain_synthesis.cu): flac -d --apply-replaygain-which-is-not-lossless
// The constants of apply_gain for one container: multi_scale, the dither context's Add / Mask / Dither (from the stream's bits),
// conv_shift and the clip factor (from the target width), and whether the hard limiter runs.
struct RgsParam { double multi, add; unsigned long long mask; long long clip; float dither; int conv_shift, hard, pad; };
RgsParam rgs_param(uint32_t bps, double scale, bool hard, uint32_t shaping);
// No shaping: values [v0, v0 + n) of the int32 scratch, CTAs from item0 on
struct RgsSeg { unsigned long long v0, n, item0; RgsParam P; };
// A delivered block (what the tool's write callback receives): samples [s, s + n) from the container's first sample
struct RgsBlock { unsigned long long s, n; };
// With shaping: channel c of a container of C channels and ns samples whose first value is v0; its blocks [b0, b0 + nb) tile
// [0, ns); draw0 is the generator's position at the container's first sample
struct RgsChain { unsigned long long v0, ns, draw0; uint32_t C, c, b0, nb; RgsParam P; };
struct RgsPlan {
	std::vector<RgsSeg> segs;
	std::vector<RgsChain> chains;
	std::vector<RgsBlock> blocks;
};
// Applies the plan to the int32 scratch in place (val32 per value): k_rg_synth0 for segs, k_rg_synth<shaping> for chains. work is
// grown as needed.
int rgs_run(const RgsPlan &plan, uint32_t shaping, int32_t *pcm, cudaStream_t st, uint8_t **work, size_t *work_cap, uint64_t *launches);
// The tool's decision for one .flac file (its bytes) of a bps-bit stream; first_draw and draws are left 0
void rgs_decide(const uint8_t *p, size_t n, uint32_t bps, const fb200_replaygain_synthesis &rg, fb200_replaygain_synthesis_info *info);
bool rgs_spec_ok(const fb200_replaygain_synthesis *rg);  // sets the error when not

// encoder.cu: the verify records of the last call, spread over nlisted entries (records[i] goes to entry at[i], the rest OK)
void encoder_spread_verify(fb200_encoder *e, const std::vector<uint32_t> &at, uint32_t nlisted);
int encoder_device(const fb200_encoder *e);

// encoder.cu, for the object-API shell (stream_api.cu): fb200_encoder_create, where bound_tiled also caps a non-zero
// max_blocks at the tiled sample budget (FB200_TILED_SAMPLE_BUDGET) when the configuration runs the tiled kernels;
// encoder_capacity is the resulting number of blocks per launch
int encoder_create(const fb200_encoder_config *cfg, int device, uint32_t max_blocks, bool bound_tiled, fb200_encoder **out);
uint32_t encoder_capacity(const fb200_encoder *e);

}  // namespace fb200
