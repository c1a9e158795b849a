// stream_api.cu -- the reference's stream encoder/decoder object API (include/flac_b200_stream.h)
// implemented as a thin host shell over the batch C ABI (include/flac_b200.h).
//
// What the shell does is what src/libFLAC/stream_encoder.c / stream_decoder.c do around the
// per-frame hot path: settings and their validation (stream_encoder.c:725-830, 1780-2511),
// metadata writing (stream_encoder_framing.c:47-243), sample range checks and block
// buffering (:2513-2620), MD5 of the input (md5.c:280-521), write callbacks in frame order
// with seek-table marking and STREAMINFO patch-up (:3038-3300). Blocks are queued and encoded
// in batches; callbacks are therefore deferred and bursty exactly as the reference documents
// for set_num_threads(n>1) (include/FLAC/stream_encoder.h:1116-1158).
// Host-only code (no kernels); everything per-frame happens inside fb200_encode_host /
// fb200_decode_host. No CPU fallback: if the engine cannot be created, init fails.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/flac_b200.h"
#include "../../include/flac_b200_stream.h"
#include "fb200_internal.h"
#include "flac_metadata.h"
#include "flac_parse.h"

// ------------------------------------------------------------------ small host utilities
namespace {

// RFC 1321 MD5 (the reference keeps its own copy in src/libFLAC/md5.c)
struct MD5 {
	uint32_t a, b, c, d;
	uint64_t bytes;
	uint8_t buf[64];
	uint32_t fill;
	void init() { a = 0x67452301; b = 0xefcdab89; c = 0x98badcfe; d = 0x10325476; bytes = 0; fill = 0; }
	static uint32_t rol(uint32_t v, int s) { return (v << s) | (v >> (32 - s)); }
	void block(const uint8_t *p)
	{
		static const uint32_t K[64] = {
			0xd76aa478, 0xe8c7b756, 0x242070db, 0xc1bdceee, 0xf57c0faf, 0x4787c62a, 0xa8304613, 0xfd469501, 0x698098d8, 0x8b44f7af, 0xffff5bb1, 0x895cd7be,
			0x6b901122, 0xfd987193, 0xa679438e, 0x49b40821, 0xf61e2562, 0xc040b340, 0x265e5a51, 0xe9b6c7aa, 0xd62f105d, 0x02441453, 0xd8a1e681, 0xe7d3fbc8,
			0x21e1cde6, 0xc33707d6, 0xf4d50d87, 0x455a14ed, 0xa9e3e905, 0xfcefa3f8, 0x676f02d9, 0x8d2a4c8a, 0xfffa3942, 0x8771f681, 0x6d9d6122, 0xfde5380c,
			0xa4beea44, 0x4bdecfa9, 0xf6bb4b60, 0xbebfbc70, 0x289b7ec6, 0xeaa127fa, 0xd4ef3085, 0x04881d05, 0xd9d4d039, 0xe6db99e5, 0x1fa27cf8, 0xc4ac5665,
			0xf4292244, 0x432aff97, 0xab9423a7, 0xfc93a039, 0x655b59c3, 0x8f0ccc92, 0xffeff47d, 0x85845dd1, 0x6fa87e4f, 0xfe2ce6e0, 0xa3014314, 0x4e0811a1,
			0xf7537e82, 0xbd3af235, 0x2ad7d2bb, 0xeb86d391};
		static const int S[64] = {7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 7, 12, 17, 22, 5, 9, 14, 20, 5, 9, 14, 20, 5, 9, 14, 20, 5, 9, 14, 20,
		                          4, 11, 16, 23, 4, 11, 16, 23, 4, 11, 16, 23, 4, 11, 16, 23, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21, 6, 10, 15, 21};
		uint32_t w[16];
		for(int i = 0; i < 16; i++) w[i] = (uint32_t)p[4 * i] | ((uint32_t)p[4 * i + 1] << 8) | ((uint32_t)p[4 * i + 2] << 16) | ((uint32_t)p[4 * i + 3] << 24);
		uint32_t A = a, B = b, C = c, D = d;
		for(int i = 0; i < 64; i++) {
			uint32_t f;
			int g;
			if(i < 16) { f = (B & C) | (~B & D); g = i; }
			else if(i < 32) { f = (D & B) | (~D & C); g = (5 * i + 1) & 15; }
			else if(i < 48) { f = B ^ C ^ D; g = (3 * i + 5) & 15; }
			else { f = C ^ (B | ~D); g = (7 * i) & 15; }
			const uint32_t t = D;
			D = C; C = B;
			B = B + rol(A + f + K[i] + w[g], S[i]);
			A = t;
		}
		a += A; b += B; c += C; d += D;
	}
	void update(const uint8_t *p, size_t n)
	{
		bytes += n;
		while(n) {
			const size_t take = std::min<size_t>(n, 64 - fill);
			memcpy(buf + fill, p, take);
			fill += (uint32_t)take; p += take; n -= take;
			if(fill == 64) { block(buf); fill = 0; }
		}
	}
	void final(uint8_t out[16])
	{
		const uint64_t bits = bytes * 8;
		const uint8_t pad = 0x80;
		update(&pad, 1);
		const uint8_t z = 0;
		while(fill != 56) update(&z, 1);
		uint8_t len[8];
		for(int i = 0; i < 8; i++) len[i] = (uint8_t)(bits >> (8 * i));
		update(len, 8);
		const uint32_t v[4] = {a, b, c, d};
		for(int i = 0; i < 16; i++) out[i] = (uint8_t)(v[i >> 2] >> (8 * (i & 3)));
	}
	// FLAC feeds the interleaved samples as little-endian integers of (bps+7)/8 bytes (md5.c:280-495)
	void update_samples(const int32_t *interleaved, size_t count, uint32_t bytes_per_sample)
	{
		uint8_t tmp[4096];
		size_t n = 0;
		for(size_t i = 0; i < count; i++) {
			const uint32_t v = (uint32_t)interleaved[i];
			for(uint32_t k = 0; k < bytes_per_sample; k++) tmp[n++] = (uint8_t)(v >> (8 * k));
			if(n + 4 > sizeof tmp) { update(tmp, n); n = 0; }
		}
		if(n) update(tmp, n);
	}
};

struct ByteWriter {
	std::vector<uint8_t> v;
	void u(uint64_t val, int nbytes) { for(int i = nbytes - 1; i >= 0; i--) v.push_back((uint8_t)(val >> (8 * i))); }
	void raw(const void *p, size_t n) { const uint8_t *b = (const uint8_t *)p; v.insert(v.end(), b, b + n); }
	void zeros(size_t n) { v.insert(v.end(), n, 0); }
};

void put_streaminfo(ByteWriter &w, const FLAC__StreamMetadata_StreamInfo &si)
{
	uint8_t body[34];
	fb200::put_streaminfo(body, si.min_blocksize, si.max_blocksize, si.min_framesize, si.max_framesize, si.sample_rate, si.channels,
	                      si.bits_per_sample, si.total_samples, si.md5sum);
	w.raw(body, sizeof body);
}

// One metadata block incl. its 4-byte header (stream_encoder_framing.c:47-243). Returns false for unsupported types.
bool serialize_metadata(const FLAC__StreamMetadata *m, bool is_last, const char *vendor, std::vector<uint8_t> &out)
{
	ByteWriter body;
	switch(m->type) {
		case FLAC__METADATA_TYPE_STREAMINFO: put_streaminfo(body, m->data.stream_info); break;
		case FLAC__METADATA_TYPE_PADDING: body.zeros(m->length); break;
		case FLAC__METADATA_TYPE_APPLICATION:
			body.raw(m->data.application.id, 4);
			if(m->length > 4 && m->data.application.data) body.raw(m->data.application.data, m->length - 4);
			break;
		case FLAC__METADATA_TYPE_SEEKTABLE:
			for(uint32_t i = 0; i < m->data.seek_table.num_points; i++) {
				body.u(m->data.seek_table.points[i].sample_number, 8);
				body.u(m->data.seek_table.points[i].stream_offset, 8);
				body.u(m->data.seek_table.points[i].frame_samples, 2);
			}
			break;
		case FLAC__METADATA_TYPE_VORBIS_COMMENT: {
			// the encoder always writes its own vendor string (stream_encoder_framing.c:118-133)
			const uint32_t vlen = (uint32_t)strlen(vendor);
			fb200::put_le32(body.v, vlen); body.raw(vendor, vlen);
			fb200::put_le32(body.v, m->data.vorbis_comment.num_comments);
			for(uint32_t i = 0; i < m->data.vorbis_comment.num_comments; i++) {
				fb200::put_le32(body.v, m->data.vorbis_comment.comments[i].length);
				body.raw(m->data.vorbis_comment.comments[i].entry, m->data.vorbis_comment.comments[i].length);
			}
			break;
		}
		case FLAC__METADATA_TYPE_CUESHEET: {
			const FLAC__StreamMetadata_CueSheet &cs = m->data.cue_sheet;
			body.raw(cs.media_catalog_number, 128);
			body.u(cs.lead_in, 8);
			body.u(cs.is_cd ? 0x80 : 0, 1); body.zeros(258);
			body.u(cs.num_tracks, 1);
			for(uint32_t t = 0; t < cs.num_tracks; t++) {
				const FLAC__StreamMetadata_CueSheet_Track &tr = cs.tracks[t];
				body.u(tr.offset, 8); body.u(tr.number, 1); body.raw(tr.isrc, 12);
				body.u((tr.type ? 0x80 : 0) | (tr.pre_emphasis ? 0x40 : 0), 1); body.zeros(13);
				body.u(tr.num_indices, 1);
				for(uint32_t k = 0; k < tr.num_indices; k++) { body.u(tr.indices[k].offset, 8); body.u(tr.indices[k].number, 1); body.zeros(3); }
			}
			break;
		}
		case FLAC__METADATA_TYPE_PICTURE: {
			const FLAC__StreamMetadata_Picture &p = m->data.picture;
			const uint32_t ml = (uint32_t)strlen(p.mime_type ? p.mime_type : ""), dl = (uint32_t)strlen(p.description ? (const char *)p.description : "");
			body.u(p.type, 4); body.u(ml, 4); body.raw(p.mime_type ? p.mime_type : "", ml);
			body.u(dl, 4); body.raw(p.description ? (const char *)p.description : "", dl);
			body.u(p.width, 4); body.u(p.height, 4); body.u(p.depth, 4); body.u(p.colors, 4);
			body.u(p.data_length, 4); body.raw(p.data, p.data_length);
			break;
		}
		default:
			if(m->data.unknown.data) body.raw(m->data.unknown.data, m->length);
			else body.zeros(m->length);
			break;
	}
	if(body.v.size() >= (1u << 24)) return false;
	out.clear();
	fb200::put_block_header(out, is_last, (uint32_t)m->type & 0x7f, (uint32_t)body.v.size());
	out.insert(out.end(), body.v.begin(), body.v.end());
	return true;
}

uint32_t batch_blocks()
{
	const char *e = getenv("FB200_BATCH_BLOCKS");
	const long v = e ? atol(e) : 1024;
	return (uint32_t)std::max<long>(1, std::min<long>(v, 65536));
}

}  // namespace

extern "C" {

const char *FLAC__VERSION_STRING = "1.5.0-b200";
const char *FLAC__VENDOR_STRING = "flac_b200 0.1 (libFLAC 1.5.0 bitstream, sm_90a)";

const char *const FLAC__StreamEncoderStateString[] = {
	"FLAC__STREAM_ENCODER_OK", "FLAC__STREAM_ENCODER_UNINITIALIZED", "FLAC__STREAM_ENCODER_OGG_ERROR",
	"FLAC__STREAM_ENCODER_VERIFY_DECODER_ERROR", "FLAC__STREAM_ENCODER_VERIFY_MISMATCH_IN_AUDIO_DATA",
	"FLAC__STREAM_ENCODER_CLIENT_ERROR", "FLAC__STREAM_ENCODER_IO_ERROR", "FLAC__STREAM_ENCODER_FRAMING_ERROR",
	"FLAC__STREAM_ENCODER_MEMORY_ALLOCATION_ERROR"};
const char *const FLAC__StreamEncoderInitStatusString[] = {
	"FLAC__STREAM_ENCODER_INIT_STATUS_OK", "FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR", "FLAC__STREAM_ENCODER_INIT_STATUS_UNSUPPORTED_CONTAINER",
	"FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_CALLBACKS", "FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_NUMBER_OF_CHANNELS",
	"FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_BITS_PER_SAMPLE", "FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_SAMPLE_RATE",
	"FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_BLOCK_SIZE", "FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_MAX_LPC_ORDER",
	"FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_QLP_COEFF_PRECISION", "FLAC__STREAM_ENCODER_INIT_STATUS_BLOCK_SIZE_TOO_SMALL_FOR_LPC_ORDER",
	"FLAC__STREAM_ENCODER_INIT_STATUS_NOT_STREAMABLE", "FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_METADATA",
	"FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED"};
// The enumerator names of the remaining status enums, in enum order (include/FLAC/stream_encoder.h:388-454,
// include/FLAC/stream_decoder.h:297-480, include/FLAC/format.h). Clients index them directly: src/flac/decode.c:1834,
// src/flac/encode.c:2677, examples/c/decode/file/main.c.
#define FB_S(x) #x
const char *const FLAC__StreamEncoderReadStatusString[] = {
	FB_S(FLAC__STREAM_ENCODER_READ_STATUS_CONTINUE), FB_S(FLAC__STREAM_ENCODER_READ_STATUS_END_OF_STREAM), FB_S(FLAC__STREAM_ENCODER_READ_STATUS_ABORT),
	FB_S(FLAC__STREAM_ENCODER_READ_STATUS_UNSUPPORTED)};
const char *const FLAC__StreamEncoderWriteStatusString[] = {FB_S(FLAC__STREAM_ENCODER_WRITE_STATUS_OK), FB_S(FLAC__STREAM_ENCODER_WRITE_STATUS_FATAL_ERROR)};
const char *const FLAC__StreamEncoderSeekStatusString[] = {
	FB_S(FLAC__STREAM_ENCODER_SEEK_STATUS_OK), FB_S(FLAC__STREAM_ENCODER_SEEK_STATUS_ERROR), FB_S(FLAC__STREAM_ENCODER_SEEK_STATUS_UNSUPPORTED)};
const char *const FLAC__StreamEncoderTellStatusString[] = {
	FB_S(FLAC__STREAM_ENCODER_TELL_STATUS_OK), FB_S(FLAC__STREAM_ENCODER_TELL_STATUS_ERROR), FB_S(FLAC__STREAM_ENCODER_TELL_STATUS_UNSUPPORTED)};
const char *const FLAC__StreamDecoderInitStatusString[] = {
	FB_S(FLAC__STREAM_DECODER_INIT_STATUS_OK), FB_S(FLAC__STREAM_DECODER_INIT_STATUS_UNSUPPORTED_CONTAINER), FB_S(FLAC__STREAM_DECODER_INIT_STATUS_INVALID_CALLBACKS),
	FB_S(FLAC__STREAM_DECODER_INIT_STATUS_MEMORY_ALLOCATION_ERROR), FB_S(FLAC__STREAM_DECODER_INIT_STATUS_ERROR_OPENING_FILE),
	FB_S(FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED)};
const char *const FLAC__StreamDecoderReadStatusString[] = {
	FB_S(FLAC__STREAM_DECODER_READ_STATUS_CONTINUE), FB_S(FLAC__STREAM_DECODER_READ_STATUS_END_OF_STREAM), FB_S(FLAC__STREAM_DECODER_READ_STATUS_ABORT),
	FB_S(FLAC__STREAM_DECODER_READ_STATUS_END_OF_LINK)};
const char *const FLAC__StreamDecoderSeekStatusString[] = {
	FB_S(FLAC__STREAM_DECODER_SEEK_STATUS_OK), FB_S(FLAC__STREAM_DECODER_SEEK_STATUS_ERROR), FB_S(FLAC__STREAM_DECODER_SEEK_STATUS_UNSUPPORTED)};
const char *const FLAC__StreamDecoderTellStatusString[] = {
	FB_S(FLAC__STREAM_DECODER_TELL_STATUS_OK), FB_S(FLAC__STREAM_DECODER_TELL_STATUS_ERROR), FB_S(FLAC__STREAM_DECODER_TELL_STATUS_UNSUPPORTED)};
const char *const FLAC__StreamDecoderLengthStatusString[] = {
	FB_S(FLAC__STREAM_DECODER_LENGTH_STATUS_OK), FB_S(FLAC__STREAM_DECODER_LENGTH_STATUS_ERROR), FB_S(FLAC__STREAM_DECODER_LENGTH_STATUS_UNSUPPORTED)};
const char *const FLAC__StreamDecoderWriteStatusString[] = {FB_S(FLAC__STREAM_DECODER_WRITE_STATUS_CONTINUE), FB_S(FLAC__STREAM_DECODER_WRITE_STATUS_ABORT)};
const char *const FLAC__StreamDecoderErrorStatusString[] = {
	FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_LOST_SYNC), FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_BAD_HEADER), FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_FRAME_CRC_MISMATCH),
	FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_UNPARSEABLE_STREAM), FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_BAD_METADATA),
	FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_OUT_OF_BOUNDS), FB_S(FLAC__STREAM_DECODER_ERROR_STATUS_MISSING_FRAME)};
// format.h tables: short names, as the analysis output of `flac -a` prints them (src/flac/analyze.c)
const char *const FLAC__EntropyCodingMethodTypeString[] = {"PARTITIONED_RICE", "PARTITIONED_RICE2"};
const char *const FLAC__SubframeTypeString[] = {"CONSTANT", "VERBATIM", "FIXED", "LPC"};
const char *const FLAC__ChannelAssignmentString[] = {"INDEPENDENT", "LEFT_SIDE", "RIGHT_SIDE", "MID_SIDE"};
const char *const FLAC__FrameNumberTypeString[] = {"FRAME_NUMBER_TYPE_FRAME_NUMBER", "FRAME_NUMBER_TYPE_SAMPLE_NUMBER"};
const char *const FLAC__MetadataTypeString[] = {"STREAMINFO", "PADDING", "APPLICATION", "SEEKTABLE", "VORBIS_COMMENT", "CUESHEET", "PICTURE"};
#undef FB_S
// built without libogg, like the oracle configuration (include/FLAC/export.h:107, stream_decoder.c:59)
int FLAC_API_SUPPORTS_OGG_FLAC = 0;

const char *const FLAC__StreamDecoderStateString[] = {
	"FLAC__STREAM_DECODER_SEARCH_FOR_METADATA", "FLAC__STREAM_DECODER_READ_METADATA", "FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC",
	"FLAC__STREAM_DECODER_READ_FRAME", "FLAC__STREAM_DECODER_END_OF_STREAM", "FLAC__STREAM_DECODER_OGG_ERROR", "FLAC__STREAM_DECODER_SEEK_ERROR",
	"FLAC__STREAM_DECODER_ABORTED", "FLAC__STREAM_DECODER_MEMORY_ALLOCATION_ERROR", "FLAC__STREAM_DECODER_UNINITIALIZED", "FLAC__STREAM_DECODER_END_OF_LINK"};

}  // extern "C"

// ================================================================== encoder object

struct FLAC__StreamEncoderProtected {
	FLAC__StreamEncoderState state;
	FLAC__bool verify, streamable_subset, do_md5;
	fb200_encoder_config cfg;          // every knob that reaches the frame path
	FLAC__bool do_escape_coding;
	uint32_t rice_parameter_search_dist, num_threads;
	FLAC__uint64 total_samples_estimate;
	FLAC__StreamMetadata **metadata;
	uint32_t num_metadata_blocks;
};

struct FLAC__StreamEncoderPrivate {
	FLAC__StreamEncoderWriteCallback write_cb;
	FLAC__StreamEncoderSeekCallback seek_cb;
	FLAC__StreamEncoderTellCallback tell_cb;
	FLAC__StreamEncoderMetadataCallback metadata_cb;
	FLAC__StreamEncoderProgressCallback progress_cb;
	void *client_data;
	FILE *file;
	bool owns_file;
	fb200_encoder *gpu;
	fb200_decoder *vdec;
	uint32_t batch;
	std::vector<int32_t> pending;  // interleaved (kept for --verify)
	std::vector<uint8_t> pending_packed;  // the same samples as little-endian 2-/3-byte PCM: what crosses PCIe (fb200_encode_host_packed)
	uint32_t pack_bytes;           // 2 (bps <= 16), 3 (bps <= 24)
	uint64_t pending_samples;
	std::vector<uint8_t> frames;
	std::vector<uint64_t> offsets;
	std::vector<int32_t> verify_pcm;
	MD5 md5;
	FLAC__StreamMetadata_StreamInfo si;
	uint32_t frames_written;
	uint64_t samples_written, bytes_written;
	uint64_t streaminfo_offset, seektable_offset, audio_offset;
	FLAC__StreamMetadata *seek_table;
	uint32_t first_seekpoint_to_check;
	// verify stats (stream_encoder.h:1322-1335)
	FLAC__uint64 v_abs_sample;
	uint32_t v_frame, v_channel, v_sample;
	FLAC__int32 v_expected, v_got;
};

static void enc_set_defaults(FLAC__StreamEncoder *e)
{
	// stream_encoder.c:2630-2690 set_defaults_ + set_compression_level(5) (:2688)
	FLAC__StreamEncoderProtected *p = e->protected_;
	p->verify = false; p->streamable_subset = true; p->do_md5 = true;
	memset(&p->cfg, 0, sizeof p->cfg);
	fb200_encoder_config_preset(&p->cfg, 2, 16, 44100, 5, 0);
	p->do_escape_coding = false; p->rice_parameter_search_dist = 0; p->num_threads = 1;
	p->total_samples_estimate = 0; p->metadata = nullptr; p->num_metadata_blocks = 0;
	FLAC__StreamEncoderPrivate *q = e->private_;
	q->write_cb = nullptr; q->seek_cb = nullptr; q->tell_cb = nullptr; q->metadata_cb = nullptr; q->progress_cb = nullptr;
	q->client_data = nullptr; q->file = nullptr; q->owns_file = false;
	q->seek_table = nullptr;
}

static void enc_release(FLAC__StreamEncoder *e)
{
	FLAC__StreamEncoderPrivate *q = e->private_;
	if(q->gpu) { fb200_encoder_destroy(q->gpu); q->gpu = nullptr; }
	if(q->vdec) { fb200_decoder_destroy(q->vdec); q->vdec = nullptr; }
	if(q->file && q->owns_file) fclose(q->file);
	q->file = nullptr;
	q->pending.clear(); q->pending.shrink_to_fit();
	q->pending_packed.clear(); q->pending_packed.shrink_to_fit();
	q->frames.clear(); q->frames.shrink_to_fit();
	q->offsets.clear(); q->verify_pcm.clear();
	q->pending_samples = 0;
}

extern "C" {

FLAC__StreamEncoder *FLAC__stream_encoder_new(void)
{
	FLAC__StreamEncoder *e = (FLAC__StreamEncoder *)calloc(1, sizeof *e);
	if(!e) return nullptr;
	e->protected_ = new FLAC__StreamEncoderProtected();
	e->private_ = new FLAC__StreamEncoderPrivate();
	e->private_->gpu = nullptr; e->private_->vdec = nullptr;
	e->private_->pending_samples = 0;
	enc_set_defaults(e);
	e->protected_->state = FLAC__STREAM_ENCODER_UNINITIALIZED;
	return e;
}

void FLAC__stream_encoder_delete(FLAC__StreamEncoder *e)
{
	if(!e) return;
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) FLAC__stream_encoder_finish(e);
	enc_release(e);
	delete e->protected_;
	delete e->private_;
	free(e);
}

#define ENC_SETTER(name, type, stmt)                                             \
	FLAC__bool FLAC__stream_encoder_##name(FLAC__StreamEncoder *e, type value)   \
	{                                                                            \
		if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return false; \
		stmt;                                                                    \
		return true;                                                             \
	}
ENC_SETTER(set_ogg_serial_number, long, (void)value)
ENC_SETTER(set_verify, FLAC__bool, e->protected_->verify = value)
ENC_SETTER(set_streamable_subset, FLAC__bool, e->protected_->streamable_subset = value)
ENC_SETTER(set_channels, uint32_t, e->protected_->cfg.channels = value)
ENC_SETTER(set_bits_per_sample, uint32_t, e->protected_->cfg.bits_per_sample = value)
ENC_SETTER(set_sample_rate, uint32_t, e->protected_->cfg.sample_rate = value)
ENC_SETTER(set_blocksize, uint32_t, e->protected_->cfg.blocksize = value)
ENC_SETTER(set_do_mid_side_stereo, FLAC__bool, e->protected_->cfg.do_mid_side_stereo = value)
ENC_SETTER(set_loose_mid_side_stereo, FLAC__bool, e->protected_->cfg.loose_mid_side_stereo = value)
ENC_SETTER(set_max_lpc_order, uint32_t, e->protected_->cfg.max_lpc_order = value)
ENC_SETTER(set_qlp_coeff_precision, uint32_t, e->protected_->cfg.qlp_coeff_precision = value)
ENC_SETTER(set_do_qlp_coeff_prec_search, FLAC__bool, e->protected_->cfg.do_qlp_coeff_prec_search = value)
ENC_SETTER(set_do_escape_coding, FLAC__bool, (void)value /* disabled outside fuzz builds, stream_encoder.c:2107-2114 */)
ENC_SETTER(set_do_exhaustive_model_search, FLAC__bool, e->protected_->cfg.do_exhaustive_model_search = value)
ENC_SETTER(set_min_residual_partition_order, uint32_t, e->protected_->cfg.min_residual_partition_order = value)
ENC_SETTER(set_max_residual_partition_order, uint32_t, e->protected_->cfg.max_residual_partition_order = value)
ENC_SETTER(set_rice_parameter_search_dist, uint32_t, e->protected_->rice_parameter_search_dist = value)
ENC_SETTER(set_limit_min_bitrate, FLAC__bool, e->protected_->cfg.limit_min_bitrate = value)
ENC_SETTER(disable_instruction_set, int, (void)value)
ENC_SETTER(disable_constant_subframes, FLAC__bool, e->protected_->cfg.disable_constant_subframes = value)
ENC_SETTER(disable_fixed_subframes, FLAC__bool, e->protected_->cfg.disable_fixed_subframes = value)
ENC_SETTER(disable_verbatim_subframes, FLAC__bool, e->protected_->cfg.disable_verbatim_subframes = value)
ENC_SETTER(set_do_md5, FLAC__bool, e->protected_->do_md5 = value)

FLAC__bool FLAC__stream_encoder_set_total_samples_estimate(FLAC__StreamEncoder *e, FLAC__uint64 value)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return false;
	e->protected_->total_samples_estimate = std::min<FLAC__uint64>(value, (1ull << 36) - 1);
	return true;
}

uint32_t FLAC__stream_encoder_set_num_threads(FLAC__StreamEncoder *e, uint32_t value)
{
	// stream_encoder.h:291-294: 0 = OK, 2 = already initialised, 3 = too many threads
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return 2;
	if(value > 64) return 3;
	e->protected_->num_threads = value ? value : 1;
	return 0;
}

FLAC__bool FLAC__stream_encoder_set_compression_level(FLAC__StreamEncoder *e, uint32_t value)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return false;
	fb200_encoder_config &c = e->protected_->cfg, t;
	fb200_encoder_config_preset(&t, c.channels, c.bits_per_sample, c.sample_rate, value, c.blocksize);
	// the preset touches exactly these fields (stream_encoder.c:1873-1904)
	c.do_mid_side_stereo = t.do_mid_side_stereo; c.loose_mid_side_stereo = t.loose_mid_side_stereo;
	c.max_lpc_order = t.max_lpc_order; c.qlp_coeff_precision = 0; c.do_qlp_coeff_prec_search = 0;
	c.do_exhaustive_model_search = 0; c.min_residual_partition_order = 0; c.max_residual_partition_order = t.max_residual_partition_order;
	c.num_apodizations = t.num_apodizations;
	memcpy(c.apodizations, t.apodizations, sizeof c.apodizations);
	e->protected_->rice_parameter_search_dist = 0;
	return true;
}

FLAC__bool FLAC__stream_encoder_set_apodization(FLAC__StreamEncoder *e, const char *spec)
{
	// stream_encoder.c:1940-2065; the parser lives with the engine configuration (encoder.cu)
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return false;
	return fb200_encoder_config_set_apodization(&e->protected_->cfg, spec) == FB200_OK;
}

FLAC__bool FLAC__stream_encoder_set_metadata(FLAC__StreamEncoder *e, FLAC__StreamMetadata **metadata, uint32_t num_blocks)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return false;
	e->protected_->metadata = num_blocks ? metadata : nullptr;   // client keeps ownership until finish (stream_encoder.h:1239-1262)
	e->protected_->num_metadata_blocks = metadata ? num_blocks : 0;
	return true;
}

FLAC__bool FLAC__stream_encoder_get_do_md5(const FLAC__StreamEncoder *e) { return e->protected_->do_md5; }
FLAC__StreamEncoderState FLAC__stream_encoder_get_state(const FLAC__StreamEncoder *e) { return e->protected_->state; }
// the verify decoder is the batch decoder of the same library: its failures surface as encoder states (stream_encoder.h:1311);
// as a decoder object it is always searching for the next frame
FLAC__StreamDecoderState FLAC__stream_encoder_get_verify_decoder_state(const FLAC__StreamEncoder *e)
{
	return e->protected_->verify ? FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC : FLAC__STREAM_DECODER_UNINITIALIZED;
}
const char *FLAC__stream_encoder_get_resolved_state_string(const FLAC__StreamEncoder *e) { return FLAC__StreamEncoderStateString[e->protected_->state]; }
void FLAC__stream_encoder_get_verify_decoder_error_stats(const FLAC__StreamEncoder *e, FLAC__uint64 *absolute_sample, uint32_t *frame_number, uint32_t *channel, uint32_t *sample, FLAC__int32 *expected, FLAC__int32 *got)
{
	const FLAC__StreamEncoderPrivate *q = e->private_;
	if(absolute_sample) *absolute_sample = q->v_abs_sample;
	if(frame_number) *frame_number = q->v_frame;
	if(channel) *channel = q->v_channel;
	if(sample) *sample = q->v_sample;
	if(expected) *expected = q->v_expected;
	if(got) *got = q->v_got;
}
FLAC__bool FLAC__stream_encoder_get_verify(const FLAC__StreamEncoder *e) { return e->protected_->verify; }
FLAC__bool FLAC__stream_encoder_get_streamable_subset(const FLAC__StreamEncoder *e) { return e->protected_->streamable_subset; }
uint32_t FLAC__stream_encoder_get_channels(const FLAC__StreamEncoder *e) { return e->protected_->cfg.channels; }
uint32_t FLAC__stream_encoder_get_bits_per_sample(const FLAC__StreamEncoder *e) { return e->protected_->cfg.bits_per_sample; }
uint32_t FLAC__stream_encoder_get_sample_rate(const FLAC__StreamEncoder *e) { return e->protected_->cfg.sample_rate; }
uint32_t FLAC__stream_encoder_get_blocksize(const FLAC__StreamEncoder *e) { return e->protected_->cfg.blocksize; }
FLAC__bool FLAC__stream_encoder_get_do_mid_side_stereo(const FLAC__StreamEncoder *e) { return e->protected_->cfg.do_mid_side_stereo; }
FLAC__bool FLAC__stream_encoder_get_loose_mid_side_stereo(const FLAC__StreamEncoder *e) { return e->protected_->cfg.loose_mid_side_stereo; }
uint32_t FLAC__stream_encoder_get_max_lpc_order(const FLAC__StreamEncoder *e) { return e->protected_->cfg.max_lpc_order; }
uint32_t FLAC__stream_encoder_get_qlp_coeff_precision(const FLAC__StreamEncoder *e) { return e->protected_->cfg.qlp_coeff_precision; }
FLAC__bool FLAC__stream_encoder_get_do_qlp_coeff_prec_search(const FLAC__StreamEncoder *e) { return e->protected_->cfg.do_qlp_coeff_prec_search; }
FLAC__bool FLAC__stream_encoder_get_do_escape_coding(const FLAC__StreamEncoder *e) { return e->protected_->do_escape_coding; }
FLAC__bool FLAC__stream_encoder_get_do_exhaustive_model_search(const FLAC__StreamEncoder *e) { return e->protected_->cfg.do_exhaustive_model_search; }
uint32_t FLAC__stream_encoder_get_min_residual_partition_order(const FLAC__StreamEncoder *e) { return e->protected_->cfg.min_residual_partition_order; }
uint32_t FLAC__stream_encoder_get_max_residual_partition_order(const FLAC__StreamEncoder *e) { return e->protected_->cfg.max_residual_partition_order; }
uint32_t FLAC__stream_encoder_get_num_threads(const FLAC__StreamEncoder *e) { return e->protected_->num_threads; }
uint32_t FLAC__stream_encoder_get_rice_parameter_search_dist(const FLAC__StreamEncoder *e) { return e->protected_->rice_parameter_search_dist; }
FLAC__uint64 FLAC__stream_encoder_get_total_samples_estimate(const FLAC__StreamEncoder *e) { return e->protected_->total_samples_estimate; }
FLAC__bool FLAC__stream_encoder_get_limit_min_bitrate(const FLAC__StreamEncoder *e) { return e->protected_->cfg.limit_min_bitrate; }

}  // extern "C"

// write `n` bytes through the client's write callback / FILE (stream_encoder.c:3038-3137 write_frame_)
static bool enc_emit(FLAC__StreamEncoder *e, const uint8_t *buf, size_t n, uint32_t samples, bool is_last_frame)
{
	FLAC__StreamEncoderPrivate *q = e->private_;
	(void)is_last_frame;
	if(samples > 0 && q->seek_table && q->seek_table->data.seek_table.num_points > 0) {
		// mark seek points that fall inside this frame (stream_encoder.c:3070-3103)
		const uint64_t frame_first = q->samples_written, frame_last = frame_first + samples - 1;
		FLAC__StreamMetadata_SeekTable &st = q->seek_table->data.seek_table;
		uint64_t pos = q->bytes_written;
		for(uint32_t i = q->first_seekpoint_to_check; i < st.num_points; i++) {
			const uint64_t test = st.points[i].sample_number;
			if(test > frame_last) break;
			if(test >= frame_first) {
				st.points[i].sample_number = frame_first;
				st.points[i].stream_offset = pos - q->audio_offset;
				st.points[i].frame_samples = samples;
				q->first_seekpoint_to_check++;
			}
			else q->first_seekpoint_to_check++;
		}
	}
	if(q->file) {
		if(fwrite(buf, 1, n, q->file) != n) { e->protected_->state = FLAC__STREAM_ENCODER_IO_ERROR; return false; }
	}
	else if(q->write_cb(e, buf, n, samples, q->frames_written, q->client_data) != FLAC__STREAM_ENCODER_WRITE_STATUS_OK) {
		e->protected_->state = FLAC__STREAM_ENCODER_CLIENT_ERROR;
		return false;
	}
	q->bytes_written += n;
	if(samples > 0) {
		q->samples_written += samples;
		q->frames_written++;
		q->si.min_framesize = q->si.min_framesize ? std::min<uint32_t>(q->si.min_framesize, (uint32_t)n) : (uint32_t)n;
		q->si.max_framesize = std::max<uint32_t>(q->si.max_framesize, (uint32_t)n);
		if(q->progress_cb) {
			const uint32_t bs = e->protected_->cfg.blocksize;
			const uint32_t est = (uint32_t)((e->protected_->total_samples_estimate + bs - 1) / bs);
			q->progress_cb(e, q->bytes_written, q->samples_written, q->frames_written, est, q->client_data);
		}
	}
	return true;
}

// encode everything pending (process_frame_ for a whole batch)
static bool enc_flush(FLAC__StreamEncoder *e)
{
	FLAC__StreamEncoderPrivate *q = e->private_;
	if(q->pending_samples == 0) return true;
	const fb200_encoder_config &c = e->protected_->cfg;
	const uint32_t bs = c.blocksize, ch = c.channels;
	const uint64_t nfr = (q->pending_samples + bs - 1) / bs;
	const size_t cap = (size_t)nfr * fb200_encoder_max_frame_bytes(q->gpu) + 64;
	if(q->frames.size() < cap) q->frames.resize(cap);
	if(q->offsets.size() < nfr + 1) q->offsets.resize(nfr + 1);
	uint32_t nframes = 0;
	// the batch goes to the device as packed 16-/24-bit PCM (half / three quarters of the int32 traffic), widened there
	if(fb200_encode_host_packed(q->gpu, q->pending_packed.data(), q->pack_bytes, q->pending_samples, q->frames_written, q->frames.data(), q->frames.size(), q->offsets.data(), &nframes) != FB200_OK) {
		e->protected_->state = FLAC__STREAM_ENCODER_FRAMING_ERROR;
		return false;
	}
	if(e->protected_->verify) {
		// --verify: decode what was just produced (on the GPU) and compare with the input (stream_encoder.c:5155-5240)
		q->verify_pcm.resize((size_t)nframes * bs * ch);
		uint64_t ns = 0;
		uint32_t bad = 0;
		if(fb200_decode_host(q->vdec, q->frames.data(), q->offsets.data(), nframes, q->verify_pcm.data(), (uint64_t)nframes * bs, &ns, &bad) != FB200_OK || bad) {
			e->protected_->state = FLAC__STREAM_ENCODER_VERIFY_DECODER_ERROR;
			return false;
		}
		for(size_t i = 0; i < (size_t)q->pending_samples * ch; i++)
			if(q->verify_pcm[i] != q->pending[i]) {
				q->v_abs_sample = q->samples_written + i / ch;
				q->v_frame = q->frames_written + (uint32_t)((i / ch) / bs);
				q->v_channel = (uint32_t)(i % ch);
				q->v_sample = (uint32_t)((i / ch) % bs);
				q->v_expected = q->pending[i]; q->v_got = q->verify_pcm[i];
				e->protected_->state = FLAC__STREAM_ENCODER_VERIFY_MISMATCH_IN_AUDIO_DATA;
				return false;
			}
	}
	uint64_t left = q->pending_samples;
	for(uint32_t i = 0; i < nframes; i++) {
		const uint32_t samples = (uint32_t)std::min<uint64_t>(bs, left);
		left -= samples;
		if(!enc_emit(e, q->frames.data() + q->offsets[i], (size_t)(q->offsets[i + 1] - q->offsets[i]), samples, false)) return false;
	}
	q->pending_samples = 0;
	return true;
}

static FLAC__StreamEncoderInitStatus enc_init_common(FLAC__StreamEncoder *e, bool is_ogg)
{
	FLAC__StreamEncoderProtected *p = e->protected_;
	FLAC__StreamEncoderPrivate *q = e->private_;
	fb200_encoder_config &c = p->cfg;
	if(p->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	if(is_ogg) return FLAC__STREAM_ENCODER_INIT_STATUS_UNSUPPORTED_CONTAINER;  // as the reference without libogg (:726)
	if(!q->file && (!q->write_cb || (q->seek_cb && !q->tell_cb))) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_CALLBACKS;
	// ---- the reference's validation order (stream_encoder.c:731-830)
	if(c.channels == 0 || c.channels > FLAC__MAX_CHANNELS) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_NUMBER_OF_CHANNELS;
	if(c.channels != 2) { c.do_mid_side_stereo = 0; c.loose_mid_side_stereo = 0; }
	else if(!c.do_mid_side_stereo) c.loose_mid_side_stereo = 0;
	if(c.bits_per_sample < FLAC__MIN_BITS_PER_SAMPLE || c.bits_per_sample > FLAC__MAX_BITS_PER_SAMPLE) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_BITS_PER_SAMPLE;
	if(c.sample_rate == 0 || c.sample_rate > FLAC__MAX_SAMPLE_RATE) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_SAMPLE_RATE;
	if(c.blocksize == 0) c.blocksize = c.max_lpc_order == 0 ? 1152 : 4096;
	if(c.blocksize < FLAC__MIN_BLOCK_SIZE || c.blocksize > FLAC__MAX_BLOCK_SIZE) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_BLOCK_SIZE;
	if(c.max_lpc_order > FLAC__MAX_LPC_ORDER) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_MAX_LPC_ORDER;
	if(c.blocksize < c.max_lpc_order) return FLAC__STREAM_ENCODER_INIT_STATUS_BLOCK_SIZE_TOO_SMALL_FOR_LPC_ORDER;
	if(c.qlp_coeff_precision != 0 && (c.qlp_coeff_precision < FLAC__MIN_QLP_COEFF_PRECISION || c.qlp_coeff_precision > FLAC__MAX_QLP_COEFF_PRECISION))
		return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_QLP_COEFF_PRECISION;
	if(p->streamable_subset) {
		// format.c FLAC__format_blocksize_is_subset / sample_rate_is_subset, stream_encoder.c:806-830
		const bool rate_ok = c.sample_rate <= 655350 && (c.sample_rate <= 65535 || c.sample_rate % 10 == 0 || c.sample_rate % 1000 == 0 ||
		                     c.sample_rate == 88200 || c.sample_rate == 176400 || c.sample_rate == 192000 || c.sample_rate == 96000);
		const uint32_t b = c.bits_per_sample;
		if(c.blocksize > 16384 || (c.sample_rate <= 48000 && c.blocksize > FLAC__SUBSET_MAX_BLOCK_SIZE_48000HZ) || !rate_ok ||
		   !(b == 8 || b == 12 || b == 16 || b == 20 || b == 24 || b == 32) || c.max_residual_partition_order > FLAC__SUBSET_MAX_RICE_PARTITION_ORDER ||
		   (c.sample_rate <= 48000 && c.max_lpc_order > FLAC__SUBSET_MAX_LPC_ORDER_48000HZ))
			return FLAC__STREAM_ENCODER_INIT_STATUS_NOT_STREAMABLE;
	}
	// metadata sanity (stream_encoder.c:838-925, abridged): no STREAMINFO, at most one SEEKTABLE / VORBIS_COMMENT
	bool has_vc = false;
	q->seek_table = nullptr;
	for(uint32_t i = 0; i < p->num_metadata_blocks; i++) {
		const FLAC__StreamMetadata *m = p->metadata[i];
		if(!m || m->type == FLAC__METADATA_TYPE_STREAMINFO) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_METADATA;
		if(m->type == FLAC__METADATA_TYPE_SEEKTABLE) {
			if(q->seek_table) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_METADATA;
			q->seek_table = p->metadata[i];
		}
		if(m->type == FLAC__METADATA_TYPE_VORBIS_COMMENT) {
			if(has_vc) return FLAC__STREAM_ENCODER_INIT_STATUS_INVALID_METADATA;
			has_vc = true;
		}
	}
	if(c.num_apodizations == 0) return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR;

	// ---- the engine (no CPU fallback)
	q->batch = batch_blocks();
	if(fb200::encoder_create(&c, 0, q->batch, true, &q->gpu) != FB200_OK) return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR;
	q->batch = fb200::encoder_capacity(q->gpu);  // tiled configurations: at most the tiled sample budget per batch
	fb200_encoder_get_config(q->gpu, &c);  // resolved blocksize / qlp precision, as the reference's getters report after init
	if(p->verify) {
		fb200_decoder_config dc = {c.channels, c.bits_per_sample, c.sample_rate, c.blocksize};
		if(fb200_decoder_create(&dc, 0, q->batch, &q->vdec) != FB200_OK) { enc_release(e); return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR; }
	}
	q->pending.resize(p->verify ? (size_t)q->batch * c.blocksize * c.channels : 0);
	q->pack_bytes = c.bits_per_sample <= 16 ? 2 : 3;
	q->pending_packed.resize((size_t)q->batch * c.blocksize * c.channels * q->pack_bytes);
	q->pending_samples = 0;
	q->md5.init();
	q->frames_written = 0; q->samples_written = 0; q->bytes_written = 0; q->first_seekpoint_to_check = 0;
	q->streaminfo_offset = q->seektable_offset = q->audio_offset = 0;
	memset(&q->si, 0, sizeof q->si);
	q->si.min_blocksize = q->si.max_blocksize = c.blocksize;
	q->si.sample_rate = c.sample_rate; q->si.channels = c.channels; q->si.bits_per_sample = c.bits_per_sample;
	q->si.total_samples = p->total_samples_estimate;
	p->state = FLAC__STREAM_ENCODER_OK;

	// ---- stream header: "fLaC", STREAMINFO, [default VORBIS_COMMENT], client blocks (stream_encoder.c:1341-1428)
	std::vector<uint8_t> blk;
	const uint8_t sync[4] = {'f', 'L', 'a', 'C'};
	if(!enc_emit(e, sync, 4, 0, false)) return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR;
	FLAC__StreamMetadata sim;
	memset(&sim, 0, sizeof sim);
	sim.type = FLAC__METADATA_TYPE_STREAMINFO; sim.length = FLAC__STREAM_METADATA_STREAMINFO_LENGTH; sim.data.stream_info = q->si;
	q->streaminfo_offset = q->bytes_written;
	serialize_metadata(&sim, false, FLAC__VENDOR_STRING, blk);
	if(!enc_emit(e, blk.data(), blk.size(), 0, false)) return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR;
	if(!has_vc) {
		FLAC__StreamMetadata vc;
		memset(&vc, 0, sizeof vc);
		vc.type = FLAC__METADATA_TYPE_VORBIS_COMMENT;
		serialize_metadata(&vc, p->num_metadata_blocks == 0, FLAC__VENDOR_STRING, blk);
		if(!enc_emit(e, blk.data(), blk.size(), 0, false)) return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR;
	}
	for(uint32_t i = 0; i < p->num_metadata_blocks; i++) {
		if(p->metadata[i] == q->seek_table) q->seektable_offset = q->bytes_written;
		if(!serialize_metadata(p->metadata[i], i + 1 == p->num_metadata_blocks, FLAC__VENDOR_STRING, blk)) { p->state = FLAC__STREAM_ENCODER_FRAMING_ERROR; return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR; }
		if(!enc_emit(e, blk.data(), blk.size(), 0, false)) return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR;
	}
	q->audio_offset = q->bytes_written;
	return FLAC__STREAM_ENCODER_INIT_STATUS_OK;
}

extern "C" {

FLAC__StreamEncoderInitStatus FLAC__stream_encoder_init_stream(FLAC__StreamEncoder *e, FLAC__StreamEncoderWriteCallback write_callback, FLAC__StreamEncoderSeekCallback seek_callback, FLAC__StreamEncoderTellCallback tell_callback, FLAC__StreamEncoderMetadataCallback metadata_callback, void *client_data)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	FLAC__StreamEncoderPrivate *q = e->private_;
	q->write_cb = write_callback; q->seek_cb = seek_callback; q->tell_cb = tell_callback; q->metadata_cb = metadata_callback;
	q->progress_cb = nullptr; q->client_data = client_data; q->file = nullptr;
	return enc_init_common(e, false);
}

FLAC__StreamEncoderInitStatus FLAC__stream_encoder_init_ogg_stream(FLAC__StreamEncoder *e, FLAC__StreamEncoderReadCallback, FLAC__StreamEncoderWriteCallback, FLAC__StreamEncoderSeekCallback, FLAC__StreamEncoderTellCallback, FLAC__StreamEncoderMetadataCallback, void *)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	return FLAC__STREAM_ENCODER_INIT_STATUS_UNSUPPORTED_CONTAINER;
}

FLAC__StreamEncoderInitStatus FLAC__stream_encoder_init_FILE(FLAC__StreamEncoder *e, FILE *file, FLAC__StreamEncoderProgressCallback progress_callback, void *client_data)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	if(!file) { e->protected_->state = FLAC__STREAM_ENCODER_IO_ERROR; return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR; }
	FLAC__StreamEncoderPrivate *q = e->private_;
	q->write_cb = nullptr; q->seek_cb = nullptr; q->tell_cb = nullptr; q->metadata_cb = nullptr;
	q->progress_cb = progress_callback; q->client_data = client_data; q->file = file; q->owns_file = true;
	const FLAC__StreamEncoderInitStatus st = enc_init_common(e, false);
	if(st != FLAC__STREAM_ENCODER_INIT_STATUS_OK) { if(q->file && q->owns_file) fclose(q->file); q->file = nullptr; }
	return st;
}

FLAC__StreamEncoderInitStatus FLAC__stream_encoder_init_ogg_FILE(FLAC__StreamEncoder *e, FILE *, FLAC__StreamEncoderProgressCallback, void *)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	return FLAC__STREAM_ENCODER_INIT_STATUS_UNSUPPORTED_CONTAINER;
}

FLAC__StreamEncoderInitStatus FLAC__stream_encoder_init_file(FLAC__StreamEncoder *e, const char *filename, FLAC__StreamEncoderProgressCallback progress_callback, void *client_data)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	FILE *f = filename ? fopen(filename, "w+b") : stdout;
	if(!f) { e->protected_->state = FLAC__STREAM_ENCODER_IO_ERROR; return FLAC__STREAM_ENCODER_INIT_STATUS_ENCODER_ERROR; }
	const FLAC__StreamEncoderInitStatus st = FLAC__stream_encoder_init_FILE(e, f, progress_callback, client_data);
	if(!filename) e->private_->owns_file = false;
	return st;
}

FLAC__StreamEncoderInitStatus FLAC__stream_encoder_init_ogg_file(FLAC__StreamEncoder *e, const char *, FLAC__StreamEncoderProgressCallback, void *)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_UNINITIALIZED) return FLAC__STREAM_ENCODER_INIT_STATUS_ALREADY_INITIALIZED;
	return FLAC__STREAM_ENCODER_INIT_STATUS_UNSUPPORTED_CONTAINER;
}

FLAC__bool FLAC__stream_encoder_process_interleaved(FLAC__StreamEncoder *e, const FLAC__int32 buffer[], uint32_t samples)
{
	FLAC__StreamEncoderProtected *p = e->protected_;
	FLAC__StreamEncoderPrivate *q = e->private_;
	if(p->state != FLAC__STREAM_ENCODER_OK) return false;
	const uint32_t ch = p->cfg.channels, bps = p->cfg.bits_per_sample;
	const FLAC__int32 smax = INT32_MAX >> (32 - bps), smin = INT32_MIN >> (32 - bps);
	const uint64_t cap = (uint64_t)q->batch * p->cfg.blocksize;
	uint32_t done = 0;
	while(done < samples) {
		const uint32_t n = (uint32_t)std::min<uint64_t>(samples - done, cap - q->pending_samples);
		const FLAC__int32 *src = buffer + (size_t)done * ch;
		uint8_t *pk = q->pending_packed.data() + (size_t)q->pending_samples * ch * q->pack_bytes;
		if(q->pack_bytes == 2) {
			for(size_t i = 0; i < (size_t)n * ch; i++) {
				const FLAC__int32 v = src[i];
				if(v < smin || v > smax) { p->state = FLAC__STREAM_ENCODER_CLIENT_ERROR; return false; }  // stream_encoder.c:2586-2596
				pk[2 * i] = (uint8_t)v; pk[2 * i + 1] = (uint8_t)(v >> 8);
			}
		}
		else {
			for(size_t i = 0; i < (size_t)n * ch; i++) {
				const FLAC__int32 v = src[i];
				if(v < smin || v > smax) { p->state = FLAC__STREAM_ENCODER_CLIENT_ERROR; return false; }
				pk[3 * i] = (uint8_t)v; pk[3 * i + 1] = (uint8_t)(v >> 8); pk[3 * i + 2] = (uint8_t)(v >> 16);
			}
		}
		if(p->verify) memcpy(q->pending.data() + (size_t)q->pending_samples * ch, src, (size_t)n * ch * sizeof(FLAC__int32));
		if(p->do_md5) q->md5.update_samples(src, (size_t)n * ch, (bps + 7) / 8);
		q->pending_samples += n;
		done += n;
		if(q->pending_samples == cap && !enc_flush(e)) return false;
	}
	return true;
}

FLAC__bool FLAC__stream_encoder_process(FLAC__StreamEncoder *e, const FLAC__int32 *const buffer[], uint32_t samples)
{
	if(e->protected_->state != FLAC__STREAM_ENCODER_OK) return false;
	const uint32_t ch = e->protected_->cfg.channels;
	std::vector<FLAC__int32> tmp;
	const uint32_t chunk = 16384;
	for(uint32_t done = 0; done < samples; done += chunk) {
		const uint32_t n = std::min(chunk, samples - done);
		tmp.resize((size_t)n * ch);
		for(uint32_t c = 0; c < ch; c++)
			for(uint32_t i = 0; i < n; i++) tmp[(size_t)i * ch + c] = buffer[c][done + i];
		if(!FLAC__stream_encoder_process_interleaved(e, tmp.data(), n)) return false;
	}
	return true;
}

FLAC__bool FLAC__stream_encoder_finish(FLAC__StreamEncoder *e)
{
	FLAC__StreamEncoderProtected *p = e->protected_;
	FLAC__StreamEncoderPrivate *q = e->private_;
	if(p->state == FLAC__STREAM_ENCODER_UNINITIALIZED) return true;
	bool error = false;
	if(p->state == FLAC__STREAM_ENCODER_OK) {
		if(!enc_flush(e)) error = true;  // includes the short last block (stream_encoder.c:1703-1711)
	}
	else error = true;
	if(!error || p->state == FLAC__STREAM_ENCODER_OK) {
		// STREAMINFO / SEEKTABLE patch-up (update_metadata_, stream_encoder.c:3139-3300)
		if(p->do_md5) q->md5.final(q->si.md5sum);
		q->si.total_samples = q->samples_written & 0xFFFFFFFFFull;
		if(q->si.total_samples < p->cfg.blocksize && q->si.total_samples > 0) { /* single short frame */ }
		ByteWriter w;
		put_streaminfo(w, q->si);
		ByteWriter stw;
		if(q->seek_table) {
			// update_metadata_ (stream_encoder.c:3250-3259): points past the end become placeholders, then FLAC__format_seektable_sort
			// (format.c:281-314) sorts, uniquifies and fills the freed places with placeholders. The sort is stable: the reference's
			// qsort leaves the order among equal keys to the C library, and template order is what fb200_encode_flac_files_* write.
			FLAC__StreamMetadata_SeekTable &st = q->seek_table->data.seek_table;
			const uint64_t ph = ~0ull;  // FLAC__STREAM_METADATA_SEEKPOINT_PLACEHOLDER
			for(uint32_t i = 0; i < st.num_points; i++)
				if(st.points[i].sample_number > q->si.total_samples) st.points[i].sample_number = ph;
			std::stable_sort(st.points, st.points + st.num_points,
			                 [](const FLAC__StreamMetadata_SeekPoint &a, const FLAC__StreamMetadata_SeekPoint &b) { return a.sample_number < b.sample_number; });
			uint32_t j = 0;
			for(uint32_t i = 0; i < st.num_points; i++) {
				if(st.points[i].sample_number != ph && j > 0 && st.points[i].sample_number == st.points[j - 1].sample_number) continue;
				st.points[j++] = st.points[i];
			}
			for(; j < st.num_points; j++) st.points[j] = FLAC__StreamMetadata_SeekPoint{ph, 0, 0};
			for(uint32_t i = 0; i < st.num_points; i++) {
				stw.u(st.points[i].sample_number, 8);
				stw.u(st.points[i].stream_offset, 8);
				stw.u(st.points[i].frame_samples, 2);
			}
		}
		if(q->file) {
			const off_t end = ftello(q->file);
			if(end >= 0 && fseeko(q->file, (off_t)q->streaminfo_offset + 4, SEEK_SET) == 0) {
				if(fwrite(w.v.data(), 1, w.v.size(), q->file) != w.v.size()) error = true;
				if(q->seek_table && q->seektable_offset && fseeko(q->file, (off_t)q->seektable_offset + 4, SEEK_SET) == 0)
					if(fwrite(stw.v.data(), 1, stw.v.size(), q->file) != stw.v.size()) error = true;
				fseeko(q->file, end, SEEK_SET);
			}
		}
		else if(q->seek_cb) {
			if(q->seek_cb(e, q->streaminfo_offset + 4, q->client_data) == FLAC__STREAM_ENCODER_SEEK_STATUS_OK) {
				if(q->write_cb(e, w.v.data(), w.v.size(), 0, 0, q->client_data) != FLAC__STREAM_ENCODER_WRITE_STATUS_OK) error = true;
				if(q->seek_table && q->seektable_offset && q->seek_cb(e, q->seektable_offset + 4, q->client_data) == FLAC__STREAM_ENCODER_SEEK_STATUS_OK)
					if(q->write_cb(e, stw.v.data(), stw.v.size(), 0, 0, q->client_data) != FLAC__STREAM_ENCODER_WRITE_STATUS_OK) error = true;
			}
		}
		if(q->metadata_cb) {
			FLAC__StreamMetadata sim;
			memset(&sim, 0, sizeof sim);
			sim.type = FLAC__METADATA_TYPE_STREAMINFO; sim.length = FLAC__STREAM_METADATA_STREAMINFO_LENGTH; sim.data.stream_info = q->si;
			q->metadata_cb(e, &sim, q->client_data);
		}
	}
	enc_release(e);
	enc_set_defaults(e);  // settings return to their defaults (stream_encoder.h:225-227)
	if(!error) p->state = FLAC__STREAM_ENCODER_UNINITIALIZED;
	const bool ok = !error;
	if(error && p->state == FLAC__STREAM_ENCODER_OK) p->state = FLAC__STREAM_ENCODER_IO_ERROR;
	if(ok) p->state = FLAC__STREAM_ENCODER_UNINITIALIZED;
	return ok;
}

}  // extern "C"

// ================================================================== decoder object

struct FrameIndexEntry : fb200::FrameHeader {
	uint64_t offset;      // byte offset into the audio buffer
	uint32_t length;
};

struct FLAC__StreamDecoderProtected {
	FLAC__StreamDecoderState state;
	FLAC__bool md5_checking;
	uint32_t channels, bits_per_sample, sample_rate, blocksize;
	FLAC__ChannelAssignment channel_assignment;
};

struct FLAC__StreamDecoderPrivate {
	FLAC__StreamDecoderReadCallback read_cb;
	FLAC__StreamDecoderSeekCallback seek_cb;
	FLAC__StreamDecoderTellCallback tell_cb;
	FLAC__StreamDecoderLengthCallback length_cb;
	FLAC__StreamDecoderEofCallback eof_cb;
	FLAC__StreamDecoderWriteCallback write_cb;
	FLAC__StreamDecoderMetadataCallback metadata_cb;
	FLAC__StreamDecoderErrorCallback error_cb;
	void *client_data;
	FILE *file;
	bool owns_file;
	bool respond[128];
	std::vector<uint8_t> in;     // everything read so far that was not consumed
	size_t in_pos;
	uint64_t consumed_before_in;  // bytes dropped from the front of `in` so far
	bool eof, metadata_done, indexed, has_streaminfo, did_seek;
	FLAC__StreamMetadata_StreamInfo si;
	std::vector<uint8_t> audio;  // all frame bytes (+ slack)
	uint64_t audio_offset;       // stream byte offset of audio[0] (for get_decode_position)
	std::vector<FrameIndexEntry> index;
	std::vector<uint64_t> first_sample;  // per frame
	size_t next_frame;
	uint64_t skip_samples;       // after a seek: samples to drop from the next frame
	fb200_decoder *gpu;
	// decoded batch
	size_t batch_first, batch_count;
	std::vector<int32_t> pcm;
	std::vector<uint64_t> offs;
	std::vector<uint32_t> batch_status, batch_bytes;       // per frame of the decoded batch
	std::vector<fb200_subframe_info> batch_sub;           // per (frame, channel) of the decoded batch
	std::vector<int32_t> residual;                        // scratch: residuals of the frame being delivered (FLAC__Subframe.residual)
	uint64_t expect_pos;          // byte offset (in `audio`) where the next frame should start
	bool lost_sync_reported;
	FLAC__FrameHeader last_header;  // the header of the last frame written, silence included (stream_decoder.c:3580-3581)
	bool last_set;
	bool error_sent;              // an error was reported while finding the frame now being delivered (error_has_been_sent)
	std::vector<int32_t> planar;
	MD5 md5;
	uint64_t samples_decoded;
};

static void dec_set_defaults(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	memset(q->respond, 0, sizeof q->respond);
	q->respond[FLAC__METADATA_TYPE_STREAMINFO] = true;  // stream_decoder.c:1557-1560
	d->protected_->md5_checking = false;
}

static void dec_release(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(q->gpu) { fb200_decoder_destroy(q->gpu); q->gpu = nullptr; }
	if(q->file && q->owns_file) fclose(q->file);
	q->file = nullptr;
	q->in.clear(); q->audio.clear(); q->index.clear(); q->first_sample.clear(); q->pcm.clear(); q->offs.clear(); q->planar.clear();
}

// pull more bytes from the client; returns false at end of stream / abort
static bool dec_fill(FLAC__StreamDecoder *d, size_t want)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	while(q->in.size() - q->in_pos < want && !q->eof) {
		const size_t chunk = std::max<size_t>(want, 1 << 20);
		const size_t old = q->in.size();
		q->in.resize(old + chunk);
		size_t got = chunk;
		if(q->file) {
			got = fread(q->in.data() + old, 1, chunk, q->file);
			if(got == 0) q->eof = true;
		}
		else {
			const FLAC__StreamDecoderReadStatus st = q->read_cb(d, q->in.data() + old, &got, q->client_data);
			if(st == FLAC__STREAM_DECODER_READ_STATUS_ABORT) { q->in.resize(old); d->protected_->state = FLAC__STREAM_DECODER_ABORTED; return false; }
			if(st == FLAC__STREAM_DECODER_READ_STATUS_END_OF_STREAM || got == 0) q->eof = true;
		}
		q->in.resize(old + got);
	}
	return q->in.size() - q->in_pos >= want;
}

// Frame index = the GPU front end's candidates (sync code + self-consistent header incl. CRC-8 at every byte position of the
// stream at once: fb200_decoder_index_host), kept when the header agrees with STREAMINFO. A candidate's END is not known
// here -- frames carry no length field -- and is not needed: the batch decode bounds every frame by the largest legal frame,
// finds its true length by parsing it and checks the CRC-16 over exactly that (fb200_decode_indexed_host). Junk between or
// after frames (ID3v1 / APE tags, padding) therefore costs nothing, and a corrupt frame loses only itself.
static bool dec_build_index(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	const uint8_t *a = q->audio.data();
	const size_t n = q->audio.size() - 64;  // slack at the end
	std::vector<uint64_t> cand;
	uint32_t ncand = 0;
	size_t cap = std::max<size_t>(1 << 16, n / 256);
	for(;;) {
		cand.resize(cap);
		const int rc = fb200_decoder_index_host(q->gpu, a, n, cand.data(), (uint32_t)std::min<size_t>(cap, 0xffffffffu), &ncand);
		if(rc == FB200_OK) break;
		if(rc != FB200_ERR_OUTPUT_TOO_SMALL || cap >= n) return false;
		cap = std::min(n, cap * 8);
	}
	uint64_t sample = 0;
	const bool fixed_bs = q->si.min_blocksize == q->si.max_blocksize && q->si.max_blocksize;
	for(uint32_t i = 0; i < ncand; i++) {
		FrameIndexEntry fe;
		memset(&fe, 0, sizeof fe);
		const size_t pos = (size_t)cand[i];
		if(fb200::parse_frame_header(a + pos, n - pos, q->si.sample_rate, q->si.bits_per_sample, fe).status != fb200::DEC_OK) continue;
		if(fe.channels != q->si.channels || fe.bps != q->si.bits_per_sample || fe.blocksize > (q->si.max_blocksize ? q->si.max_blocksize : 65535u)) continue;
		fe.offset = pos; fe.length = 0;
		q->index.push_back(fe);
		const uint64_t fs = fe.variable ? fe.number : (fixed_bs ? fe.number * q->si.max_blocksize : sample);
		q->first_sample.push_back(fs);
		sample = fs + fe.blocksize;
	}
	q->indexed = true;
	return true;
}

static bool dec_read_metadata(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(q->metadata_done) return true;
	// optional ID3v2 tag, then "fLaC" (stream_decoder.c:1654-1742)
	if(!dec_fill(d, 4)) { d->protected_->state = FLAC__STREAM_DECODER_END_OF_STREAM; return false; }
	if(memcmp(q->in.data() + q->in_pos, "ID3", 3) == 0) {
		if(!dec_fill(d, 10)) return false;
		const size_t skip = fb200::id3v2_tag_bytes(q->in.data() + q->in_pos);
		if(!dec_fill(d, skip + 4)) return false;
		q->in_pos += skip;
	}
	if(memcmp(q->in.data() + q->in_pos, "fLaC", 4) != 0) {
		// the reference also accepts streams that start at a frame; here a STREAMINFO is required
		if(q->error_cb) q->error_cb(d, FLAC__STREAM_DECODER_ERROR_STATUS_LOST_SYNC, q->client_data);
		d->protected_->state = FLAC__STREAM_DECODER_ABORTED;
		return false;
	}
	q->in_pos += 4;
	bool last = false;
	while(!last) {
		if(!dec_fill(d, 4)) { d->protected_->state = FLAC__STREAM_DECODER_END_OF_STREAM; return false; }
		const fb200::MetaBlockHeader h = fb200::metadata_block_header(q->in.data() + q->in_pos);
		last = h.last;
		const uint32_t type = h.type, len = h.length;
		if(!dec_fill(d, 4 + (size_t)len)) { d->protected_->state = FLAC__STREAM_DECODER_END_OF_STREAM; return false; }
		const uint8_t *b = q->in.data() + q->in_pos + 4;
		FLAC__StreamMetadata m;
		memset(&m, 0, sizeof m);
		m.type = type <= 6 ? (FLAC__MetadataType)type : FLAC__METADATA_TYPE_UNDEFINED;
		m.is_last = last; m.length = len;
		std::vector<FLAC__StreamMetadata_SeekPoint> pts;
		std::vector<FLAC__StreamMetadata_VorbisComment_Entry> ents;
		std::vector<std::vector<uint8_t>> strs;
		bool deliver = q->respond[type < 128 ? type : 127] && q->metadata_cb;
		if(type == FLAC__METADATA_TYPE_STREAMINFO && len >= 34) {
			FLAC__StreamMetadata_StreamInfo &s = m.data.stream_info;
			fb200::get_streaminfo(b, s);
			q->si = s; q->has_streaminfo = true;
			d->protected_->channels = s.channels; d->protected_->bits_per_sample = s.bits_per_sample; d->protected_->sample_rate = s.sample_rate;
			d->protected_->blocksize = s.max_blocksize;
		}
		else if(type == FLAC__METADATA_TYPE_APPLICATION && len >= 4) {
			memcpy(m.data.application.id, b, 4);
			m.data.application.data = len > 4 ? const_cast<uint8_t *>(b + 4) : nullptr;
		}
		else if(type == FLAC__METADATA_TYPE_SEEKTABLE) {
			pts.resize(len / 18);
			for(size_t i = 0; i < pts.size(); i++) {
				const uint8_t *s = b + 18 * i;
				pts[i].sample_number = fb200::be64(s); pts[i].stream_offset = fb200::be64(s + 8); pts[i].frame_samples = fb200::be(s + 16, 2);
			}
			m.data.seek_table.num_points = (uint32_t)pts.size(); m.data.seek_table.points = pts.data();
		}
		else if(type == FLAC__METADATA_TYPE_VORBIS_COMMENT && len >= 8) {
			size_t pos = 0;
			auto rd = [&](uint32_t &v) { if(pos + 4 > len) return false; v = fb200::le32(b + pos); pos += 4; return true; };
			uint32_t vl = 0, nc = 0;
			bool ok = rd(vl) && pos + vl <= len;
			if(ok) { strs.emplace_back(b + pos, b + pos + vl); strs.back().push_back(0); pos += vl; ok = rd(nc); }
			for(uint32_t i = 0; ok && i < nc; i++) {
				uint32_t l = 0;
				ok = rd(l) && pos + l <= len;
				if(ok) { strs.emplace_back(b + pos, b + pos + l); strs.back().push_back(0); pos += l; }
			}
			if(ok) {
				m.data.vorbis_comment.vendor_string.length = (uint32_t)strs[0].size() - 1; m.data.vorbis_comment.vendor_string.entry = strs[0].data();
				ents.resize(strs.size() - 1);
				for(size_t i = 1; i < strs.size(); i++) { ents[i - 1].length = (uint32_t)strs[i].size() - 1; ents[i - 1].entry = strs[i].data(); }
				m.data.vorbis_comment.num_comments = (uint32_t)ents.size(); m.data.vorbis_comment.comments = ents.data();
			}
			else { if(q->error_cb) q->error_cb(d, FLAC__STREAM_DECODER_ERROR_STATUS_BAD_METADATA, q->client_data); deliver = false; }
		}
		else if(type == FLAC__METADATA_TYPE_PADDING) { /* nothing */ }
		else {
			// CUESHEET / PICTURE / unknown: handed over as raw bytes (FLAC__StreamMetadata_Unknown layout)
			m.type = type <= 6 ? (FLAC__MetadataType)type : FLAC__METADATA_TYPE_UNDEFINED;
			if(type == FLAC__METADATA_TYPE_CUESHEET || type == FLAC__METADATA_TYPE_PICTURE) deliver = false;  // structured view not provided
			m.data.unknown.data = const_cast<uint8_t *>(b);
		}
		if(deliver) q->metadata_cb(d, &m, q->client_data);
		q->in_pos += 4 + (size_t)len;
	}
	if(!q->has_streaminfo) {
		if(q->error_cb) q->error_cb(d, FLAC__STREAM_DECODER_ERROR_STATUS_BAD_METADATA, q->client_data);
		d->protected_->state = FLAC__STREAM_DECODER_ABORTED;
		return false;
	}
	q->metadata_done = true;
	d->protected_->state = FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC;
	return true;
}

// read the rest of the stream, index it and create the engine
static bool dec_prepare_audio(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(q->indexed) return true;
	while(!q->eof) {
		if(!dec_fill(d, (q->in.size() - q->in_pos) + (4 << 20)) && d->protected_->state == FLAC__STREAM_DECODER_ABORTED) return false;
	}
	q->audio_offset = q->consumed_before_in + q->in_pos;
	q->audio.assign(q->in.begin() + (long)q->in_pos, q->in.end());
	q->audio.resize(q->audio.size() + 64, 0);
	q->in.clear(); q->in.shrink_to_fit(); q->in_pos = 0;
	const uint32_t bs = q->si.max_blocksize ? q->si.max_blocksize : 4096;
	if(q->si.bits_per_sample > 24) {
		if(q->error_cb) q->error_cb(d, FLAC__STREAM_DECODER_ERROR_STATUS_UNPARSEABLE_STREAM, q->client_data);
		d->protected_->state = FLAC__STREAM_DECODER_ABORTED;
		return false;
	}
	fb200_decoder_config dc = {q->si.channels, q->si.bits_per_sample, q->si.sample_rate, bs};
	if(fb200_decoder_create(&dc, 0, batch_blocks(), &q->gpu) != FB200_OK) {
		d->protected_->state = FLAC__STREAM_DECODER_MEMORY_ALLOCATION_ERROR;
		return false;
	}
	fb200_decoder_enable_subframe_info(q->gpu, 1);
	if(!dec_build_index(d)) {
		d->protected_->state = FLAC__STREAM_DECODER_MEMORY_ALLOCATION_ERROR;
		return false;
	}
	q->expect_pos = 0; q->lost_sync_reported = false;
	q->md5.init();
	return true;
}

// decode the batch that starts at index entry `first`
static bool dec_decode_batch(FLAC__StreamDecoder *d, size_t first)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	const size_t count = std::min<size_t>(batch_blocks(), q->index.size() - first);
	const uint32_t bs = q->si.max_blocksize ? q->si.max_blocksize : 4096, ch = q->si.channels;
	q->offs.resize(count);
	for(size_t i = 0; i < count; i++) q->offs[i] = q->index[first + i].offset;
	// how far a frame may reach: twice the verbatim worst case (STREAMINFO's max_framesize is advisory and may be absent);
	// the bound only limits how far a broken parse can run, the true length comes out of the parse
	const uint32_t max_fb = 64 + 2 * ch * (uint32_t)(((uint64_t)bs * (q->si.bits_per_sample + 2) + 7) / 8 + 64);
	q->pcm.resize(count * (size_t)bs * ch);
	q->batch_status.resize(count); q->batch_bytes.resize(count); q->batch_sub.resize(count * (size_t)ch);
	if(fb200_decode_indexed_host(q->gpu, q->offs.data(), (uint32_t)count, max_fb, q->audio.size() - 64, q->pcm.data(), (uint64_t)count * bs,
	                             q->batch_status.data(), q->batch_bytes.data()) != FB200_OK ||
	   fb200_decoder_get_subframe_info(q->gpu, q->batch_sub.data(), (uint32_t)count) != FB200_OK) {
		d->protected_->state = FLAC__STREAM_DECODER_ABORTED;
		return false;
	}
	q->batch_first = first; q->batch_count = count;
	return true;
}

static void dec_error(FLAC__StreamDecoder *d, FLAC__StreamDecoderErrorStatus status)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	q->error_sent = true;
	if(q->error_cb) q->error_cb(d, status, q->client_data);
}

// A gap in the sample numbers before the frame `next` (stream_decoder.c:2483-2554): MISSING_FRAME unless an error was already
// reported while finding `next`; then, when the last written frame agrees with `next` on rate, channels and bits per sample and
// has at least 16 samples, silence frames shaped like it (its header, the sample number advanced by its blocksize, the last one
// shortened), at most 5 seconds and 50 of its blocks. Past those caps the gap stays: the stream comes out shorter.
static bool dec_fill_gap(FLAC__StreamDecoder *d, const FrameIndexEntry &next, uint64_t next_sample)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(!q->last_set) return true;
	const FLAC__FrameHeader &last = q->last_header;
	if(last.number.sample_number + last.blocksize >= next_sample) return true;
	uint32_t need = (uint32_t)(next_sample - (last.number.sample_number + last.blocksize));  // uint32_t as in the reference
	if(!q->error_sent) dec_error(d, FLAC__STREAM_DECODER_ERROR_STATUS_MISSING_FRAME);
	if(last.sample_rate != next.sample_rate || last.channels != next.channels || last.bits_per_sample != next.bps || last.blocksize < 16)
		return true;
	need = std::min(need, 5 * last.sample_rate);
	need = std::min(need, 50 * last.blocksize);
	FLAC__Frame fr;
	memset(&fr, 0, sizeof fr);
	fr.header = last;
	for(uint32_t c = 0; c < last.channels; c++) fr.subframes[c].type = FLAC__SUBFRAME_TYPE_CONSTANT;
	std::vector<int32_t> zero((size_t)last.blocksize * last.channels, 0);
	const int32_t *chan[FLAC__MAX_CHANNELS];
	for(uint32_t c = 0; c < last.channels; c++) chan[c] = zero.data();
	while(need) {
		fr.header.number.sample_number += fr.header.blocksize;
		if(need < fr.header.blocksize) fr.header.blocksize = need;
		need -= fr.header.blocksize;
		d->protected_->blocksize = fr.header.blocksize;
		q->samples_decoded = fr.header.number.sample_number + fr.header.blocksize;
		if(d->protected_->md5_checking && !q->did_seek)
			q->md5.update_samples(zero.data(), (size_t)fr.header.blocksize * fr.header.channels, (fr.header.bits_per_sample + 7) / 8);
		q->last_header = fr.header;
		if(q->write_cb(d, &fr, chan, q->client_data) != FLAC__STREAM_DECODER_WRITE_STATUS_CONTINUE) {
			d->protected_->state = FLAC__STREAM_DECODER_ABORTED;
			return false;
		}
	}
	return true;
}

// hand one frame to the client (write_audio_frame_to_client_, stream_decoder.c:3578-3635); frames that fail are reported
// through the error callback and NOT delivered, like the reference (stream_decoder.c:2443-2590), and a gap they leave in the
// sample numbers is filled with the reference's silence frames
static bool dec_deliver_next(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	for(;;) {
		if(q->next_frame >= q->index.size()) { d->protected_->state = FLAC__STREAM_DECODER_END_OF_STREAM; return true; }
		if(q->batch_count == 0 || q->next_frame < q->batch_first || q->next_frame >= q->batch_first + q->batch_count)
			if(!dec_decode_batch(d, q->next_frame)) return false;
		const size_t bi = q->next_frame - q->batch_first;
		const FrameIndexEntry &fe = q->index[q->next_frame];
		const uint32_t st = q->batch_status[bi] & 0xffu;
		if(fe.offset < q->expect_pos && !q->did_seek) { q->next_frame++; continue; }  // a header look-alike inside the previous frame
		q->error_sent = false;  // the reference clears error_has_been_sent after every frame it reads, good or bad (:2556)
		if(st != 0) {
			// a broken frame (or a look-alike in junk): report once per damaged stretch, move on to the next candidate
			dec_error(d, st == 7 ? FLAC__STREAM_DECODER_ERROR_STATUS_FRAME_CRC_MISMATCH :
			             (st == 2 || st == 3) ? FLAC__STREAM_DECODER_ERROR_STATUS_BAD_HEADER :
			             st == 4 ? FLAC__STREAM_DECODER_ERROR_STATUS_UNPARSEABLE_STREAM :
			             st == 9 ? FLAC__STREAM_DECODER_ERROR_STATUS_OUT_OF_BOUNDS : FLAC__STREAM_DECODER_ERROR_STATUS_LOST_SYNC);
			q->next_frame++;
			continue;
		}
		if(fe.offset > q->expect_pos && !q->did_seek && q->expect_pos != 0)
			dec_error(d, FLAC__STREAM_DECODER_ERROR_STATUS_LOST_SYNC);  // junk between two frames
		q->expect_pos = fe.offset + q->batch_bytes[bi];
		if(!dec_fill_gap(d, fe, q->first_sample[q->next_frame])) return false;
		break;
	}
	const size_t bi = q->next_frame - q->batch_first;
	const FrameIndexEntry &fe = q->index[q->next_frame];
	const uint32_t bsmax = q->si.max_blocksize ? q->si.max_blocksize : 4096, ch = q->si.channels;
	const int32_t *src = q->pcm.data() + bi * (size_t)bsmax * ch;
	uint32_t bs = fe.blocksize;
	uint64_t first_sample = q->first_sample[q->next_frame];
	uint32_t skip = 0;
	if(q->skip_samples) { skip = (uint32_t)std::min<uint64_t>(q->skip_samples, bs); q->skip_samples = 0; }
	// total_samples from STREAMINFO truncates the last frame like the reference does (:3590-3600)
	if(q->si.total_samples && first_sample + bs > q->si.total_samples) bs = first_sample >= q->si.total_samples ? 0 : (uint32_t)(q->si.total_samples - first_sample);
	q->next_frame++;
	if(bs <= skip) return true;
	q->planar.resize((size_t)ch * bs);
	const int32_t *chan[FLAC__MAX_CHANNELS];
	for(uint32_t c = 0; c < ch; c++) {
		int32_t *dst = q->planar.data() + (size_t)c * bs;
		for(uint32_t i = 0; i < bs; i++) dst[i] = src[(size_t)i * ch + c];
		chan[c] = dst + skip;
	}
	FLAC__Frame fr;
	memset(&fr, 0, sizeof fr);
	fr.header.blocksize = bs - skip; fr.header.sample_rate = fe.sample_rate; fr.header.channels = ch;
	fr.header.channel_assignment = (FLAC__ChannelAssignment)fe.ca; fr.header.bits_per_sample = fe.bps;
	fr.header.number_type = FLAC__FRAME_NUMBER_TYPE_SAMPLE_NUMBER;  // the reference always hands out sample numbers (:2936-2944)
	fr.header.number.sample_number = first_sample + skip;
	fr.header.crc = fe.crc8;
	{   // FLAC__Frame.subframes[] (format.h:211-484; consumer: src/flac/analyze.c) from what the decode kernels parsed;
		// the CRC-16 footer from the frame's last two bytes
		const uint8_t *fb = q->audio.data() + fe.offset;
		const uint32_t flen = q->batch_bytes[bi];
		if(flen >= 2) fr.footer.crc = (FLAC__uint16)((fb[flen - 2] << 8) | fb[flen - 1]);
		for(uint32_t c = 0; c < ch; c++) {
			const fb200_subframe_info &I = q->batch_sub[bi * ch + c];
			FLAC__Subframe &sf = fr.subframes[c];
			sf.wasted_bits = I.wasted_bits;
			switch(I.type) {
				case 0: sf.type = FLAC__SUBFRAME_TYPE_CONSTANT; sf.data.constant.value = I.warmup[0]; break;
				case 1: sf.type = FLAC__SUBFRAME_TYPE_VERBATIM; sf.data.verbatim.data.int32 = nullptr; sf.data.verbatim.data_type = FLAC__VERBATIM_SUBFRAME_DATA_TYPE_INT32; break;
				case 2:
					sf.type = FLAC__SUBFRAME_TYPE_FIXED;
					sf.data.fixed.order = I.order;
					sf.data.fixed.entropy_coding_method.type = (FLAC__EntropyCodingMethodType)I.entropy_method;
					sf.data.fixed.entropy_coding_method.data.partitioned_rice.order = I.partition_order;
					for(uint32_t k = 0; k < I.order && k < 4; k++) sf.data.fixed.warmup[k] = I.warmup[k];
					break;
				default:
					sf.type = FLAC__SUBFRAME_TYPE_LPC;
					sf.data.lpc.order = I.order; sf.data.lpc.qlp_coeff_precision = I.qlp_coeff_precision; sf.data.lpc.quantization_level = I.quantization_level;
					sf.data.lpc.entropy_coding_method.type = (FLAC__EntropyCodingMethodType)I.entropy_method;
					sf.data.lpc.entropy_coding_method.data.partitioned_rice.order = I.partition_order;
					for(uint32_t k = 0; k < I.order; k++) { sf.data.lpc.qlp_coeff[k] = I.qlp_coeff[k]; sf.data.lpc.warmup[k] = I.warmup[k]; }
					break;
			}
		}
	}
	d->protected_->channels = ch; d->protected_->bits_per_sample = fe.bps; d->protected_->sample_rate = fe.sample_rate;
	d->protected_->blocksize = bs - skip; d->protected_->channel_assignment = fr.header.channel_assignment;
	if(d->protected_->md5_checking && !q->did_seek) q->md5.update_samples(src, (size_t)bs * ch, (fe.bps + 7) / 8);
	q->samples_decoded = first_sample + bs;
	d->protected_->state = FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC;
	q->last_header = fr.header; q->last_set = true;
	if(q->write_cb(d, &fr, chan, q->client_data) != FLAC__STREAM_DECODER_WRITE_STATUS_CONTINUE) {
		d->protected_->state = FLAC__STREAM_DECODER_ABORTED;
		return false;
	}
	return true;
}

extern "C" {

FLAC__StreamDecoder *FLAC__stream_decoder_new(void)
{
	FLAC__StreamDecoder *d = (FLAC__StreamDecoder *)calloc(1, sizeof *d);
	if(!d) return nullptr;
	d->protected_ = new FLAC__StreamDecoderProtected();
	d->private_ = new FLAC__StreamDecoderPrivate();
	memset(d->protected_, 0, sizeof *d->protected_);
	d->private_->gpu = nullptr; d->private_->file = nullptr; d->private_->owns_file = false;
	dec_set_defaults(d);
	d->protected_->state = FLAC__STREAM_DECODER_UNINITIALIZED;
	return d;
}

void FLAC__stream_decoder_delete(FLAC__StreamDecoder *d)
{
	if(!d) return;
	FLAC__stream_decoder_finish(d);
	delete d->protected_;
	delete d->private_;
	free(d);
}

#define DEC_UNINIT(d) ((d)->protected_->state == FLAC__STREAM_DECODER_UNINITIALIZED)
FLAC__bool FLAC__stream_decoder_set_ogg_serial_number(FLAC__StreamDecoder *d, long) { return DEC_UNINIT(d); }
FLAC__bool FLAC__stream_decoder_set_decode_chained_stream(FLAC__StreamDecoder *d, FLAC__bool) { return DEC_UNINIT(d); }
FLAC__bool FLAC__stream_decoder_set_md5_checking(FLAC__StreamDecoder *d, FLAC__bool value) { if(!DEC_UNINIT(d)) return false; d->protected_->md5_checking = value; return true; }
FLAC__bool FLAC__stream_decoder_set_metadata_respond(FLAC__StreamDecoder *d, FLAC__MetadataType type) { if(!DEC_UNINIT(d) || (uint32_t)type > FLAC__MAX_METADATA_TYPE_CODE) return false; d->private_->respond[type] = true; return true; }
FLAC__bool FLAC__stream_decoder_set_metadata_respond_application(FLAC__StreamDecoder *d, const FLAC__byte[4]) { if(!DEC_UNINIT(d)) return false; d->private_->respond[FLAC__METADATA_TYPE_APPLICATION] = true; return true; }
FLAC__bool FLAC__stream_decoder_set_metadata_respond_all(FLAC__StreamDecoder *d) { if(!DEC_UNINIT(d)) return false; memset(d->private_->respond, 1, sizeof d->private_->respond); return true; }
FLAC__bool FLAC__stream_decoder_set_metadata_ignore(FLAC__StreamDecoder *d, FLAC__MetadataType type) { if(!DEC_UNINIT(d) || (uint32_t)type > FLAC__MAX_METADATA_TYPE_CODE) return false; d->private_->respond[type] = false; return true; }
FLAC__bool FLAC__stream_decoder_set_metadata_ignore_application(FLAC__StreamDecoder *d, const FLAC__byte[4]) { if(!DEC_UNINIT(d)) return false; d->private_->respond[FLAC__METADATA_TYPE_APPLICATION] = false; return true; }
FLAC__bool FLAC__stream_decoder_set_metadata_ignore_all(FLAC__StreamDecoder *d) { if(!DEC_UNINIT(d)) return false; memset(d->private_->respond, 0, sizeof d->private_->respond); return true; }

FLAC__StreamDecoderState FLAC__stream_decoder_get_state(const FLAC__StreamDecoder *d) { return d->protected_->state; }
const char *FLAC__stream_decoder_get_resolved_state_string(const FLAC__StreamDecoder *d) { return FLAC__StreamDecoderStateString[d->protected_->state]; }
FLAC__bool FLAC__stream_decoder_get_md5_checking(const FLAC__StreamDecoder *d) { return d->protected_->md5_checking; }
FLAC__uint64 FLAC__stream_decoder_get_total_samples(const FLAC__StreamDecoder *d) { return d->private_->has_streaminfo ? d->private_->si.total_samples : 0; }
uint32_t FLAC__stream_decoder_get_channels(const FLAC__StreamDecoder *d) { return d->protected_->channels; }
FLAC__ChannelAssignment FLAC__stream_decoder_get_channel_assignment(const FLAC__StreamDecoder *d) { return d->protected_->channel_assignment; }
uint32_t FLAC__stream_decoder_get_bits_per_sample(const FLAC__StreamDecoder *d) { return d->protected_->bits_per_sample; }
uint32_t FLAC__stream_decoder_get_sample_rate(const FLAC__StreamDecoder *d) { return d->protected_->sample_rate; }
uint32_t FLAC__stream_decoder_get_blocksize(const FLAC__StreamDecoder *d) { return d->protected_->blocksize; }
FLAC__bool FLAC__stream_decoder_get_decode_position(const FLAC__StreamDecoder *d, FLAC__uint64 *position)
{
	// byte offset (from the start of the stream) of the next frame to be delivered -- what the reference's tell callback minus
	// its unconsumed input gives (stream_decoder.c:1087-1110); undefined (false) before the audio has been indexed
	const FLAC__StreamDecoderPrivate *q = d->private_;
	if(!position || !q->indexed) return false;
	const uint64_t audio_bytes = q->audio.size() >= 64 ? q->audio.size() - 64 : 0;
	*position = q->audio_offset + (q->next_frame < q->index.size() ? q->index[q->next_frame].offset : audio_bytes);
	return true;
}
// native FLAC has exactly one link; the chained-stream calls of API 14 (stream_decoder.h:970, 1022, 1150, 1538, 1664, 1754)
// reduce to their single-link meaning, as in the reference when the stream is not Ogg
FLAC__bool FLAC__stream_decoder_get_decode_chained_stream(const FLAC__StreamDecoder *) { return false; }
FLAC__uint64 FLAC__stream_decoder_find_total_samples(FLAC__StreamDecoder *d)
{
	// stream_decoder.c: native FLAC returns STREAMINFO's total when known; 0 = unknown
	return d->private_->has_streaminfo ? d->private_->si.total_samples : 0;
}
int32_t FLAC__stream_decoder_get_link_lengths(FLAC__StreamDecoder *, FLAC__uint64 **link_lengths)
{
	if(link_lengths) *link_lengths = nullptr;
	return -1;  // FLAC__STREAM_DECODER_GET_LINK_LENGTHS_INVALID: not an Ogg chain
}
uint32_t FLAC__stream_decoder_get_input_bytes_unconsumed(const FLAC__StreamDecoder *d)
{
	const FLAC__StreamDecoderPrivate *q = d->private_;
	return (uint32_t)std::min<size_t>(q->in.size() - q->in_pos, 0xffffffffu);
}
const void *FLAC__stream_decoder_get_client_data(FLAC__StreamDecoder *d) { return d->private_->client_data; }

static FLAC__StreamDecoderInitStatus dec_init_common(FLAC__StreamDecoder *d)
{
	FLAC__StreamDecoderPrivate *q = d->private_;
	q->in.clear(); q->in_pos = 0; q->consumed_before_in = 0; q->audio_offset = 0; q->eof = false; q->metadata_done = false; q->indexed = false; q->has_streaminfo = false; q->did_seek = false;
	q->next_frame = 0; q->skip_samples = 0; q->batch_first = q->batch_count = 0; q->samples_decoded = 0; q->last_set = false; q->error_sent = false;
	memset(&q->si, 0, sizeof q->si);
	d->protected_->state = FLAC__STREAM_DECODER_SEARCH_FOR_METADATA;
	return FLAC__STREAM_DECODER_INIT_STATUS_OK;
}

FLAC__StreamDecoderInitStatus FLAC__stream_decoder_init_stream(FLAC__StreamDecoder *d, FLAC__StreamDecoderReadCallback read_callback, FLAC__StreamDecoderSeekCallback seek_callback, FLAC__StreamDecoderTellCallback tell_callback, FLAC__StreamDecoderLengthCallback length_callback, FLAC__StreamDecoderEofCallback eof_callback, FLAC__StreamDecoderWriteCallback write_callback, FLAC__StreamDecoderMetadataCallback metadata_callback, FLAC__StreamDecoderErrorCallback error_callback, void *client_data)
{
	if(!DEC_UNINIT(d)) return FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED;
	if(!read_callback || !write_callback || !error_callback || (seek_callback && (!tell_callback || !length_callback || !eof_callback)))
		return FLAC__STREAM_DECODER_INIT_STATUS_INVALID_CALLBACKS;
	FLAC__StreamDecoderPrivate *q = d->private_;
	q->read_cb = read_callback; q->seek_cb = seek_callback; q->tell_cb = tell_callback; q->length_cb = length_callback; q->eof_cb = eof_callback;
	q->write_cb = write_callback; q->metadata_cb = metadata_callback; q->error_cb = error_callback; q->client_data = client_data; q->file = nullptr;
	return dec_init_common(d);
}

FLAC__StreamDecoderInitStatus FLAC__stream_decoder_init_ogg_stream(FLAC__StreamDecoder *d, FLAC__StreamDecoderReadCallback, FLAC__StreamDecoderSeekCallback, FLAC__StreamDecoderTellCallback, FLAC__StreamDecoderLengthCallback, FLAC__StreamDecoderEofCallback, FLAC__StreamDecoderWriteCallback, FLAC__StreamDecoderMetadataCallback, FLAC__StreamDecoderErrorCallback, void *)
{
	return DEC_UNINIT(d) ? FLAC__STREAM_DECODER_INIT_STATUS_UNSUPPORTED_CONTAINER : FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED;
}

FLAC__StreamDecoderInitStatus FLAC__stream_decoder_init_FILE(FLAC__StreamDecoder *d, FILE *file, FLAC__StreamDecoderWriteCallback write_callback, FLAC__StreamDecoderMetadataCallback metadata_callback, FLAC__StreamDecoderErrorCallback error_callback, void *client_data)
{
	if(!DEC_UNINIT(d)) return FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED;
	if(!file || !write_callback || !error_callback) return FLAC__STREAM_DECODER_INIT_STATUS_INVALID_CALLBACKS;
	FLAC__StreamDecoderPrivate *q = d->private_;
	q->read_cb = nullptr; q->seek_cb = nullptr; q->tell_cb = nullptr; q->length_cb = nullptr; q->eof_cb = nullptr;
	q->write_cb = write_callback; q->metadata_cb = metadata_callback; q->error_cb = error_callback; q->client_data = client_data;
	q->file = file; q->owns_file = file != stdin;
	return dec_init_common(d);
}

FLAC__StreamDecoderInitStatus FLAC__stream_decoder_init_ogg_FILE(FLAC__StreamDecoder *d, FILE *, FLAC__StreamDecoderWriteCallback, FLAC__StreamDecoderMetadataCallback, FLAC__StreamDecoderErrorCallback, void *)
{
	return DEC_UNINIT(d) ? FLAC__STREAM_DECODER_INIT_STATUS_UNSUPPORTED_CONTAINER : FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED;
}

FLAC__StreamDecoderInitStatus FLAC__stream_decoder_init_file(FLAC__StreamDecoder *d, const char *filename, FLAC__StreamDecoderWriteCallback write_callback, FLAC__StreamDecoderMetadataCallback metadata_callback, FLAC__StreamDecoderErrorCallback error_callback, void *client_data)
{
	if(!DEC_UNINIT(d)) return FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED;
	if(!write_callback || !error_callback) return FLAC__STREAM_DECODER_INIT_STATUS_INVALID_CALLBACKS;
	FILE *f = filename ? fopen(filename, "rb") : stdin;
	if(!f) return FLAC__STREAM_DECODER_INIT_STATUS_ERROR_OPENING_FILE;
	return FLAC__stream_decoder_init_FILE(d, f, write_callback, metadata_callback, error_callback, client_data);
}

FLAC__StreamDecoderInitStatus FLAC__stream_decoder_init_ogg_file(FLAC__StreamDecoder *d, const char *, FLAC__StreamDecoderWriteCallback, FLAC__StreamDecoderMetadataCallback, FLAC__StreamDecoderErrorCallback, void *)
{
	return DEC_UNINIT(d) ? FLAC__STREAM_DECODER_INIT_STATUS_UNSUPPORTED_CONTAINER : FLAC__STREAM_DECODER_INIT_STATUS_ALREADY_INITIALIZED;
}

FLAC__bool FLAC__stream_decoder_finish(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return true;
	FLAC__StreamDecoderPrivate *q = d->private_;
	FLAC__bool md5_ok = true;
	if(d->protected_->md5_checking && q->has_streaminfo && !q->did_seek && q->indexed && q->next_frame >= q->index.size()) {
		static const uint8_t zero[16] = {0};
		if(memcmp(q->si.md5sum, zero, 16) != 0) {
			uint8_t got[16];
			q->md5.final(got);
			md5_ok = memcmp(got, q->si.md5sum, 16) == 0;
		}
	}
	dec_release(d);
	dec_set_defaults(d);
	d->protected_->state = FLAC__STREAM_DECODER_UNINITIALIZED;
	return md5_ok;
}

FLAC__bool FLAC__stream_decoder_flush(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return false;
	d->private_->batch_count = 0;
	d->protected_->state = FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC;
	return true;
}

FLAC__bool FLAC__stream_decoder_reset(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return false;
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(q->indexed) { q->next_frame = 0; q->skip_samples = 0; q->batch_count = 0; q->did_seek = false; q->expect_pos = 0; q->last_set = false; q->md5.init(); d->protected_->state = FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC; return true; }
	return !q->metadata_done && q->in.empty();
}

FLAC__bool FLAC__stream_decoder_process_until_end_of_metadata(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return false;
	if(d->protected_->state == FLAC__STREAM_DECODER_ABORTED) return false;
	return dec_read_metadata(d) || d->protected_->state == FLAC__STREAM_DECODER_END_OF_STREAM;
}

FLAC__bool FLAC__stream_decoder_process_single(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return false;
	if(d->protected_->state == FLAC__STREAM_DECODER_ABORTED) return false;
	if(d->protected_->state == FLAC__STREAM_DECODER_END_OF_STREAM) return true;
	if(!d->private_->metadata_done) return dec_read_metadata(d) || d->protected_->state == FLAC__STREAM_DECODER_END_OF_STREAM;
	if(!dec_prepare_audio(d)) return false;
	return dec_deliver_next(d);
}

FLAC__bool FLAC__stream_decoder_process_until_end_of_stream(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return false;
	if(d->protected_->state == FLAC__STREAM_DECODER_ABORTED) return false;
	if(!d->private_->metadata_done && !dec_read_metadata(d)) return d->protected_->state == FLAC__STREAM_DECODER_END_OF_STREAM;
	if(!dec_prepare_audio(d)) return false;
	while(d->protected_->state != FLAC__STREAM_DECODER_END_OF_STREAM)
		if(!dec_deliver_next(d)) return false;
	return true;
}

FLAC__bool FLAC__stream_decoder_finish_link(FLAC__StreamDecoder *d)
{
	// only meaningful in END_OF_LINK state, which native FLAC never enters (stream_decoder.h:1538)
	return !DEC_UNINIT(d) && d->protected_->state == FLAC__STREAM_DECODER_END_OF_LINK;
}
FLAC__bool FLAC__stream_decoder_process_until_end_of_link(FLAC__StreamDecoder *d) { return FLAC__stream_decoder_process_until_end_of_stream(d); }
FLAC__bool FLAC__stream_decoder_skip_single_link(FLAC__StreamDecoder *d)
{
	// one link == the whole stream: skip to its end without decoding
	if(DEC_UNINIT(d)) return false;
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(!q->metadata_done && !dec_read_metadata(d)) return d->protected_->state == FLAC__STREAM_DECODER_END_OF_STREAM;
	if(!dec_prepare_audio(d)) return false;
	q->next_frame = q->index.size();
	q->did_seek = true;
	d->protected_->state = FLAC__STREAM_DECODER_END_OF_STREAM;
	return true;
}

FLAC__bool FLAC__stream_decoder_skip_single_frame(FLAC__StreamDecoder *d)
{
	if(DEC_UNINIT(d)) return false;
	if(!d->private_->metadata_done) return dec_read_metadata(d);
	if(!dec_prepare_audio(d)) return false;
	if(d->private_->next_frame < d->private_->index.size()) d->private_->next_frame++;
	else d->protected_->state = FLAC__STREAM_DECODER_END_OF_STREAM;
	return true;
}

FLAC__bool FLAC__stream_decoder_seek_absolute(FLAC__StreamDecoder *d, FLAC__uint64 sample)
{
	if(DEC_UNINIT(d)) return false;
	FLAC__StreamDecoderPrivate *q = d->private_;
	if(!q->metadata_done && !dec_read_metadata(d)) return false;
	if(!dec_prepare_audio(d)) return false;
	if(q->index.empty() || (q->si.total_samples && sample >= q->si.total_samples)) { d->protected_->state = FLAC__STREAM_DECODER_SEEK_ERROR; return false; }
	// frame whose range contains `sample`
	size_t lo = std::upper_bound(q->first_sample.begin(), q->first_sample.end(), sample) - q->first_sample.begin();
	if(lo == 0) { d->protected_->state = FLAC__STREAM_DECODER_SEEK_ERROR; return false; }
	lo--;
	if(sample >= q->first_sample[lo] + q->index[lo].blocksize) { d->protected_->state = FLAC__STREAM_DECODER_SEEK_ERROR; return false; }
	q->next_frame = lo;
	q->skip_samples = sample - q->first_sample[lo];
	q->did_seek = true;
	q->last_set = false;  // the frame a seek lands on is not compared with what came before it (is_seeking, :2484)
	d->protected_->state = FLAC__STREAM_DECODER_SEARCH_FOR_FRAME_SYNC;
	return dec_deliver_next(d);  // the reference delivers the frame containing the target right away (stream_decoder.c:1282-1340)
}

}  // extern "C"
