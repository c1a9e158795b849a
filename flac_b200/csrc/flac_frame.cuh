// flac_frame.cuh -- the FLAC frame rules, one copy for host and device code: the frame header's layout (writer side), its
// reader, the CRC-8 and CRC-16 steps and the GF(2) arithmetic that combines the CRCs of pieces of a frame.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#define FB200_HD __host__ __device__ __forceinline__

namespace fb200 {

// Per-frame decode status (low byte of fb200_decoder_get_frame_status).
enum : uint32_t {
	DEC_OK = 0, DEC_BAD_SYNC = 1, DEC_BAD_HEADER = 2, DEC_CRC8 = 3, DEC_UNSUPPORTED = 4, DEC_PARSE = 5,
	DEC_LENGTH = 6, DEC_CRC16 = 7, DEC_MISMATCH = 8, DEC_RANGE = 9,
	DEC_WRONG_FRAME = 10  // verify: the coded frame number or blocksize is not this frame's (FB200_VERIFY_WRONG_FRAME)
};

// ---------------------------------------------------------------- CRCs (crc.c)
// CRC-8, poly 0x07, of `byte` appended to a message whose CRC is `crc`
FB200_HD uint32_t crc8_byte(uint32_t crc, uint32_t byte)
{
	uint32_t c = (crc ^ byte) & 0xffu;
	for(int j = 0; j < 8; j++) c = (c & 0x80u) ? ((c << 1) ^ 0x07u) & 0xffu : (c << 1) & 0xffu;
	return c;
}

// a * b in GF(2)[x] / (x^8 + x^2 + x + 1): moves a CRC-8 past zero bytes when b = x^(8k)
FB200_HD uint32_t gf8_mul(uint32_t a, uint32_t b)
{
	uint32_t r = 0;
	for(int j = 7; j >= 0; j--) {
		r = (r & 0x80u) ? ((r << 1) ^ 0x07u) & 0xffu : (r << 1) & 0xffu;
		if((b >> j) & 1u) r ^= a;
	}
	return r;
}

// CRC-16, poly 0x8005, init 0, of the one byte b: the entry b of the byte-wise table
FB200_HD uint32_t crc16_entry(uint32_t b)
{
	uint32_t c = b << 8;
	for(int j = 0; j < 8; j++) c = (c & 0x8000u) ? ((c << 1) ^ 0x8005u) & 0xffffu : (c << 1) & 0xffffu;
	return c;
}

// a * b in GF(2)[x] / (x^16 + x^15 + x^2 + 1): crc(A || B) = crc(A) * x^(8|B|) + crc(B) for CRC-16s with init 0
FB200_HD uint32_t gf16_mul(uint32_t a, uint32_t b)
{
	uint32_t r = 0;
	for(int i = 15; i >= 0; i--) {
		r = (r & 0x8000u) ? ((r << 1) ^ 0x8005u) & 0xffffu : (r << 1);
		if((b >> i) & 1u) r ^= a;
	}
	return r;
}

// x^e mod (x^16 + x^15 + x^2 + 1), square and multiply
FB200_HD uint32_t gf16_xpow(unsigned long long e)
{
	uint32_t m = 1, b = 2;
	for(; e; e >>= 1) {
		if(e & 1ull) m = gf16_mul(m, b);
		b = gf16_mul(b, b);
	}
	return m;
}

// ---------------------------------------------------------------- frame header, writer side (stream_encoder_framing.c:245-391)
struct FrameHdr {
	uint32_t bs_code, bs_hint, sr_code, sr_hint, utf8_len, bits;  // bits: the whole header, CRC-8 included
};

FB200_HD FrameHdr frame_header_layout(int bs, int sample_rate, uint32_t frame_number)
{
	FrameHdr H;
	H.bs_hint = 0; H.sr_hint = 0;
	switch(bs) {
		case 192: H.bs_code = 1; break; case 576: H.bs_code = 2; break; case 1152: H.bs_code = 3; break;
		case 2304: H.bs_code = 4; break; case 4608: H.bs_code = 5; break; case 256: H.bs_code = 8; break;
		case 512: H.bs_code = 9; break; case 1024: H.bs_code = 10; break; case 2048: H.bs_code = 11; break;
		case 4096: H.bs_code = 12; break; case 8192: H.bs_code = 13; break; case 16384: H.bs_code = 14; break;
		case 32768: H.bs_code = 15; break;
		default: H.bs_code = H.bs_hint = (bs <= 0x100) ? 6 : 7; break;
	}
	switch(sample_rate) {
		case 88200: H.sr_code = 1; break; case 176400: H.sr_code = 2; break; case 192000: H.sr_code = 3; break;
		case 8000: H.sr_code = 4; break; case 16000: H.sr_code = 5; break; case 22050: H.sr_code = 6; break;
		case 24000: H.sr_code = 7; break; case 32000: H.sr_code = 8; break; case 44100: H.sr_code = 9; break;
		case 48000: H.sr_code = 10; break; case 96000: H.sr_code = 11; break;
		default:
			if(sample_rate <= 255000 && sample_rate % 1000 == 0) H.sr_code = H.sr_hint = 12;
			else if(sample_rate <= 655350 && sample_rate % 10 == 0) H.sr_code = H.sr_hint = 14;
			else if(sample_rate <= 0xffff) H.sr_code = H.sr_hint = 13;
			else H.sr_code = 0;
			break;
	}
	if(frame_number < 0x80) H.utf8_len = 1;
	else if(frame_number < 0x800) H.utf8_len = 2;
	else if(frame_number < 0x10000) H.utf8_len = 3;
	else if(frame_number < 0x200000) H.utf8_len = 4;
	else if(frame_number < 0x4000000) H.utf8_len = 5;
	else H.utf8_len = 6;
	H.bits = 32 + 8 * H.utf8_len + (H.bs_hint ? (H.bs_hint == 6 ? 8 : 16) : 0) + (H.sr_hint ? (H.sr_hint == 12 ? 8 : 16) : 0) + 8;
	return H;
}

// channel assignment code: ca 0 independent, 1 left/side, 2 side/right, 3 mid/side
FB200_HD uint32_t ca_code(int ca, int channels)
{
	switch(ca) { case 0: return (uint32_t)channels - 1; case 1: return 8; case 2: return 9; default: return 10; }
}

FB200_HD uint32_t bps_code(int bps)
{
	switch(bps) { case 8: return 1; case 12: return 2; case 16: return 4; case 20: return 5; case 24: return 6; case 32: return 7; default: return 0; }
}

// byte i of the header of a fixed-blocksize stream's frame laid out as H; 0 from the CRC-8 byte on
FB200_HD uint32_t frame_header_byte(const FrameHdr &H, int bs, int sample_rate, uint32_t frame_number, uint32_t cac, uint32_t bpsc, int i)
{
	const int pos_bs = 4 + (int)H.utf8_len;
	const int bs_bytes = H.bs_hint ? (H.bs_hint == 6 ? 1 : 2) : 0;
	const int pos_sr = pos_bs + bs_bytes;
	const int sr_bytes = H.sr_hint ? (H.sr_hint == 12 ? 1 : 2) : 0;
	const uint32_t v = frame_number;
	uint32_t byte = 0;
	if(i == 0) byte = 0xff;  // sync 0x3ffe, reserved 0, fixed-blocksize stream
	else if(i == 1) byte = 0xf8;
	else if(i == 2) byte = (H.bs_code << 4) | H.sr_code;
	else if(i == 3) byte = (cac << 4) | (bpsc << 1);
	else if(i < pos_bs) {  // UTF-8 style frame number (bitwriter.c:832-933)
		const int j = i - 4;
		if(j == 0) {
			switch(H.utf8_len) {
				case 1: byte = v; break;
				case 2: byte = 0xC0 | (v >> 6); break;
				case 3: byte = 0xE0 | (v >> 12); break;
				case 4: byte = 0xF0 | (v >> 18); break;
				case 5: byte = 0xF8 | (v >> 24); break;
				default: byte = 0xFC | (v >> 30); break;
			}
		}
		else byte = 0x80 | ((v >> (6 * ((int)H.utf8_len - 1 - j))) & 0x3F);
	}
	else if(i < pos_sr) byte = ((uint32_t)bs - 1) >> (8 * (bs_bytes - 1 - (i - pos_bs)));
	else if(i < pos_sr + sr_bytes) {
		const uint32_t sv = H.sr_hint == 12 ? (uint32_t)sample_rate / 1000 : H.sr_hint == 13 ? (uint32_t)sample_rate : (uint32_t)sample_rate / 10;
		byte = sv >> (8 * (sr_bytes - 1 - (i - pos_sr)));
	}
	return byte & 0xffu;
}

// ---------------------------------------------------------------- frame header, reader side (stream_decoder.c:2624-2947)
struct FrameHeader {
	uint32_t blocksize;
	uint64_t number;      // frame or sample number from the header
	uint32_t variable;    // blocking strategy bit
	uint32_t sample_rate, channels, bps, ca;
	uint8_t crc8;
};

struct FrameHeaderRead {
	uint32_t status;  // DEC_OK, DEC_LENGTH, DEC_BAD_SYNC, DEC_BAD_HEADER or DEC_CRC8
	uint32_t bytes;   // header length, CRC-8 included (DEC_OK)
};

// Reads the frame header at p, of which `avail` bytes may be read; rate / bps code 0 take the stream's values. Reports the first
// rule the header breaks: fewer than 6 bytes; the sync code; the reserved bits, the UTF-8 number's first byte, blocksize code 0,
// rate code 15; a header longer than `avail`; a UTF-8 continuation byte; the CRC-8; channel code > 10, bps code 3. The length
// comes from the code bits before any byte behind them is read, so no byte at or past `avail` is read.
FB200_HD FrameHeaderRead parse_frame_header(const uint8_t *p, size_t avail, uint32_t stream_rate, uint32_t stream_bps, FrameHeader &fh)
{
	FrameHeaderRead r = {DEC_LENGTH, 0};
	if(avail < 6) return r;
	r.status = DEC_BAD_SYNC;
	if(p[0] != 0xFF || (p[1] & 0xFC) != 0xF8) return r;
	r.status = DEC_BAD_HEADER;
	const uint32_t variable = p[1] & 1, bs_code = p[2] >> 4, sr_code = p[2] & 15, cac = p[3] >> 4, bpsc = (p[3] >> 1) & 7;
	if((p[1] & 2) || (p[3] & 1) || bs_code == 0 || sr_code == 15) return r;
	const bool late_bad = cac > 10 || bpsc == 3;  // reported after the CRC-8
	const uint32_t first = p[4];
	uint32_t n;  // UTF-8 continuation bytes
	uint64_t number;
	if(!(first & 0x80)) { n = 0; number = first; }
	else if((first & 0xE0) == 0xC0) { n = 1; number = first & 0x1F; }
	else if((first & 0xF0) == 0xE0) { n = 2; number = first & 0x0F; }
	else if((first & 0xF8) == 0xF0) { n = 3; number = first & 0x07; }
	else if((first & 0xFC) == 0xF8) { n = 4; number = first & 0x03; }
	else if((first & 0xFE) == 0xFC) { n = 5; number = first & 0x01; }
	else if(first == 0xFE && variable) { n = 6; number = 0; }
	else return r;
	const uint32_t len = 5 + n + (bs_code == 6 ? 1 : bs_code == 7 ? 2 : 0) + (sr_code == 12 ? 1 : sr_code >= 13 ? 2 : 0);
	if(len >= avail) { r.status = DEC_LENGTH; return r; }
	uint32_t pos = 5;
	for(uint32_t k = 0; k < n; k++, pos++) {
		if((p[pos] & 0xC0) != 0x80) return r;
		number = (number << 6) | (p[pos] & 0x3F);
	}
	uint32_t blocksize;
	switch(bs_code) {
		case 1: blocksize = 192; break;
		case 2: case 3: case 4: case 5: blocksize = 576u << (bs_code - 2); break;
		case 6: blocksize = p[pos++] + 1u; break;
		case 7: blocksize = (((uint32_t)p[pos] << 8) | p[pos + 1]) + 1u; pos += 2; break;
		default: blocksize = 256u << (bs_code - 8); break;
	}
	uint32_t rate;
	switch(sr_code) {
		case 0: rate = stream_rate; break;
		case 1: rate = 88200; break; case 2: rate = 176400; break; case 3: rate = 192000; break; case 4: rate = 8000; break;
		case 5: rate = 16000; break; case 6: rate = 22050; break; case 7: rate = 24000; break; case 8: rate = 32000; break;
		case 9: rate = 44100; break; case 10: rate = 48000; break; case 11: rate = 96000; break;
		case 12: rate = p[pos] * 1000u; break;
		case 13: rate = ((uint32_t)p[pos] << 8) | p[pos + 1]; break;
		default: rate = (((uint32_t)p[pos] << 8) | p[pos + 1]) * 10u; break;
	}
	uint32_t crc = 0;
	for(uint32_t b = 0; b < len; b++) crc = crc8_byte(crc, p[b]);
	if(crc != p[len]) { r.status = DEC_CRC8; return r; }
	if(late_bad) return r;
	uint32_t bps;
	switch(bpsc) {
		case 0: bps = stream_bps; break;
		case 1: bps = 8; break; case 2: bps = 12; break; case 4: bps = 16; break;
		case 5: bps = 20; break; case 6: bps = 24; break; default: bps = 32; break;
	}
	fh.blocksize = blocksize; fh.number = number; fh.variable = variable; fh.sample_rate = rate;
	fh.channels = cac < 8 ? cac + 1 : 2; fh.ca = cac < 8 ? 0 : cac - 7; fh.bps = bps; fh.crc8 = (uint8_t)crc;
	r.status = DEC_OK;
	r.bytes = len + 1;
	return r;
}

}  // namespace fb200
