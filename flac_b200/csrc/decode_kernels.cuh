// decode_kernels.cuh -- sm_90a kernels of the FLAC batch frame decoder.
//
// Frames carry no length field and Rice codes have data-dependent lengths: where subframe c+1 starts is only known
// once subframe c has been walked, and the LPC restore is a serial recurrence (SURVEY.md 7.3-6). Round 1 ran the whole
// frame in one thread (header, every subframe, Rice decode fused with the restore, planar scratch, then a merge pass):
// most of the decode step at a small fraction of HBM bandwidth, divergent (32 different frames per warp, each in a
// different loop nest) and with 4-byte stores 16 KB apart. This generation splits the frame along its only parallel axis, the channels:
//   k_dec_walk   : one thread per frame -- header (stream_decoder.c:2624-2947) + CRC-8, then a WALK over subframes
//                  0..channels-2 that only measures them (unary length + k per code, no sample is formed): the bit
//                  offset of every subframe. ~10 instructions per code.
//   k_dec_frames : one LANE per (frame, channel), the lanes of a frame adjacent in a warp and in lock step over the
//                  sample index: Rice decode (deduplication/bitreader_read_rice_signed_block.c) fused with the
//                  fixed/LPC restore (lpc.c:978-1491, fixed.c:571-629) with the history in registers, inter-channel
//                  decorrelation undone through a shuffle (stream_decoder.c:3476-3527), interleaved PCM written
//                  directly (the lanes of a frame store adjacent words). No scratch, no merge pass. All per-sample
//                  decisions (partition change, escape, verbatim, constant) are data, not control flow, so the 32 lanes
//                  of a warp stay converged although they decode different subframes.
//   k_dec_crc    : one warp per frame -- CRC-16 of the frame bytes (crc.c:78-396), slicing-by-4 + GF(2) combine.
// Reads never leave the frame: the bit reader returns zeros past the frame's last word (untrusted input).
// k_dec_frames<MAXQ, true> is the compare mode behind the encoder's verify (fb200_encoder_set_verify): every decoded sample is
// compared in registers with the input value at its place instead of being stored, and k_verify_files reduces the per-frame
// verdicts to each file's first failure (stream_encoder.c:5186-5231).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "fb200_internal.h"
#include "flac_frame.cuh"

namespace fb200 {

struct DecK {
	int channels, bps, sample_rate, blocksize;  // STREAMINFO facts
	int loose_end;                               // 1: a frame's given end is an upper bound (index mode); 0: it must be exact
};

struct DecFrameMeta {
	uint32_t status;
	uint32_t blocksize;
	uint32_t channel_assignment;  // 0 independent, 1 left/side, 2 right/side, 3 mid/side
	uint32_t channels;
	uint32_t sub_bit[FB200_MAX_CHANNELS];  // bit offset (from the frame's first byte) of every subframe
	uint32_t frame_bytes;         // parsed length including the CRC-16 (k_dec_frames)
	uint32_t frame_number_lo;     // low 32 bits of the coded frame / sample number
	uint32_t variable;            // 1: variable blocksize stream (the number is a sample number)
	uint32_t sample_rate;
	uint32_t max_order;           // largest predictor order among the frame's subframes (selects the k_dec_frames instantiation)
};

// What a client sees of one subframe (FLAC__Subframe, include/FLAC/format.h:211-484) -- filled on request.
struct DecSubframeInfo {
	uint8_t type;       // 0 constant, 1 verbatim, 2 fixed, 3 lpc
	uint8_t order;
	uint8_t wasted;
	uint8_t precision;  // lpc
	int8_t shift;       // lpc
	uint8_t method;     // 0 RICE, 1 RICE2
	uint8_t porder;
	uint8_t pad;
	int32_t qlp[FB200_MAX_LPC_ORDER];
	int32_t warmup[FB200_MAX_LPC_ORDER];  // warm-up samples (constant: [0] = the value)
};

// MSB-first bit reader over global memory. The reader holds the two words the current position straddles (w0, w1: one funnel
// shift yields the next 32 bits at any bit position) and TWO words of look-ahead (w2, w3) that were loaded one and two word
// crossings earlier. A lane walks its own frame, so nothing but the reader itself can hide its load latency: two crossings
// (~5 Rice codes of the whole warp) cover an L2 hit, and whenever the reader enters a new 128-byte line it prefetches the line
// after the next into L2. Consuming bits is an add and a test; only a word crossing (every ~2.5 codes) moves registers and
// loads. Words past `nwords` read as zeros: no read leaves the frame's last 16-byte granule. (Earlier versions, for the
// record: one dependent 32-bit load per refill, i.e. a full load latency per Rice code; a three-deep queue of 128-bit loads
// whose rotation cost 5 moves per word; a 64-bit left-aligned accumulator whose branch-free refill cost many instructions per
// code.)
struct BitRd {
	const uint32_t *words;         // 128-byte aligned address at or below the frame's first byte
	uint32_t nwords;               // words (from `words`) that may be read
	uint32_t widx;                 // index of the next word to LOAD (w3 holds word widx - 1, w0 word widx - 4 = pos >> 5)
	uint32_t pos, end;             // bit position / end of the frame, relative to `words`
	uint32_t w0, w1, w2, w3;       // byte-swapped words
	__device__ __forceinline__ uint32_t load(uint32_t i) const
	{
		uint32_t v = 0u;
		if(i < nwords) v = __ldg(words + i);
		return __byte_perm(v, 0, 0x0123);
	}
	__device__ __forceinline__ void prefetch_line(uint32_t i) const  // i: first word of a 128-byte line
	{
		if(i < nwords) asm volatile("prefetch.global.L2 [%0];" ::"l"(words + i));
	}
	__device__ __forceinline__ void reseat()  // (re)load the window at bit position `pos`
	{
		widx = pos >> 5;
		w0 = load(widx); w1 = load(widx + 1u); w2 = load(widx + 2u); w3 = load(widx + 3u);
		prefetch_line((widx & ~31u) + 32u);
		prefetch_line((widx & ~31u) + 64u);
		widx += 4u;
	}
	// p: first byte of the frame, len: frame bytes, bit: bit offset inside the frame to start at
	__device__ __forceinline__ void init(const uint8_t *p, uint32_t len, uint32_t bit)
	{
		const uintptr_t a = reinterpret_cast<uintptr_t>(p);
		words = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)127);  // line aligned: prefetch decisions are on widx % 32
		const uint32_t lead = (uint32_t)(a & 127) * 8;
		nwords = len ? (lead + len * 8 + 31) >> 5 : 0u;
		end = lead + len * 8;
		pos = lead + bit;
		reseat();
	}
	__device__ __forceinline__ uint32_t peek32() const { return __funnelshift_l(w1, w0, pos); }  // shift amount wraps at 32
	__device__ __forceinline__ void consume(uint32_t n)  // 0..32
	{
		const uint32_t np = pos + n;
		const bool cross = ((pos ^ np) & 32u) != 0u;  // n <= 32: at most one word boundary
		pos = np;
		if(cross) {
			w0 = w1; w1 = w2; w2 = w3;
			w3 = load(widx);
			if((widx & 31u) == 0u) prefetch_line(widx + 64u);
			widx++;
		}
	}
	__device__ __forceinline__ uint32_t get(uint32_t n)  // 1..32
	{
		const uint32_t v = peek32() >> (32u - n);
		consume(n);
		return v;
	}
	__device__ __forceinline__ int32_t get_signed(uint32_t n)  // 1..32
	{
		const int32_t v = (int32_t)peek32() >> (32u - n);
		consume(n);
		return v;
	}
	__device__ __forceinline__ void skip(uint32_t n)  // any number of bits
	{
		if(n <= 32u) consume(n);
		else {
			pos = (n > 0x7fffffffu - pos) ? 0x7fffffffu : pos + n;  // saturate: corrupt streams must not wrap the position
			reseat();
		}
	}
	// number of 0 bits before the next 1, consumed together with the 1 (bitreader.c:725)
	__device__ __forceinline__ uint32_t unary()
	{
		uint32_t q = 0;
		uint32_t v = peek32();
		while(v == 0) {
			if(pos > end) return q;
			q += 32;
			consume(32);
			v = peek32();
		}
		const uint32_t z = (uint32_t)__clz((int)v);
		consume(z + 1);
		return q + z;
	}
	__device__ __forceinline__ bool overrun() const { return pos > end; }
};

__device__ __forceinline__ uint32_t dec_silog2(long long v)
{
	if(v == 0) return 0;
	if(v == -1) return 2;
	v = (v < 0) ? (-(v + 1)) : v;
	return (63u - (uint32_t)__clzll(v)) + 2;
}

// ---------------------------------------------------------------- subframe header (stream_decoder.c:2949-3297)
struct SubHdr {
	uint32_t type;     // 0 constant, 1 verbatim, 2 fixed, 3 lpc, 255 invalid
	uint32_t order, wasted, bps;  // bps: after wasted bits
	uint32_t precision;
	int shift;
};

// reads the 8-bit subframe header (+ unary wasted bits); the reader is left at the first warm-up / constant / verbatim bit
__device__ __forceinline__ SubHdr read_sub_header(BitRd &br, uint32_t bps)
{
	SubHdr h;
	h.type = 255; h.order = 0; h.wasted = 0; h.bps = bps; h.precision = 0; h.shift = 0;
	uint32_t x = br.get(8);
	if(x & 0x80) return h;
	if(x & 1) {
		h.wasted = br.unary() + 1;
		if(h.wasted >= bps) return h;
		h.bps = bps - h.wasted;
	}
	x &= 0xfe;
	if(x == 0) h.type = 0;
	else if(x == 2) h.type = 1;
	else if(x >= 16 && x <= 24) { h.type = 2; h.order = (x >> 1) & 7; if(h.order > 4) h.type = 255; }
	else if(x >= 64) { h.type = 3; h.order = ((x >> 1) & 31) + 1; }
	return h;
}

// ================================================================ k_dec_scan
// The decoder front end (frame_sync_ + read_frame_header_, stream_decoder.c:2321-2371, 2624-2947) for a whole stream at
// once: every byte position is tested for sync code + a self-consistent header (reserved bits, code points, UTF-8 number,
// CRC-8). Candidates are appended unordered (the host sorts the short list); false positives (~2^-25 per byte) are weeded
// out later by decoding: a candidate that does not parse / fails its CRC-16, or lies inside an accepted frame, is dropped.
__global__ void __launch_bounds__(256) k_dec_scan(const uint8_t *__restrict__ data, unsigned long long n, unsigned long long *__restrict__ cand,
                                                 unsigned cap, unsigned *__restrict__ count)
{
	const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
	for(unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; p + 6 <= n; p += stride) {
		if(data[p] != 0xFF || (data[p + 1] & 0xFE) != 0xF8) continue;
		FrameHeader fh;
		if(parse_frame_header(data + p, n - p, 0, 0, fh).status != DEC_OK) continue;
		const unsigned slot = atomicAdd(count, 1u);
		if(slot < cap) cand[slot] = p;
	}
}

// ================================================================ k_dec_walk
// A frame is the byte range [begins[f], ends[f]): exact (ends = begins + 1 of one offsets array) or, with P.loose_end, an upper bound.
__global__ void __launch_bounds__(128) k_dec_walk(DecK P, const uint8_t *__restrict__ frames, const unsigned long long *__restrict__ begins,
                                                 const unsigned long long *__restrict__ ends, int nframes, DecFrameMeta *__restrict__ meta)
{
	const int f = blockIdx.x * blockDim.x + threadIdx.x;
	if(f >= nframes) return;
	const unsigned long long off = begins[f];
	const uint32_t len = (uint32_t)min(ends[f] - off, 0x0fffffffull);
	DecFrameMeta M;
	M.status = DEC_OK; M.blocksize = 0; M.channel_assignment = 0; M.channels = 0; M.frame_bytes = 0; M.frame_number_lo = 0; M.variable = 0; M.sample_rate = 0; M.max_order = 0;
#pragma unroll
	for(int c = 0; c < FB200_MAX_CHANNELS; c++) M.sub_bit[c] = 0;
	FrameHeader fh;
	const FrameHeaderRead hr = parse_frame_header(frames + off, len, (uint32_t)P.sample_rate, (uint32_t)P.bps, fh);
	if(hr.status != DEC_OK) { M.status = hr.status; meta[f] = M; return; }
	const uint32_t blocksize = fh.blocksize, ca = fh.ca, channels = fh.channels, bps = fh.bps;
	BitRd br;
	br.init(frames + off, len, 8 * hr.bytes);
	const uint32_t start = br.pos - 8 * hr.bytes;
	M.blocksize = blocksize; M.channel_assignment = ca; M.channels = channels; M.frame_number_lo = (uint32_t)fh.number; M.variable = fh.variable; M.sample_rate = fh.sample_rate;
	if(blocksize > (uint32_t)P.blocksize || channels != (uint32_t)P.channels || bps != (uint32_t)P.bps || bps > 24) {
		M.status = (bps > 24) ? DEC_UNSUPPORTED : DEC_MISMATCH;
		meta[f] = M;
		return;
	}

	// ---- measure subframes 0 .. channels-2 (the last one is measured by the lane that decodes it)
	for(uint32_t c = 0; c < channels; c++) {
		M.sub_bit[c] = br.pos - start;
		uint32_t sub_bps = bps;
		if((ca == 1 && c == 1) || (ca == 2 && c == 0) || (ca == 3 && c == 1)) sub_bps++;
		const SubHdr h = read_sub_header(br, sub_bps);
		if(h.type != 255 && h.order > M.max_order) M.max_order = h.order;
		if(c + 1 == channels) break;  // the last subframe: only its header (for max_order) is looked at here
		bool ok = h.type != 255;
		if(ok && h.type == 0) br.skip(h.bps);
		else if(ok && h.type == 1) br.skip(blocksize * h.bps);
		else if(ok) {
			if(blocksize <= h.order) ok = false;
			else {
				br.skip(h.order * h.bps);
				if(h.type == 3) {
					const uint32_t prec = br.get(4);
					if(prec == 15) ok = false;
					br.skip(5 + h.order * (prec + 1));
				}
			}
			if(ok) {
				// stream_decoder.c:3299-3357 read_residual_partitioned_rice_, lengths only
				const uint32_t method = br.get(2);
				const uint32_t plen = method ? kRice2ParamLen : kRiceParamLen, pesc = method ? kRice2Escape : kRiceEscape;
				const uint32_t po = br.get(4);
				const uint32_t psamples = blocksize >> po;
				if(method > 1 || (po > 0 ? (psamples < h.order || (psamples << po) != blocksize) : blocksize < h.order)) ok = false;
				uint32_t i = h.order;
				for(uint32_t p = 0; ok && p < (1u << po); p++) {
					const uint32_t k = br.get(plen);
					const uint32_t pend = (po == 0) ? blocksize : (p + 1) * psamples;
					if(k >= pesc) {
						const uint32_t raw = br.get(5);
						br.skip(raw * (pend - i));
						i = pend;
					}
					else {
						for(; i < pend; i++) {
							// one Rice code: zeros, a one, k low bits
							const uint32_t n = (uint32_t)__clz((int)br.peek32()) + 1u + k;  // clz(0) = 32
							if(n <= 32u) br.consume(n);
							else { (void)br.unary(); br.skip(k); }
						}
					}
					if(br.overrun()) ok = false;
				}
			}
		}
		if(!ok || br.overrun()) { M.status = DEC_PARSE; break; }
	}
	meta[f] = M;
}

// ================================================================ k_dec_frames
// One lane per (frame, channel); CHL lanes per frame (channels rounded up to a power of two), 32 / CHL frames per warp.
// The lanes run in lock step over the sample index i; sample i of a lane lives in history slot i % MAXORD, and the loop
// is unrolled MAXORD times so that every history access has a compile-time register index.
// The rare events of the sample loop live out of line (by value in, by value out: the reader stays in registers on the hot path):
// the loop body is unrolled MAXORD times, and with every slow path inlined at every site it outgrew the instruction cache
// (instruction fetches showed up among the stall reasons).
struct DecPart {
	uint32_t k, raw, next_part, part_end, esc;
};
struct DecPartOut {
	BitRd br;
	DecPart st;
};
// a partition starts at sample i (or the lane's block ended): Rice parameter (+ escape width), stream_decoder.c:3299-3357
__device__ __noinline__ DecPartOut dec_partition_start(BitRd br, DecPart st, uint32_t i, uint32_t bs_lane, uint32_t psamples, uint32_t plen, uint32_t pesc)
{
	do {
		if(i >= bs_lane) { st.esc = 1; st.raw = 0; st.next_part = 0xffffffffu; break; }
		st.k = br.get(plen);
		st.esc = st.k >= pesc;
		if(st.esc) st.raw = br.get(5);
		st.next_part = st.part_end;
		st.part_end += psamples;
	} while(i == st.next_part);
	DecPartOut o;
	o.br = br; o.st = st;
	return o;
}
struct DecCodeOut {
	BitRd br;
	uint32_t uu;
	bool over;  // the quotient does not fit 32 bits with the k low bits: the frame is lost (bitreader_read_rice_signed_block.c:17,69)
};
// a Rice code whose unary part and k low bits do not fit the 32-bit window (the inline path's codes, z + 1 + k <= 32, never
// reach the quotient limit)
__device__ __noinline__ DecCodeOut dec_long_code(BitRd br, uint32_t k)
{
	const uint32_t msbs = br.unary();
	DecCodeOut o;
	o.over = k != 0u && msbs > (0xffffffffu >> k);
	o.uu = (msbs << k) | (k ? br.get(k) : 0u);
	o.br = br;
	return o;
}

// Every subframe type runs through ONE loop body: CONSTANT is a first-order predictor with one warm-up sample and all-zero
// residuals, VERBATIM a zero predictor whose residuals are escape-coded with the sample width; both enter as an "escaped
// partition" that spans the block (esc0 / raw0), so the body has no per-sample type test. A lane that is past its block (or has
// no block) is switched into the same zero-width escape mode at the partition-start test, reads nothing and stores nothing.
// CMP: dst is the expected input; each sample is loaded and compared instead of stored, and the lane's first mismatch kept in mm.
struct DecLaneMismatch {
	bool hit;
	uint32_t sample;
	int32_t expected, got;
};
template <int MAXORD, bool WIDE, int CH, bool CMP>
__device__ __forceinline__ void dec_lane_loop(BitRd &br, const uint32_t bs_lane, const uint32_t bs_max, const uint32_t order, const uint32_t wasted,
                                              const int shift, const bool lane_wide, const int (&q)[MAXORD], const int (&warm)[MAXORD],
                                              const bool esc0, const uint32_t raw0, const uint32_t po, const uint32_t plen, const uint32_t pesc,
                                              int32_t *__restrict__ dst, const uint32_t ch_rt, const uint32_t ca, const uint32_t cidx,
                                              const uint32_t out_bps, bool &bad, DecLaneMismatch &mm)
{
	const uint32_t ch = CH ? (uint32_t)CH : ch_rt;
	int H[MAXORD];
#pragma unroll
	for(int j = 0; j < MAXORD; j++) H[j] = 0;
	const uint32_t psamples = bs_lane >> po;
	DecPart st;
	st.k = 0; st.raw = raw0; st.next_part = esc0 ? bs_lane : order; st.part_end = psamples; st.esc = esc0 ? 1u : 0u;
	const uint32_t lim = 1u << (out_bps - 1);
	uint32_t range_or = 0;  // OR of (sample + lim): any bit at or above out_bps = a sample out of range (stream_decoder.c:2458-2472)
	// how this lane's output is formed from its own value v and its partner's o (stream_decoder.c:3476-3527), as
	// (ca * v + cb * o + (o & mo) + (v & mv)) >> cs: own value; right = left - side; left = side + right; mid/side: the lane that
	// holds mid: ((mid << 1 | side & 1) + side) >> 1, the lane that holds side: ((mid << 1 | side & 1) - side) >> 1
	int cA = 1, cB = 0, cs = 0;
	uint32_t mo = 0, mv = 0;
	if(ch == 2) {
		if(ca == 1 && cidx == 1) { cA = -1; cB = 1; }
		else if(ca == 2 && cidx == 0) { cA = 1; cB = 1; }
		else if(ca == 3 && cidx == 0) { cA = 2; cB = 1; cs = 1; mo = 1; }
		else if(ca == 3 && cidx == 1) { cA = -1; cB = 2; cs = 1; mv = 1; }
	}
	int32_t *op = dst;
	// CMP: the expected samples of the next MAXORD are loaded together when a group starts, so a lane waits for the load
	// latency once per group rather than at every sample (a lone warp of a short chunk would otherwise run at one load per step)
	int32_t E[CMP ? MAXORD : 1];
	const int32_t *ep = dst;
	auto load_group = [&](const uint32_t i0) {
		if constexpr(CMP) {
#pragma unroll
			for(int u = 0; u < MAXORD; u++) E[u] = (i0 + (uint32_t)u < bs_lane) ? ep[(uint32_t)u * ch] : 0;
			ep += MAXORD * ch;
		}
	};

	// one sample; FIRST: the first MAXORD samples of the block, where warm-up samples still come straight from the header
	auto step = [&](auto first_tag, const int u, const uint32_t i) {
		constexpr bool FIRST = decltype(first_tag)::value;
		int32_t x;
		if(FIRST && i < order) x = warm[u];
		else {
			if(i == st.next_part) {
				const DecPartOut o = dec_partition_start(br, st, i, bs_lane, psamples, plen, pesc);
				br = o.br; st = o.st;
			}
			int32_t r;
			if(!st.esc) {
				// deduplication/bitreader_read_rice_signed_block.c: unary MSBs, k LSBs, zig-zag
				const uint32_t v = br.peek32();
				const uint32_t z = (uint32_t)__clz((int)v);  // 32 for v == 0
				uint32_t uu;
				if(z + 1u + st.k <= 32u) {
					const uint32_t low = ((v << z) & 0x7fffffffu) >> (31u - st.k);  // the k bits after the terminating 1
					uu = (z << st.k) | low;
					br.consume(z + 1u + st.k);
				}
				else {
					const DecCodeOut o = dec_long_code(br, st.k);
					br = o.br; uu = o.uu;
					if(o.over) bad = true;
				}
				r = (int32_t)(uu >> 1) ^ -(int32_t)(uu & 1u);
			}
			else r = st.raw ? br.get_signed(st.raw) : 0;
			// prediction from the last `order` samples: x[i-1-j] sits in slot (u - 1 - j) mod MAXORD
			int32_t pred;
			if(WIDE && lane_wide) {
				long long s0 = 0, s1 = 0;
#pragma unroll
				for(int j = 0; j < MAXORD; j += 2) {
					s0 += (long long)q[j] * (long long)H[(u - 1 - j + 2 * MAXORD) % MAXORD];
					if(j + 1 < MAXORD) s1 += (long long)q[j + 1] * (long long)H[(u - 2 - j + 2 * MAXORD) % MAXORD];
				}
				pred = (int32_t)((s0 + s1) >> shift);
			}
			else {
				int s0 = 0, s1 = 0;
#pragma unroll
				for(int j = 0; j < MAXORD; j += 2) {
					s0 += q[j] * H[(u - 1 - j + 2 * MAXORD) % MAXORD];
					if(j + 1 < MAXORD) s1 += q[j + 1] * H[(u - 2 - j + 2 * MAXORD) % MAXORD];
				}
				pred = (s0 + s1) >> shift;
			}
			x = r + pred;
		}
		H[u] = x;
		// ---- undo the channel decorrelation and store interleaved
		const int32_t val = (int32_t)((uint32_t)x << wasted);
		int32_t out = val;
		if(ch == 2) {
			const int32_t other = __shfl_xor_sync(0xffffffffu, val, 1);
			out = (cA * val + cB * other + (int32_t)((uint32_t)other & mo) + (int32_t)((uint32_t)val & mv)) >> cs;
		}
		const bool on = i < bs_lane;
		range_or |= on ? (uint32_t)out + lim : 0u;
		if constexpr(CMP) {
			if(on && E[u] != out && !mm.hit) { mm.hit = true; mm.sample = i; mm.expected = E[u]; mm.got = out; }
		}
		else if(on) op[(CH ? (uint32_t)u : 0u) * ch] = out;
		if(!CH) op += ch;
	};
	if(bs_max > 0) {
		load_group(0u);
#pragma unroll
		for(int u = 0; u < MAXORD; u++) step(std::true_type{}, u, (uint32_t)u);
		if(CH) op += MAXORD * CH;
	}
#pragma unroll 1
	for(uint32_t i0 = MAXORD; i0 < bs_max; i0 += MAXORD) {
		load_group(i0);
#pragma unroll
		for(int u = 0; u < MAXORD; u++) step(std::false_type{}, u, i0 + (uint32_t)u);
		if(CH) op += MAXORD * CH;
	}
	if(range_or >> out_bps) bad = true;
}

// CMP (verify): pcm holds the expected samples, nothing is stored there; verdict[f] gets the frame's lowest mismatching channel
// and that channel's first mismatch (channel ~0u: none)
template <int MAXQ, bool CMP = false>
__global__ void __launch_bounds__(128) k_dec_frames(DecK P, const uint8_t *__restrict__ frames, const unsigned long long *__restrict__ begins,
                                                   const unsigned long long *__restrict__ ends, int nframes,
                                                   DecFrameMeta *__restrict__ meta, int32_t *__restrict__ pcm, unsigned long long capacity_samples,
                                                   uint32_t *__restrict__ status_out, DecSubframeInfo *__restrict__ subinfo,
                                                   DecVerdict *__restrict__ verdict = nullptr)
{
	const int ch = P.channels;
	const int chl = ch <= 1 ? 1 : ch <= 2 ? 2 : ch <= 4 ? 4 : 8;
	const int fpw = 32 / chl;  // frames per warp
	const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	const int f = warp_global * fpw + lane / chl;
	const uint32_t cidx = (uint32_t)(lane % chl);
	if(warp_global * fpw >= nframes) return;  // whole warp idle
	const bool have = f < nframes && (int)cidx < ch;
	DecFrameMeta M;
	M.status = DEC_LENGTH; M.blocksize = 0; M.channel_assignment = 0; M.channels = 0;
	unsigned long long off = 0;
	uint32_t len = 0;
	if(f < nframes) {
		M = meta[f];
		off = begins[f];
		len = (uint32_t)min(ends[f] - off, 0x0fffffffull);
	}
	const unsigned long long first = (unsigned long long)f * (unsigned long long)P.blocksize;
	// this instantiation's share of the frames: MAXQ = 12 takes every frame whose predictors have at most 12 taps, MAXQ = 32 the rest
	const bool mine = (MAXQ == 12) ? M.max_order <= 12 : M.max_order > 12;
	if(!__any_sync(0xffffffffu, f < nframes && (mine || M.status != DEC_OK))) return;
	const bool report = f < nframes && (MAXQ == 12 ? (mine || M.status != DEC_OK) : (mine && M.status == DEC_OK));
	bool live = have && mine && M.status == DEC_OK && first + M.blocksize <= capacity_samples;
	const bool fits = !(have && mine && M.status == DEC_OK) || live;
	const uint32_t bs_lane = live ? M.blocksize : 0u;
	const uint32_t ca = M.channel_assignment;
	const uint32_t bps = (uint32_t)P.bps;
	uint32_t sub_bps = bps;
	if((ca == 1 && cidx == 1) || (ca == 2 && cidx == 0) || (ca == 3 && cidx == 1)) sub_bps++;

	// ---- per-lane set-up: subframe header, warm-up samples, predictor (stream_decoder.c:2949-3297)
	BitRd br;
	br.init(frames + off, live ? len : 0u, live ? M.sub_bit[cidx < FB200_MAX_CHANNELS ? cidx : 0] : 0u);
	const uint32_t lead = br.pos - (live ? M.sub_bit[cidx < FB200_MAX_CHANNELS ? cidx : 0] : 0u);
	SubHdr h;
	h.type = 255; h.order = 0; h.wasted = 0; h.bps = sub_bps; h.precision = 0; h.shift = 0;
	bool bad = false;
	if(live) {
		h = read_sub_header(br, sub_bps);
		if(h.type == 255 || (h.type >= 2 && bs_lane <= h.order) || h.order > (uint32_t)MAXQ) { bad = true; h.type = 0; h.order = 0; }
	}
	const uint32_t order = live ? h.order : 0u;
	// the widest predictor in the warp picks the instantiation (warp-uniform)
	uint32_t omax = order;
#pragma unroll
	for(int o = 16; o > 0; o >>= 1) omax = max(omax, __shfl_xor_sync(0xffffffffu, omax, o));
	uint32_t bs_max = bs_lane;
#pragma unroll
	for(int o = 16; o > 0; o >>= 1) bs_max = max(bs_max, __shfl_xor_sync(0xffffffffu, bs_max, o));

	int32_t cval = 0;
	int qbuf[MAXQ], wbuf[MAXQ];
#pragma unroll
	for(int j = 0; j < MAXQ; j++) { qbuf[j] = 0; wbuf[j] = 0; }
	uint32_t po = 0, method = 0;
	bool lane_wide = false;
	if(live && !bad) {
		if(h.type == 0) cval = br.get_signed(h.bps);
		else if(h.type >= 2) {
#pragma unroll
			for(int j = 0; j < MAXQ; j++)
				if(j < (int)order) wbuf[j] = br.get_signed(h.bps);
			if(h.type == 3) {
				const uint32_t prec = br.get(4);
				if(prec == 15) bad = true;
				h.precision = prec + 1;
				h.shift = br.get_signed(5);
				if(h.shift < 0) bad = true;
				uint32_t abs_sum = 0;
#pragma unroll
				for(int j = 0; j < MAXQ; j++)
					if(j < (int)order) { qbuf[j] = br.get_signed(h.precision); abs_sum += (uint32_t)abs(qbuf[j]); }
				// variant rule of stream_decoder.c:3243-3247 (lpc.c:942-968)
				const unsigned long long max_abs = 1ull << (h.bps - 1);
				const unsigned long long max_pred = max_abs * abs_sum;
				const unsigned long long max_after = (unsigned long long)(-1 * ((-1 * (long long)max_pred) >> (h.shift < 0 ? 0 : h.shift)));
				lane_wide = !(dec_silog2((long long)(max_abs + max_after)) <= 32 && dec_silog2((long long)max_pred) <= 32);
			}
			else {
				// fixed predictors as taps (fixed.c:571-629); 32-bit arithmetic agrees with the reference's for bps <= 25
				const int tab[5][4] = {{0, 0, 0, 0}, {1, 0, 0, 0}, {2, -1, 0, 0}, {3, -3, 1, 0}, {4, -6, 4, -1}};
#pragma unroll
				for(int j = 0; j < 4; j++) qbuf[j] = tab[order][j];
			}
			method = br.get(2);
			po = br.get(4);
			const uint32_t psamples = bs_lane >> po;
			if(method > 1 || (po > 0 ? (psamples < order || (psamples << po) != bs_lane) : bs_lane < order)) bad = true;
		}
		if(br.overrun()) bad = true;
	}
	if(bad) live = false;  // a broken subframe decodes nothing; its partner lanes still run (the frame is reported bad)
	if(subinfo && have && report) {
		DecSubframeInfo &I = subinfo[(size_t)f * ch + cidx];
		I.type = (uint8_t)(h.type == 255 ? 0 : h.type); I.order = (uint8_t)order; I.wasted = (uint8_t)h.wasted; I.precision = (uint8_t)h.precision;
		I.shift = (int8_t)h.shift; I.method = (uint8_t)method; I.porder = (uint8_t)po; I.pad = 0;
		for(int j = 0; j < FB200_MAX_LPC_ORDER; j++) { I.qlp[j] = (h.type == 3 && j < MAXQ) ? qbuf[j < MAXQ ? j : 0] : 0; I.warmup[j] = j < MAXQ ? wbuf[j < MAXQ ? j : 0] : 0; }
		if(h.type == 0) I.warmup[0] = cval;
	}
	const uint32_t plen = method ? kRice2ParamLen : kRiceParamLen, pesc = method ? kRice2Escape : kRiceEscape;
	const int shift = h.type == 3 ? h.shift : 0;
	int32_t *dst = pcm + (size_t)first * ch + cidx;
	const bool any_wide = __any_sync(0xffffffffu, lane_wide && live);
	const uint32_t bs_eff = live ? bs_lane : 0u;

	// CONSTANT: one warm-up sample, first-order predictor, no residual bits; VERBATIM: escape-coded "residuals" of the sample width
	bool esc0 = !live;
	uint32_t raw0 = 0, order_eff = order;
	if(live && h.type == 0) { esc0 = true; order_eff = 1; wbuf[0] = cval; qbuf[0] = 1; }
	if(live && h.type == 1) { esc0 = true; raw0 = h.bps; }
	if(!live) order_eff = 0;

	DecLaneMismatch mm;
	mm.hit = false; mm.sample = 0; mm.expected = 0; mm.got = 0;
#define FB200_DEC_RUN2(MO, WD, CHT)                                                                                                          \
	dec_lane_loop<MO, WD, CHT, CMP>(br, bs_eff, bs_max, order_eff, h.wasted, shift, WD && lane_wide, q, w, esc0, raw0, po, plen, pesc, dst,    \
	                                (uint32_t)ch, ca, cidx, bps, bad, mm)
#define FB200_DEC_RUN(MO)                                                                                                                    \
	do {                                                                                                                                       \
		int q[MO], w[MO];                                                                                                                      \
		_Pragma("unroll") for(int j = 0; j < MO; j++) { q[j] = qbuf[j < MAXQ ? j : 0]; w[j] = wbuf[j < MAXQ ? j : 0]; }                       \
		if(any_wide) { if(ch == 2) FB200_DEC_RUN2(MO, true, 2); else FB200_DEC_RUN2(MO, true, 0); }                                            \
		else { if(ch == 2) FB200_DEC_RUN2(MO, false, 2); else FB200_DEC_RUN2(MO, false, 0); }                                                  \
	} while(0)
	if(MAXQ == 12) {
		if(omax <= 8) FB200_DEC_RUN(8);
		else FB200_DEC_RUN(12);
	}
	else FB200_DEC_RUN(MAXQ);
#undef FB200_DEC_RUN
#undef FB200_DEC_RUN2

	// ---- frame end: zero padding to a byte boundary (stream_decoder.c:3359-3373, read_zero_padding_) + CRC-16 must end at
	// (or, in index mode, before) the given end
	uint32_t status = M.status;
	uint32_t frame_bytes = 0;
	if(have && mine && M.status == DEC_OK) {
		if(!fits) status = DEC_LENGTH;
		if(br.overrun()) bad = true;
		if((int)cidx == ch - 1 && live) {
			const uint32_t npad = (8u - ((br.pos - lead) & 7u)) & 7u;
			if(npad && br.get(npad) != 0u) bad = true;
			const uint32_t consumed = (br.pos - lead + 7) >> 3;
			frame_bytes = consumed + 2;
			if(P.loose_end ? frame_bytes > len : frame_bytes != len) status = DEC_LENGTH;
		}
	}
	// fold the lanes of a frame: any bad subframe makes the frame bad; the last channel's lane knows the length
	uint32_t badmask = (have && bad) ? 1u : 0u, st = status, fb = frame_bytes;
	for(int o = 1; o < chl; o <<= 1) {
		badmask |= __shfl_xor_sync(0xffffffffu, badmask, o);
		const uint32_t so = __shfl_xor_sync(0xffffffffu, st, o);
		st = st != DEC_OK ? st : so;
		fb = max(fb, __shfl_xor_sync(0xffffffffu, fb, o));
	}
	if(report && cidx == 0) {
		if(st == DEC_OK && badmask) st = DEC_PARSE;
		meta[f].status = st;
		meta[f].frame_bytes = fb;
		if(status_out && st != DEC_OK) status_out[f] = st | (M.blocksize << 8);  // good frames get theirs after the CRC-16 check
	}
	if constexpr(CMP) {
		// the lowest channel with a mismatch, then its first mismatching sample (stream_encoder.c:5203-5212: channel first)
		uint32_t key = (have && mm.hit) ? cidx : ~0u, smp = mm.sample;
		int32_t ex = mm.expected, got = mm.got;
		for(int o = 1; o < chl; o <<= 1) {
			const uint32_t ko = __shfl_xor_sync(0xffffffffu, key, o), so = __shfl_xor_sync(0xffffffffu, smp, o);
			const int32_t eo = __shfl_xor_sync(0xffffffffu, ex, o), go = __shfl_xor_sync(0xffffffffu, got, o);
			if(ko < key) { key = ko; smp = so; ex = eo; got = go; }
		}
		if(report && cidx == 0) {
			DecVerdict V;
			V.channel = key; V.sample = smp; V.expected = ex; V.got = got;
			verdict[f] = V;
		}
	}
}

// ================================================================ k_dec_pack
// int32 samples -> packed little-endian 16- / 24-bit PCM (the inverse of the encoder's k_unpack): the layout a WAV / AIFF
// writer stores, and half / three quarters of the bytes on the way back over PCIe. One thread = 4 samples.
template <int BYTES>
__global__ void __launch_bounds__(256) k_dec_pack(const int32_t *__restrict__ pcm, uint8_t *__restrict__ out, unsigned long long n)
{
	const unsigned long long i0 = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
	if(i0 >= n) return;
	if(i0 + 4 <= n && ((reinterpret_cast<uintptr_t>(pcm + i0) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out + i0 * BYTES) & 3) == 0)) {
		const int4 v = *reinterpret_cast<const int4 *>(pcm + i0);
		uint32_t *o = reinterpret_cast<uint32_t *>(out + i0 * BYTES);
		if(BYTES == 2) {
			o[0] = ((uint32_t)v.x & 0xffffu) | ((uint32_t)v.y << 16);
			o[1] = ((uint32_t)v.z & 0xffffu) | ((uint32_t)v.w << 16);
		}
		else {
			const uint32_t a = (uint32_t)v.x & 0xffffffu, b = (uint32_t)v.y & 0xffffffu, c = (uint32_t)v.z & 0xffffffu, e = (uint32_t)v.w & 0xffffffu;
			o[0] = a | (b << 24);
			o[1] = (b >> 8) | (c << 16);
			o[2] = (c >> 16) | (e << 8);
		}
		return;
	}
	for(unsigned long long i = i0; i < n && i < i0 + 4; i++) {
		const uint32_t v = (uint32_t)pcm[i];
		out[i * BYTES] = (uint8_t)v;
		out[i * BYTES + 1] = (uint8_t)(v >> 8);
		if(BYTES == 3) out[i * BYTES + 2] = (uint8_t)(v >> 16);
	}
}

// ================================================================ k_dec_crc
// Device table of the CRC-16 pass (uint16): [0, 1024) slicing-by-4 tables T[k][b] = CRC of byte b followed by k zero bytes;
// [1024 + (Lw - 1) * 5 + s] = x^(32 Lw 2^s) mod (x^16+x^15+x^2+1) for Lw = 1..kDecCrcLw, s < 5: the multipliers that combine
// the 32 lane CRCs of a frame (crc(A || B) = crc(A) x^|B| + crc(B), init 0).
constexpr int kDecCrcLw = 1024;
constexpr int kDecCrcTabEntries = 1024 + kDecCrcLw * 5;
__global__ void k_dec_crc_tables(uint16_t *__restrict__ tab)
{
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if(t < 256) {
		uint32_t prev = crc16_entry((uint32_t)t);
		tab[t] = (uint16_t)prev;
		for(int k = 1; k < 4; k++) {
			prev = ((prev << 8) & 0xffffu) ^ crc16_entry(prev >> 8);  // one more zero byte
			tab[k * 256 + t] = (uint16_t)prev;
		}
	}
	if(t < kDecCrcLw * 5) {
		const uint32_t Lw = (uint32_t)(t / 5) + 1u;
		const uint32_t m = gf16_xpow((32ull * Lw) << (t % 5));
		tab[1024 + t] = (uint16_t)m;
	}
}

// One warp per frame; lane l owns Lw 4-byte groups ending (32 - l - 1) * Lw groups before the frame's last data byte. The
// frame starts at an arbitrary byte address: a group is assembled from two aligned words with a funnel shift; groups that
// would start in front of the frame are zero bytes, which a CRC with initial value 0 ignores -- so every lane runs the same
// Lw slicing-by-4 steps with no alignment cases, and the combine multipliers depend on Lw only. Writes the final status.
__global__ void __launch_bounds__(128) k_dec_crc(const uint8_t *__restrict__ frames, const unsigned long long *__restrict__ begins,
                                                int nframes, DecFrameMeta *__restrict__ meta, uint32_t *__restrict__ status_out, uint32_t *__restrict__ bytes_out,
                                                const uint16_t *__restrict__ crc_tab)
{
	__shared__ uint16_t s_tab[4 * 256];
	for(int e = threadIdx.x; e < 4 * 256 / 2; e += blockDim.x) reinterpret_cast<uint32_t *>(s_tab)[e] = __ldg(reinterpret_cast<const uint32_t *>(crc_tab) + e);
	__syncthreads();
	const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if(f >= nframes) return;
	const DecFrameMeta M = meta[f];
	if(M.status != DEC_OK) return;
	const unsigned long long off = begins[f];
	const uint32_t len = M.frame_bytes;
	if(len < 3) return;
	const uint32_t nbytes = len - 2;
	const uint8_t *p = frames + off;
	const uint32_t Lw = (nbytes + 127) / 128;                       // groups per lane
	const long long first = (long long)nbytes - (long long)(32 - lane) * Lw * 4;  // frame offset of this lane's first byte (may be < 0)
	const uintptr_t a0 = reinterpret_cast<uintptr_t>(p);
	uint32_t crc = 0;
	// aligned word stream: word index relative to the aligned word holding frame byte 0
	const uint32_t lead = (uint32_t)(a0 & 3);
	const uint32_t *wbase = reinterpret_cast<const uint32_t *>(a0 - lead);
	long long o = first;
	// previous aligned word (big-endian) for the funnel; loaded lazily when the group touches the frame
	uint32_t wprev = 0;
	bool have_prev = false;
	for(uint32_t g = 0; g < Lw; g++, o += 4) {
		uint32_t x = 0;
		if(o + 3 >= 0) {
			// bytes o .. o+3 of the frame sit at byte (lead + o) of the aligned stream
			const long long sb = (long long)lead + o;               // may be negative only by up to 3 when o < 0 <= o + 3
			const long long wi = sb >= 0 ? (sb >> 2) : -1;
			const uint32_t sh = (uint32_t)(sb & 3) * 8;
			uint32_t w0;
			if(wi < 0) w0 = 0;
			else if(have_prev) w0 = wprev;
			else w0 = __byte_perm(__ldg(wbase + wi), 0, 0x0123);
			const uint32_t w1 = sh ? __byte_perm(__ldg(wbase + wi + 1), 0, 0x0123) : 0u;  // never past the CRC-16 bytes' word
			x = sh ? __funnelshift_l(w1, w0, sh) : w0;
			if(sh) { wprev = w1; have_prev = true; }
			if(o < 0) x &= 0xffffffffu >> (8u * (uint32_t)(-o));      // bytes in front of the frame are zeros
		}
		crc = (uint32_t)s_tab[3 * 256 + (((crc >> 8) ^ (x >> 24)) & 0xffu)] ^ (uint32_t)s_tab[2 * 256 + ((crc ^ (x >> 16)) & 0xffu)] ^
		      (uint32_t)s_tab[256 + ((x >> 8) & 0xffu)] ^ (uint32_t)s_tab[x & 0xffu];
	}
#pragma unroll
	for(int s = 0; s < 5; s++) {
		const uint32_t m = Lw <= (uint32_t)kDecCrcLw ? __ldg(&crc_tab[1024 + (Lw - 1) * 5 + s]) : gf16_xpow((32ull * Lw) << s);
		const uint32_t other = __shfl_down_sync(0xffffffffu, crc, 1 << s);
		if((lane & ((2 << s) - 1)) == 0) crc = gf16_mul(crc, m) ^ other;
	}
	if(lane == 0) {
		const uint32_t want = ((uint32_t)p[nbytes] << 8) | p[nbytes + 1];
		uint32_t st = DEC_OK;
		if(crc != want) { st = DEC_CRC16; meta[f].status = DEC_CRC16; }
		if(status_out) status_out[f] = st | (M.blocksize << 8);  // low byte: status, upper: decoded blocksize
		if(bytes_out) bytes_out[f] = len;
	}
}

// ================================================================ verify of fb200_encode_files_*
// vb[i] = min(voff[i], cap), i <= nframes: the frames of the encode-order scratch as the decode kernels see them. A frame the
// scratch could not hold ends up shorter than a header (DEC_LENGTH) and is never read past cap.
__global__ void __launch_bounds__(256) k_verify_bounds(const unsigned long long *__restrict__ voff, unsigned long long nframes, unsigned long long cap,
                                                      unsigned long long *__restrict__ vb)
{
	const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
	if(i <= nframes) vb[i] = min(voff[i], cap);
}

// One warp per file, over its frames in file order: the first frame that fails (decode, CRC, header facts, frame number,
// blocksize, then samples) gives the file's record, as the reference's verify stops at its first bad frame.
__global__ void __launch_bounds__(128) k_verify_files(const DecFrameMeta *__restrict__ meta, const DecVerdict *__restrict__ verdict,
                                                     const FileFrames *__restrict__ files, const FileSeg *__restrict__ segs, int nfiles,
                                                     uint32_t channels, uint32_t blocksize, uint32_t sample_rate, fb200_file_verify_info *__restrict__ info)
{
	const int f = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
	if(f >= nfiles) return;
	const FileFrames F = files[f];
	const uint32_t n = F.nfull + (F.tail != ~0u ? 1u : 0u);
	const uint32_t tail_bs = (uint32_t)(segs[2 * f + 1].n / channels);
	fb200_file_verify_info r;
	memset(&r, 0, sizeof r);
	for(uint32_t j0 = 0; j0 < n; j0 += 32) {
		const uint32_t j = j0 + (uint32_t)lane;
		uint32_t why = FB200_VERIFY_OK, fs = DEC_OK, v = 0;
		if(j < n) {
			v = j < F.nfull ? F.first + j : F.tail;
			const DecFrameMeta &M = meta[v];
			why = FB200_VERIFY_DECODER_ERROR;
			if(M.status != DEC_OK) fs = M.status;
			else if(M.sample_rate != sample_rate) fs = DEC_MISMATCH;
			else if(M.variable || M.frame_number_lo != j || M.blocksize != (j < F.nfull ? blocksize : tail_bs)) fs = DEC_WRONG_FRAME;
			else why = verdict[v].channel != ~0u ? FB200_VERIFY_MISMATCH : FB200_VERIFY_OK;
		}
		const unsigned bad = __ballot_sync(0xffffffffu, why != FB200_VERIFY_OK);
		if(!bad) continue;
		if(lane == __ffs(bad) - 1) {
			r.status = why;
			r.frame_number = j;
			r.frame_status = fs;
			if(why == FB200_VERIFY_MISMATCH) {
				const DecVerdict V = verdict[v];
				r.channel = V.channel; r.sample = V.sample;
				r.absolute_sample = (unsigned long long)j * blocksize + V.sample;
				r.expected = V.expected; r.got = V.got;
			}
			info[f] = r;
		}
		return;
	}
	if(lane == 0) info[f] = r;
}

}  // namespace fb200
