// emit_kernel.cuh -- k_emit3: one CTA per frame, frame assembled in shared memory and stored straight to its
// final place in the output stream.
//
// Replaces k_emit2 + k_scan + k_gather and the per-frame slot buffer for 1- and 2-channel streams.
// Reference semantics kept bit for bit: FLAC__frame_add_header (stream_encoder_framing.c:245-391),
// FLAC__subframe_add_* (:393-520), add_residual_partitioned_rice_ (:538-594),
// FLAC__bitwriter_write_rice_signed_block (bitwriter.c:575-706), zero pad + CRC-16 (stream_encoder.c:3465-3480,
// crc.c:376-396), channel assignment argmin (stream_encoder.c:3937-3972).
//
// What round 1's k_emit2 spent its time on (profiled): many thread-instructions per sample, stalls at block
// barriers (14+ barriers per frame: one exclusive scan and one re-staging per channel), shared-memory bank
// conflicts, a byte-at-a-time CRC, a worst-case zero fill and a slot -> gather double copy.  This kernel:
//   * stages the caller's interleaved int32 block ONCE with a 1-D TMA bulk copy (cp.async.bulk + mbarrier), forms
//     the two signals the channel assignment picked (L/R/M/S, wasted bits shifted out) in place;
//   * a thread owns one run of R_T consecutive samples of one channel (row layout of k_search4: 36-word rows ->
//     every 128-bit access is conflict free); residual, zig-zag and bit count in one rolled pass that writes the
//     zig-zagged residuals back in place; ONE block scan for the whole frame (both channels);
//   * runs are packed independently MSB-first (unary zeros + stop bit + k low bits go out as one field whenever they
//     fit 32 bits); only the first/last word of a run is shared with a neighbour (atomicOr);
//   * the frame is laid into shared memory so that its END is word aligned: the CRC-16 is a slicing-by-4 pass over
//     equal word chunks + GF(2) combine, with no alignment cases;
//   * frame offsets come from a single-pass decoupled look-back over frame byte counts; the frame is written
//     directly to out + offset.
#pragma once

#include <type_traits>

#include "device_common.cuh"
#include "search_kernel.cuh"  // row layout constants (kSearch4ZeroRow)

namespace fb200 {

// ---------------------------------------------------------------- CRC-16 slicing tables
// T[k][b] = CRC-16 (poly 0x8005, init 0, MSB first; crc.c:78-342) of byte b followed by k zero bytes.
// Filled once per device by k_crc16_tables (encoder.cu uploads nothing: the table is computed on the device).
__global__ void k_crc16_tables(uint16_t *__restrict__ tab)
{
	const int b = threadIdx.x;
	uint32_t c = (uint32_t)b << 8;
#pragma unroll
	for(int j = 0; j < 8; j++) c = (c & 0x8000u) ? ((c << 1) ^ 0x8005u) & 0xffffu : (c << 1) & 0xffffu;
	tab[b] = (uint16_t)c;
	__syncthreads();
	uint32_t prev = c;
	for(int k = 1; k < 4; k++) {
		prev = ((prev << 8) & 0xffffu) ^ tab[prev >> 8];
		tab[k * 256 + b] = (uint16_t)prev;
	}
	// combine multipliers: tab[1024 + (Lw >> 1) * 9 + s] = x^(32 Lw 2^s) mod (x^16+x^15+x^2+1) for odd Lw < 64, s < 9
	for(int idx = b; idx < kCrcLwRows * 9; idx += blockDim.x) {
		const uint32_t Lw = 2u * (uint32_t)(idx / 9) + 1u;
		unsigned long long e = (32ull * Lw) << (idx % 9);
		uint32_t m = 1;
		for(int j = 0; e; j++, e >>= 1)
			if(e & 1ull) m = gf16_mul(m, kCrcXPow2[j % 15]);
		tab[1024 + idx] = (uint16_t)m;
	}
	__syncthreads();
	// nibble products: tab[kCrcMulBase + ((row * 9 + s) * 4 + pos) * 16 + n] = (n << 4 pos) * x^(32 Lw 2^s): a GF(2^16) product by a
	// level multiplier becomes four 16-entry lookups instead of a 16-step shift-and-add
	for(int idx = b; idx < kCrcLwRows * 9 * 64; idx += blockDim.x) {
		const uint32_t m = tab[1024 + idx / 64];
		const uint32_t pos = (uint32_t)(idx >> 4) & 3u, n = (uint32_t)idx & 15u;
		tab[kCrcMulBase + idx] = (uint16_t)gf16_mul(n << (4 * pos), m);
	}
}

// decoupled look-back status word: value << 24 | epoch (22 bits) << 2 | flag (1 aggregate, 2 inclusive prefix)
__device__ __forceinline__ unsigned long long lb_pack(unsigned long long value, unsigned epoch, unsigned flag)
{
	return (value << 24) | ((unsigned long long)(epoch & kLbEpochMask) << 2) | flag;
}
__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long *p)
{
	unsigned long long v;
	asm volatile("ld.volatile.global.u64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long *p, unsigned long long v)
{
	asm volatile("st.volatile.global.u64 [%0], %1;\n" ::"l"(p), "l"(v) : "memory");
}

// Bit packer of one run (the paths whose Rice parameter changes inside a run, and verbatim subframes). Store discipline of
// the pack pass: a word is plain-stored by the one run whose bits reach the word's last bit; a run's trailing partial word is
// NOT written by it but handed back (last_word / last_bits) and OR-ed in after the CTA barrier that ends the pass, together
// with the header fields -- so the pass itself has no atomics and no read-modify-write.
struct RunPacker {
	uint32_t *words;
	uint32_t cur, pos;
	int widx;
	__device__ __forceinline__ void init(uint32_t *w, uint32_t bitpos)
	{
		words = w; pos = bitpos; widx = (int)(bitpos >> 5); cur = 0;
	}
	// n zero bits
	__device__ __forceinline__ void skip(uint32_t n)
	{
		pos += n;
		const int nw = (int)(pos >> 5);
		if(nw != widx) { words[widx] = cur; widx = nw; cur = 0; }  // words skipped over entirely stay zero (pre-zeroed buffer)
	}
	// 1..32 bits, value < 2^nbits
	__device__ __forceinline__ void put(uint32_t value, uint32_t nbits)
	{
		const uint32_t off = pos & 31u;
		const unsigned long long v = (unsigned long long)value << (64u - off - nbits);
		cur |= (uint32_t)(v >> 32);
		pos += nbits;
		if(off + nbits >= 32u) {
			words[widx] = cur;
			widx++;
			cur = (uint32_t)v;
		}
	}
};

// residuals of G consecutive outputs (narrow: 32-bit accumulation, lpc.c:321-553; wide: the 64-bit predictor on
// the FP64 pipe, exact -- see group_abs_sum_f64)
template <int G, int MAXORD, int NTAPS>
__device__ __forceinline__ void group_residual_narrow(const int (&xg)[MAXORD + G], const int (&q)[MAXORD], int shift, int (&r)[G])
{
#pragma unroll
	for(int m = 0; m < G; m++) {
		int sum = 0;
#pragma unroll
		for(int j = 0; j < NTAPS; j++) sum += q[j] * xg[MAXORD + m - 1 - j];
		r[m] = xg[MAXORD + m] - (sum >> shift);
	}
}

template <int G, int MAXORD, int NTAPS>
__device__ __forceinline__ void group_residual_wide(const int (&xg)[MAXORD + G], const int (&q)[MAXORD], int shift, int (&r)[G])
{
	constexpr double kFloorMagic = 6755399441055744.0;  // 1.5 * 2^52
	const double scale = __hiloint2double((1023 - shift) << 20, 0);  // 2^-shift: qd = q / 2^shift keeps the significand
	double qd[NTAPS];
#pragma unroll
	for(int j = 0; j < NTAPS; j++) qd[j] = __dmul_rn((double)q[j], scale);
	double xd[MAXORD + G];
#pragma unroll
	for(int i = MAXORD - NTAPS; i < MAXORD + G; i++) xd[i] = int_to_double_exact(xg[i]);
#pragma unroll
	for(int m = 0; m < G; m++) {
		double sum = 0.0;
#pragma unroll
		for(int j = 0; j < NTAPS; j++) sum = fma(qd[j], xd[MAXORD + m - 1 - j], sum);
		const double t = __dadd_rd(sum, kFloorMagic);                            // floor(sum) + magic
		const double rr = __dadd_rn(__dsub_rn(xd[MAXORD + m], t), kFloorMagic);  // x - floor(sum), an exact integer
		r[m] = __double2loint(__dadd_rn(rr, kFloorMagic));                        // low word of (magic + rr) == (int)rr
	}
}

// Frame header (stream_encoder_framing.c:245-391): returns its length in bits (CRC-8 included); the warp that passes build = true
// writes the header bytes to hdr[4] (big-endian words, left aligned): one header byte per lane, CRC-8 from per-byte CRCs. Its
// content does not depend on anything the emit passes compute, only its position does.
__device__ __forceinline__ uint32_t emit3_frame_header(const EncK &P, int blk, int ca, bool build, int lane, uint32_t *hdr)
{
	const int bs = P.bs;
	const uint32_t gblk = P.blk0 + (uint32_t)blk;
	const uint32_t frame_number = P.first_frame + (P.file_blocks ? gblk % (uint32_t)P.file_blocks : gblk);
	uint32_t bs_code, bs_hint = 0, sr_code, sr_hint = 0;
	switch(bs) {
		case 192: bs_code = 1; break; case 576: bs_code = 2; break; case 1152: bs_code = 3; break;
		case 2304: bs_code = 4; break; case 4608: bs_code = 5; break; case 256: bs_code = 8; break;
		case 512: bs_code = 9; break; case 1024: bs_code = 10; break; case 2048: bs_code = 11; break;
		case 4096: bs_code = 12; break; case 8192: bs_code = 13; break; case 16384: bs_code = 14; break;
		case 32768: bs_code = 15; break;
		default: bs_code = bs_hint = (bs <= 0x100) ? 6 : 7; break;
	}
	switch(P.sample_rate) {
		case 88200: sr_code = 1; break; case 176400: sr_code = 2; break; case 192000: sr_code = 3; break;
		case 8000: sr_code = 4; break; case 16000: sr_code = 5; break; case 22050: sr_code = 6; break;
		case 24000: sr_code = 7; break; case 32000: sr_code = 8; break; case 44100: sr_code = 9; break;
		case 48000: sr_code = 10; break; case 96000: sr_code = 11; break;
		default:
			if(P.sample_rate <= 255000 && P.sample_rate % 1000 == 0) sr_code = sr_hint = 12;
			else if(P.sample_rate <= 655350 && P.sample_rate % 10 == 0) sr_code = sr_hint = 14;
			else if(P.sample_rate <= 0xffff) sr_code = sr_hint = 13;
			else sr_code = 0;
			break;
	}
	uint32_t utf8_len;
	if(frame_number < 0x80) utf8_len = 1;
	else if(frame_number < 0x800) utf8_len = 2;
	else if(frame_number < 0x10000) utf8_len = 3;
	else if(frame_number < 0x200000) utf8_len = 4;
	else if(frame_number < 0x4000000) utf8_len = 5;
	else utf8_len = 6;
	const uint32_t header_bits = 32 + 8 * utf8_len + (bs_hint ? (bs_hint == 6 ? 8 : 16) : 0) + (sr_hint ? (sr_hint == 12 ? 8 : 16) : 0) + 8;
	if(build) {
		// one header byte per lane; CRC-8 (poly 0x07, crc.c:39-76) of the whole header from per-byte CRCs weighted by
		// x^(8 * bytes behind) -- no serial loop over the header
		const int nb8 = (int)(header_bits >> 3);  // bytes including the CRC-8
		const int pos_bs = 4 + (int)utf8_len;
		const int bs_bytes = bs_hint ? (bs_hint == 6 ? 1 : 2) : 0;
		const int pos_sr = pos_bs + bs_bytes;
		const int sr_bytes = sr_hint ? (sr_hint == 12 ? 1 : 2) : 0;
		uint32_t ca_code;
		switch(ca) { case 0: ca_code = (uint32_t)P.channels - 1; break; case 1: ca_code = 8; break; case 2: ca_code = 9; break; default: ca_code = 10; break; }
		uint32_t bps_code;
		switch(P.bps) { case 8: bps_code = 1; break; case 12: bps_code = 2; break; case 16: bps_code = 4; break; case 20: bps_code = 5; break; case 24: bps_code = 6; break; case 32: bps_code = 7; break; default: bps_code = 0; break; }
		const uint32_t v = frame_number;
		uint32_t byte = 0;
		const int i = lane;
		if(i == 0) byte = 0xff;                                   // sync 0x3ffe, reserved 0, fixed-blocksize stream
		else if(i == 1) byte = 0xf8;
		else if(i == 2) byte = (bs_code << 4) | sr_code;
		else if(i == 3) byte = (ca_code << 4) | (bps_code << 1);
		else if(i < pos_bs) {                                     // UTF-8 style frame number (bitwriter.c:832-933)
			const int j = i - 4;
			if(j == 0) {
				switch(utf8_len) {
					case 1: byte = v; break;
					case 2: byte = 0xC0 | (v >> 6); break;
					case 3: byte = 0xE0 | (v >> 12); break;
					case 4: byte = 0xF0 | (v >> 18); break;
					case 5: byte = 0xF8 | (v >> 24); break;
					default: byte = 0xFC | (v >> 30); break;
				}
			}
			else byte = 0x80 | ((v >> (6 * ((int)utf8_len - 1 - j))) & 0x3F);
		}
		else if(i < pos_sr) byte = ((uint32_t)bs - 1) >> (8 * (bs_bytes - 1 - (i - pos_bs)));
		else if(i < nb8 - 1) {
			const uint32_t sv = sr_hint == 12 ? (uint32_t)P.sample_rate / 1000 : sr_hint == 13 ? (uint32_t)P.sample_rate : (uint32_t)P.sample_rate / 10;
			byte = sv >> (8 * (sr_bytes - 1 - (i - pos_sr)));
		}
		byte &= 0xffu;
		uint32_t c = 0;
		if(i < nb8 - 1) {
			c = byte;
#pragma unroll
			for(int j = 0; j < 8; j++) c = (c & 0x80u) ? ((c << 1) ^ 0x07u) & 0xffu : (c << 1) & 0xffu;
			// times x^(8 * (nb8 - 2 - i)) in GF(2)[x] / (x^8 + x^2 + x + 1)
			const uint32_t wgt = kCrc8XPow8[nb8 - 2 - i];
			uint32_t r = 0;
#pragma unroll
			for(int j = 7; j >= 0; j--) {
				r = (r & 0x80u) ? ((r << 1) ^ 0x07u) & 0xffu : (r << 1) & 0xffu;
				if((wgt >> j) & 1u) r ^= c;
			}
			c = r;
		}
#pragma unroll
		for(int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
		if(i == nb8 - 1) byte = c;
		if(i >= nb8) byte = 0;
		uint32_t w = byte << (24 - 8 * (i & 3));
		w |= __shfl_xor_sync(0xffffffffu, w, 1);
		w |= __shfl_xor_sync(0xffffffffu, w, 2);
		if((i & 3) == 0 && i < 16) hdr[i >> 2] = w;  // big-endian words, left aligned
	}

	return header_bits;
}

// The end of a frame that sits in `words` with its END word aligned (s0 leading pad bytes, CRC-16 slot at word wend): CRC-16,
// decoupled look-back for the frame's byte offset, copy to its place in the stream. crc_tab: shared memory for the slicing
// tables and the nibble-product tables (>= 3.2 KB, may alias anything that is dead by now). Called by every thread of the CTA
// after a barrier that completed `words`.
__device__ __forceinline__ void emit3_finish(const Emit3Args &A, Emit3Shared &S, uint32_t *words, uint16_t *crc_tab, int blk, int ca, uint32_t nbytes,
                                             uint32_t s0, uint32_t wend, bool fits)
{
	const int tid = threadIdx.x, NT = blockDim.x, lane = tid & 31, warp = tid >> 5;
	// ---- CRC-16 over the frame: equal word chunks aligned to the (word aligned) end, slicing-by-4, GF(2) combine.
	// The signals are dead: the slicing tables go where they were.
	int Lw = ((int)wend + NT - 1) / NT;
	Lw |= 1;  // odd chunk length: conflict-free strided reads
	const bool lw_tab = Lw < 2 * kCrcLwRows;
	uint16_t *const mul_tab = crc_tab + 1024;  // [9 levels][4 nibble positions][16]: products by x^(32 Lw 2^s)
	for(int i = tid; i < 4 * 256 / 2; i += NT) reinterpret_cast<uint32_t *>(crc_tab)[i] = __ldg(reinterpret_cast<const uint32_t *>(A.crc_tab) + i);
	if(lw_tab)
		for(int i = tid; i < 9 * 64 / 2; i += NT)
			reinterpret_cast<uint32_t *>(mul_tab)[i] = __ldg(reinterpret_cast<const uint32_t *>(A.crc_tab + kCrcMulBase + (Lw >> 1) * (9 * 64)) + i);
	// crc * x^(32 Lw 2^lev): four 16-entry lookups (a 16-step shift-and-add when Lw is outside the table)
	auto mul_level = [&](uint32_t c, int lev) -> uint32_t {
		if(lw_tab) {
			const uint16_t *t = mul_tab + lev * 64;
			return (uint32_t)t[c & 15u] ^ (uint32_t)t[16 + ((c >> 4) & 15u)] ^ (uint32_t)t[32 + ((c >> 8) & 15u)] ^ (uint32_t)t[48 + (c >> 12)];
		}
		return gf16_mul(c, S.mlev[lev]);
	};
	// level s of the combine tree multiplies by x^(32 Lw 2^s) (crc(A || B) = crc(A) x^|B| + crc(B), init 0)
	if(tid < 9) {
		uint32_t m;
		if(Lw < 2 * kCrcLwRows) m = __ldg(&A.crc_tab[1024 + (Lw >> 1) * 9 + tid]);
		else {
			unsigned long long e = (32ull * (unsigned)Lw) << tid;
			m = 1;
			for(int j = 0; e; j++, e >>= 1)
				if(e & 1ull) m = gf16_mul(m, kCrcXPow2[j % 15]);
		}
		S.mlev[tid] = m;
	}
	// the look-back runs here too (warp 1, or warp 0 of a one-warp CTA): its latency hides under the CRC pass
	{
		const int lbw = (NT > 32) ? 1 : 0;
		if(warp == lbw) {
			unsigned long long excl = 0;
			int idx = blk - 1;
			while(idx >= 0) {
				const int j = idx - lane;
				unsigned long long w;
				unsigned flag;
				do {
					flag = 2;  // lanes in front of frame 0 stand for "inclusive prefix 0"
					w = 0;
					if(j >= 0) {
						w = ld_volatile_u64(&A.lookback[j]);
						flag = (((unsigned)(w >> 2)) & kLbEpochMask) == (A.epoch & kLbEpochMask) ? (unsigned)(w & 3u) : 0u;
					}
				} while(__any_sync(0xffffffffu, flag == 0));
				const unsigned incl_mask = __ballot_sync(0xffffffffu, flag == 2);
				const int f = incl_mask ? __ffs((int)incl_mask) - 1 : 32;  // nearest predecessor that already holds an inclusive prefix
				unsigned long long contrib = (lane <= f) ? (w >> 24) : 0ull;
#pragma unroll
				for(int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
				excl += contrib;
				if(incl_mask) break;
				idx -= 32;
			}
			if(lane == 0) {
				st_volatile_u64(&A.lookback[blk], lb_pack(excl + nbytes + 2, A.epoch, 2));
				const unsigned long long basebytes = *A.running_in;
				S.off = basebytes + excl;
				A.offsets[blk] = basebytes + excl;
				if(blk == A.nb - 1) {
					A.offsets[A.nb] = basebytes + excl + nbytes + 2;
					*A.running_out = basebytes + excl + nbytes + 2;
				}
				if(A.chan_assign_out) A.chan_assign_out[blk] = (uint32_t)ca;
			}
		}
	}
	__syncthreads();
	if(fits) {
		const int cstart = (int)wend - (NT - tid) * Lw;
		uint32_t crc = 0;
		for(int w = cstart < 0 ? 0 : cstart; w < cstart + Lw; w++) {
			const uint32_t x = words[w];
			crc = (uint32_t)crc_tab[3 * 256 + (((crc >> 8) ^ (x >> 24)) & 0xffu)] ^ (uint32_t)crc_tab[2 * 256 + ((crc ^ (x >> 16)) & 0xffu)] ^
			      (uint32_t)crc_tab[256 + ((x >> 8) & 0xffu)] ^ (uint32_t)crc_tab[x & 0xffu];
		}
#pragma unroll
		for(int sl = 0; sl < 5; sl++) {
			const uint32_t other = __shfl_down_sync(0xffffffffu, crc, 1 << sl);
			crc = mul_level(crc, sl) ^ other;  // meaningful in lanes that are multiples of 2 << sl; lane 0 is what counts
		}
		if(lane == 0) S.part[warp] = crc;
	}
	__syncthreads();
	if(fits && warp == 0) {
		const int nw = NT >> 5;
		uint32_t crc = lane < nw ? S.part[lane] : 0;
		for(int sl = 0; (1 << sl) < nw; sl++) {
			const uint32_t other = __shfl_down_sync(0xffffffffu, crc, 1 << sl);
			crc = mul_level(crc, 5 + sl) ^ other;
		}
		if(lane == 0) words[wend] = (words[wend] & 0xffffu) | (crc << 16);  // CRC-16, big-endian, right after the frame
	}
	__syncthreads();

	// ---- copy the frame to its place in the stream (byte-granular destination alignment)
	if(fits) {
		const unsigned long long off = S.off;
		const uint32_t totalb = nbytes + 2;
		if(off + totalb > A.out_cap) {
			if(tid == 0) atomicExch(A.err, 1);
			return;
		}
		uint8_t *dst = A.out + off;
		const uint32_t head = min(totalb, (uint32_t)((4u - ((uint32_t)(uintptr_t)dst & 3u)) & 3u));
		auto frame_byte = [&](uint32_t j) -> uint8_t { const uint32_t bb = s0 + j; return (uint8_t)((words[bb >> 2] >> (24 - 8 * (bb & 3))) & 0xffu); };
		if((uint32_t)tid < head) dst[tid] = frame_byte((uint32_t)tid);
		const uint32_t nwd = (totalb - head) >> 2;
		uint32_t *d32 = reinterpret_cast<uint32_t *>(dst + head);
		const uint32_t sb = s0 + head;  // shared-memory byte index of the first aligned destination word
		const uint32_t wsrc = sb >> 2, sh = (sb & 3u) * 8u;
		for(uint32_t i = tid; i < nwd; i += NT) {
			const uint32_t be = sh ? __funnelshift_l(words[wsrc + i + 1], words[wsrc + i], sh) : words[wsrc + i];
			d32[i] = __byte_perm(be, 0, 0x0123);
		}
		const uint32_t tail0 = head + nwd * 4;
		if(tail0 + (uint32_t)tid < totalb) dst[tail0 + tid] = frame_byte(tail0 + (uint32_t)tid);
	}
}

// R_T: samples per run (32 or 36); MAXORD: 8 / 12 / 32; CH: channels in the stream (1 or 2).
// blockDim.x = NT = (bs / R_T) * CH <= 256 (a power of two, TPC = bs / R_T >= 32).
// WIDEK: the stream is deeper than 16 bits, i.e. a predictor may need 64-bit accumulation (lpc.c:786-884); the 16-bit
// instantiations carry no wide code and fit four CTAs per SM.
// PAIR (streams of more than two channels): one CTA per (frame, channel pair) packs the pair's two subframes -- independent
// channels, samples gathered from the interleaved block -- exactly as above, but from bit 0 of its own staging region
// (A.stage) instead of behind a frame header; k_join then splices the pairs of a frame behind its header.
template <int R_T, int MAXORD, int CH, bool WIDEK, bool PAIR>
__global__ void __launch_bounds__(256, WIDEK ? 3 : 4) k_emit3(EncK P, Emit3Args A)
{
	static_assert(R_T == 32 || R_T == 36, "run length");
	static_assert(CH == 1 || CH == 2, "resident emit path: 1 or 2 channels");
	static_assert(!PAIR || CH == 2, "pair mode packs two channels");
	constexpr int G = (R_T == 32) ? 16 : 12, NG = R_T / G, ROWPAD = 36 - R_T;
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int tid = threadIdx.x, NT = blockDim.x, bs = P.bs, lane = tid & 31, warp = tid >> 5;
	const int TPC = bs / R_T;  // threads (runs) per channel
	const int planar_words = kSearch4ZeroRow + TPC * 36;
	Emit3Shared &S = *reinterpret_cast<Emit3Shared *>(smem_raw);
	int32_t *const planar = reinterpret_cast<int32_t *>(smem_raw + (sizeof(Emit3Shared) + 15) / 16 * 16);
	uint32_t *const words = reinterpret_cast<uint32_t *>(reinterpret_cast<unsigned char *>(planar) + emit3_sig_bytes(bs, R_T, CH));
	const int words_cap = (PAIR ? A.pair_words : P.emit3_words) + 8;
	uint16_t *const crc_tab = reinterpret_cast<uint16_t *>(planar);  // loaded after the pack pass, when the signals are dead
	uint64_t *const mbar = reinterpret_cast<uint64_t *>(&S.mbar);

	// ---- which frame: tickets are handed out in launch order, so every lower-numbered frame's CTA is already running
	int blk, pair = 0, npairs = 1;
	if(PAIR) {
		npairs = (P.channels + 1) >> 1;
		blk = (int)blockIdx.x / npairs;
		pair = (int)blockIdx.x - blk * npairs;
	}
	else {
		if(tid == 0) S.blk = (int)(atomicAdd(A.ticket, 1u) - A.ticket_base);
		__syncthreads();
		blk = S.blk;
	}
	const SubframePlan *bp = A.plans + (size_t)blk * P.nsig;

	// ---- raw block -> shared memory with one TMA bulk copy; issued first so that it overlaps the prologue
	const unsigned raw_bytes = (unsigned)bs * CH * 4u;
	int32_t *const raw = planar;  // lands where the planar signals will be: it is pulled into registers first
	if(!PAIR && tid == 0) {
		mbar_init(mbar, 1);
		mbar_fence_init();
		mbar_expect_tx(mbar, raw_bytes);
		tma_bulk_g2s(raw, A.pcm + (size_t)blk * bs * CH, raw_bytes, mbar);
	}

	// ---- channel assignment (stream_encoder.c:3937-3972) and what it implies
	int ca = 0;
	if(!PAIR && CH == 2 && P.do_ms) {
		if(P.loose_ms) ca = (__ldg(&A.blkflags[blk]) & 2) ? 3 : 0;
		else {
			const uint32_t e0 = __ldg(&bp[0].est_bits), e1 = __ldg(&bp[1].est_bits), e2 = __ldg(&bp[2].est_bits), e3 = __ldg(&bp[3].est_bits);
			const uint32_t b0 = e0 + e1, b1 = e0 + e3, b2 = e1 + e3, b3 = e2 + e3;
			uint32_t mn = b0;
			if(b1 < mn) { mn = b1; ca = 1; }
			if(b2 < mn) { mn = b2; ca = 2; }
			if(b3 < mn) { mn = b3; ca = 3; }
		}
	}
	int sidx0 = 0, sidx1 = 1;
	if(PAIR) { sidx0 = 2 * pair; sidx1 = 2 * pair + 1; }
	else if(CH == 2) {
		sidx0 = (ca == 0 || ca == 1) ? 0 : (ca == 2 ? 3 : 2);
		sidx1 = (ca == 0 || ca == 2) ? 1 : 3;
	}
	const bool have1 = !PAIR || sidx1 < P.channels;  // an odd channel count leaves the last pair with one channel
	// this thread's channel / run
	const int myc = (CH == 2 && tid >= TPC) ? 1 : 0;
	const int run = tid - myc * TPC;
	const bool absent = myc == 1 && !have1;
	const SubframePlan *pl = bp + ((myc && have1) ? sidx1 : sidx0);
	const int type = absent ? -1 : __ldg(&pl->type), order = __ldg(&pl->order), wasted = __ldg(&pl->wasted), sbps = __ldg(&pl->bps);
	const int po = __ldg(&pl->porder), method = __ldg(&pl->method), precision = __ldg(&pl->precision), shift = __ldg(&pl->shift);
	const int wide = __ldg(&pl->wide);

	const uint32_t header_bits = PAIR ? 0u : emit3_frame_header(P, blk, ca, warp == (NT >> 5) - 1, lane, S.hdr);

	// ---- zero the word buffer up to an upper bound of the frame: a Rice partition's true length exceeds its
	// estimate (count_rice_bits_in_partition_, stream_encoder.c:4929-4951) by at most n/2 + 1 bits
	int zero_words;
	{
		unsigned long long bound = header_bits + 64;
		bound += (unsigned long long)__ldg(&bp[sidx0].est_bits) + (unsigned)(bs >> 1) + (1u << kMaxPartitionOrder) + 64u;
		if(CH == 2 && have1) bound += (unsigned long long)__ldg(&bp[sidx1].est_bits) + (unsigned)(bs >> 1) + (1u << kMaxPartitionOrder) + 64u;
		unsigned long long zw = (bound >> 5) + 4;
		if(zw > (unsigned long long)words_cap) zw = (unsigned long long)words_cap;
		zero_words = (int)zw;
		for(int i = tid; i < zero_words; i += NT) words[i] = 0;
	}

	// ---- pull the raw block into registers, then (after a barrier) write the planar signals over it
	if(PAIR) {
		// gather the pair's channels from the interleaved block (wasted bits shifted out, stream_encoder.c:3842-3867)
		__syncthreads();
		int32_t *const p0 = planar + kSearch4ZeroRow;
		int32_t *const p1 = planar + planar_words + kSearch4ZeroRow;
		for(int i = tid; i < kSearch4ZeroRow; i += NT) { planar[i] = 0; planar[planar_words + i] = 0; }  // history of row 0
		const int nch = P.channels;
		const int32_t *g = A.pcm + (size_t)blk * bs * nch;
		const int w0 = __ldg(&bp[sidx0].wasted), w1 = have1 ? __ldg(&bp[sidx1].wasted) : 0;
		for(int i = tid; i < bs; i += NT) {
			const int row = i / R_T, col = i - row * R_T;
			p0[row * 36 + col] = __ldg(g + (size_t)i * nch + sidx0) >> w0;
			p1[row * 36 + col] = have1 ? (__ldg(g + (size_t)i * nch + sidx1) >> w1) : 0;
		}
	}
	else {
	__syncthreads();  // mbarrier init visible to every waiter
	mbar_wait(mbar, 0);
	{
		int4 rv[R_T / 4];
#pragma unroll
		for(int k = 0; k < R_T / 4; k++) rv[k] = *reinterpret_cast<const int4 *>(raw + 4 * (k * NT + tid));
		__syncthreads();
		int32_t *const p0 = planar + kSearch4ZeroRow;
		int32_t *const p1 = planar + planar_words + kSearch4ZeroRow;
		for(int i = tid; i < kSearch4ZeroRow; i += NT) { planar[i] = 0; if(CH == 2) planar[planar_words + i] = 0; }  // history of row 0
		if(CH == 2) {
			// signal = (a L + b R) >> sh: L (1,0), R (0,1), mid (1,1) >> 1, side (1,-1) (stream_encoder.c:3823-3836); the wasted-bits
			// shift (:3842-3867) folds into sh
			const int a0c = sidx0 != 1, b0c = sidx0 == 0 ? 0 : sidx0 == 3 ? -1 : 1, sh0 = __ldg(&bp[sidx0].wasted) + (sidx0 == 2);
			const int a1c = sidx1 != 1, b1c = sidx1 == 0 ? 0 : sidx1 == 3 ? -1 : 1, sh1 = __ldg(&bp[sidx1].wasted) + (sidx1 == 2);
#pragma unroll
			for(int k = 0; k < R_T / 4; k++) {
				const int i = 2 * (k * NT + tid);  // first of the two sample pairs in this vector
				const int row = i / R_T, col = i - row * R_T;
				*reinterpret_cast<int2 *>(p0 + row * 36 + col) = make_int2((a0c * rv[k].x + b0c * rv[k].y) >> sh0, (a0c * rv[k].z + b0c * rv[k].w) >> sh0);
				*reinterpret_cast<int2 *>(p1 + row * 36 + col) = make_int2((a1c * rv[k].x + b1c * rv[k].y) >> sh1, (a1c * rv[k].z + b1c * rv[k].w) >> sh1);
			}
		}
		else {
#pragma unroll
			for(int k = 0; k < R_T / 4; k++) {
				const int i = 4 * (k * NT + tid);
				const int row = i / R_T, col = i - row * R_T;
				*reinterpret_cast<int4 *>(p0 + row * 36 + col) = make_int4(rv[k].x >> wasted, rv[k].y >> wasted, rv[k].z >> wasted, rv[k].w >> wasted);
			}
		}
	}
	}  // !PAIR
	__syncthreads();

	// ---- pass 1: residual -> zig-zag (in place) -> bit count of this run
	int32_t *const xs = planar + myc * planar_words + kSearch4ZeroRow;
	int32_t *const rowp = xs + run * 36;
	const int base = run * R_T;  // first sample of the run
	const bool predicted = type == SF_FIXED || type == SF_LPC;
	const int psize = bs >> po;
	const uint32_t plen = method ? kRice2ParamLen : kRiceParamLen;
	const bool one_partition = (psize % R_T) == 0;
	uint32_t mybits = 0;
	uint32_t k_run = 0;
	if(run < FB200_MAX_LPC_ORDER) S.warm[myc][run] = xs[run];  // warm-up samples (all inside row 0: order <= 32 <= R_T)
	if(predicted) {
		int xg[MAXORD + G];
		// history: the MAXORD samples before the run (previous row, or the zero row for run 0); loaded before ANY thread
		// overwrites its row with zig-zagged residuals
#pragma unroll
		for(int k = 0; k < MAXORD / 4; k++) {
			const int4 v = *reinterpret_cast<const int4 *>(rowp - MAXORD + 4 * k - ROWPAD);
			xg[4 * k] = v.x; xg[4 * k + 1] = v.y; xg[4 * k + 2] = v.z; xg[4 * k + 3] = v.w;
		}
		__syncthreads();
		int q[MAXORD];
		if(type == SF_FIXED) {
#pragma unroll
			for(int j = 0; j < MAXORD; j++) q[j] = fixed_tap(order, j);
		}
		else {
#pragma unroll
			for(int j = 0; j < MAXORD; j++) q[j] = __ldg(&pl->qlp[j]);
		}
		const int qshift = type == SF_FIXED ? 0 : shift;
		constexpr int NT12 = MAXORD < 12 ? MAXORD : 12;
		const int cls = (WIDEK && wide) ? (order <= 8 ? 4 : 5) : (order <= 4 ? 0 : order <= 8 ? 1 : (MAXORD > 8 && order <= 12) ? 2 : 3);
		int p = base / psize;
		int next = (p + 1) * psize;
		uint32_t k = __ldg(&pl->params[p]);
		k_run = k;
		uint32_t qsum = 0, ncoded = 0;
#pragma unroll 1
		for(int g = 0; g < NG; g++) {
#pragma unroll
			for(int kk = 0; kk < G / 4; kk++) {
				const int4 v = *reinterpret_cast<const int4 *>(rowp + g * G + 4 * kk);
				xg[MAXORD + 4 * kk] = v.x; xg[MAXORD + 4 * kk + 1] = v.y; xg[MAXORD + 4 * kk + 2] = v.z; xg[MAXORD + 4 * kk + 3] = v.w;
			}
			int r[G];
			switch(cls) {
				case 0: group_residual_narrow<G, MAXORD, 4>(xg, q, qshift, r); break;
				case 1: group_residual_narrow<G, MAXORD, 8>(xg, q, qshift, r); break;
				case 2: group_residual_narrow<G, MAXORD, NT12>(xg, q, qshift, r); break;
				case 3: group_residual_narrow<G, MAXORD, MAXORD>(xg, q, qshift, r); break;
				case 4: if(WIDEK) group_residual_wide<G, MAXORD, 8>(xg, q, qshift, r); break;
				default: if(WIDEK) group_residual_wide<G, MAXORD, MAXORD>(xg, q, qshift, r); break;
			}
			uint32_t u[G];
#pragma unroll
			for(int m = 0; m < G; m++) u[m] = ((uint32_t)r[m] << 1) ^ (uint32_t)(r[m] >> 31);
#pragma unroll
			for(int kk = 0; kk < G / 4; kk++)
				*reinterpret_cast<uint4 *>(rowp + g * G + 4 * kk) = make_uint4(u[4 * kk], u[4 * kk + 1], u[4 * kk + 2], u[4 * kk + 3]);
			if(one_partition) {
				if(base + g * G >= order) {
#pragma unroll
					for(int m = 0; m < G; m++) qsum += u[m] >> k;
					ncoded += G;
				}
				else {
#pragma unroll
					for(int m = 0; m < G; m++)
						if(base + g * G + m >= order) { qsum += u[m] >> k; ncoded++; }
				}
			}
			else {
#pragma unroll
				for(int m = 0; m < G; m++) {
					const int i = base + g * G + m;
					if(i >= order) {
						if(i == next) { p++; next += psize; k = __ldg(&pl->params[p]); }
						if(i == p * psize || i == order) mybits += plen;
						mybits += (u[m] >> k) + 1 + k;
					}
				}
			}
			// rotate: the last MAXORD samples just consumed become the history of the next group
#pragma unroll
			for(int j = 0; j < MAXORD; j++) xg[j] = xg[j + G];
		}
		if(one_partition) {
			const int first_res = p == 0 ? order : p * psize;
			mybits = qsum + ncoded * (k + 1) + ((first_res >= base && first_res < base + R_T) ? plen : 0u);
		}
	}
	else {
		__syncthreads();  // matches the barrier of the predicted branch (the type is per channel, barriers are per CTA)
		if(type == SF_VERBATIM) mybits = (uint32_t)R_T * (uint32_t)sbps;
	}
	// bits in front of the first run of a channel: subframe header, warm-up, coefficients, entropy header
	uint32_t pre = 0;
	if(run == 0 && !absent) {
		pre = kSubframeHeaderBits + (uint32_t)wasted;
		if(type == SF_CONSTANT) pre += (uint32_t)sbps;
		else if(predicted) {
			pre += (uint32_t)order * (uint32_t)sbps + kEntropyTypeLen + kRiceOrderLen;
			if(type == SF_LPC) pre += kQlpPrecisionLen + kQlpShiftLen + (uint32_t)order * (uint32_t)precision;
		}
	}

	// ---- ONE exclusive scan over all runs of the frame (channel 0's runs, then channel 1's)
	uint32_t start, total;
	{
		const uint32_t v = mybits + pre;
		uint32_t inc = v;
#pragma unroll
		for(int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
			if(lane >= o) inc += t;
		}
		if(lane == 31) S.scan[warp] = inc;
		__syncthreads();
		const int nw = NT >> 5;
		uint32_t wbase = 0, tot = 0;
		for(int w = 0; w < nw; w++) {
			const uint32_t s = S.scan[w];
			if(w < warp) wbase += s;
			tot += s;
		}
		start = header_bits + wbase + inc - v;  // first bit of `pre` (run 0) or of the run's residual codes
		total = header_bits + tot;
	}
	const uint32_t nbytes = (total + 7) >> 3;      // frame bytes without the CRC-16
	const uint32_t s0 = PAIR ? 0u : (4u - (nbytes & 3u)) & 3u;  // leading pad bytes: the frame's END is word aligned in `words`
	const uint32_t bit0 = s0 * 8;
	const uint32_t wend = (s0 + nbytes) >> 2;       // word index of the CRC-16
	const bool fits = (int)wend + 2 <= zero_words;  // always, by the estimate's construction; fail loudly otherwise
	// publish this frame's size for the frames behind it
	if(tid == 0) {
		if(!PAIR) st_volatile_u64(&A.lookback[blk], lb_pack(nbytes + 2, A.epoch, 1));
		if(!fits) atomicExch(A.err, 2);
	}

	// ---- pass 2: pack. Before the barrier: plain stores only (a word is stored by the run that reaches its last bit); after
	// it: every run's trailing partial word, the frame header and the subframe header fields are OR-ed in.
	int last_word = 0;
	uint32_t last_bits = 0;
	if(fits) {
		// residual codes of this run (stream_encoder_framing.c:538-594, bitwriter.c:575-706)
		if(predicted) {
			if(one_partition) {
				// ONE partition per run: zeros + stop bit + k low bits go out as one field of n = q + k + 1 bits; the pending word
				// `cur` (fill bits used) is stored when it completes. Every run -- the one with the warm-up samples included --
				// runs this same loop (skipn leading samples are not residuals), so the warps of a frame finish together.
				const uint32_t k = k_run, k1 = k + 1;
				const uint32_t stop = 1u << k, lowmask = stop - 1u;
				const uint32_t pos0 = bit0 + start + pre;
				int widx = (int)(pos0 >> 5);
				uint32_t fill = pos0 & 31u, cur = 0;
				auto put = [&](uint32_t val, uint32_t n) {  // 0 <= n <= 32, val < 2^n; branch-free: the store is predicated
					const unsigned long long t = (unsigned long long)val << (64u - fill - n);
					cur |= (uint32_t)(t >> 32);
					const uint32_t f2 = fill + n;
					const bool full = f2 >= 32u;
					if(full) words[widx] = cur;
					cur = full ? (uint32_t)t : cur;
					widx += (int)(f2 >> 5);
					fill = f2 & 31u;
				};
				const int pidx = base / psize;
				const int skipn = order > base ? order - base : 0;                       // leading warm-up samples of this run
				const int prel = (pidx == 0 ? order : pidx * psize) - base;               // the partition's first residual, relative to the run
				// partitions are whole runs here: the parameter, if this run carries one, sits in front of its first coded sample
				if(prel == skipn && skipn < R_T) put(k, plen);
				auto pack_run = [&](auto skip_tag) {
					constexpr bool SKIP = decltype(skip_tag)::value;  // only the run that holds the warm-up samples tests for them
#pragma unroll 1
					for(int v4 = 0; v4 < R_T / 4; v4++) {
						const uint4 uv = *reinterpret_cast<const uint4 *>(rowp + 4 * v4);
#pragma unroll
						for(int e = 0; e < 4; e++) {
							const int m = 4 * v4 + e;
							if(SKIP && m < skipn) continue;
							const uint32_t u = e == 0 ? uv.x : e == 1 ? uv.y : e == 2 ? uv.z : uv.w;
							const uint32_t qz = u >> k;
							const uint32_t val = stop | (u & lowmask);
							if(qz + k1 <= 32u) put(val, qz + k1);
							else {
								// a long unary run (rare): zeros word by word, then the stop bit + low bits
								uint32_t z = qz;
								while(z) { const uint32_t c = z < 32u - fill ? z : 32u - fill; put(0u, c); z -= c; }
								put(val, k1);
							}
						}
					}
				};
				if(skipn) pack_run(std::true_type{});
				else pack_run(std::false_type{});
				last_word = widx; last_bits = cur;
			}
			else {
				// partitions shorter than a run (partition orders above log2(bs / R_T)): the parameter changes inside the run
				RunPacker pk;
				pk.init(words, bit0 + start + pre);
				int p = base / psize;
				int next = (p + 1) * psize;
				uint32_t k = __ldg(&pl->params[p]);
#pragma unroll 1
				for(int m = 0; m < R_T; m++) {
					const int i = base + m;
					if(i >= order) {
						if(i == next) { p++; next += psize; k = __ldg(&pl->params[p]); }
						if(i == p * psize || i == order) pk.put(k, plen);
						const uint32_t u = (uint32_t)rowp[m];
						pk.skip(u >> k);
						pk.put((1u << k) | (u & ((1u << k) - 1u)), k + 1);
					}
				}
				last_word = pk.widx; last_bits = pk.cur;
			}
		}
		else if(type == SF_VERBATIM) {
			RunPacker pk;
			pk.init(words, bit0 + start + pre);
#pragma unroll 1
			for(int m = 0; m < R_T; m++) pk.put(mask_bits(rowp[m], (uint32_t)sbps), (uint32_t)sbps);
			last_word = pk.widx; last_bits = pk.cur;
		}
	}
	__syncthreads();
	if(fits) {
		if(last_bits) atomicOr(&words[last_word], last_bits);
		if(!PAIR && warp == (NT >> 5) - 1 && lane < 5) {
			// place the pre-built frame header at byte s0 (S.hdr was written before the barriers above)
			const uint32_t sh = 8 * s0;
			const uint32_t hi = lane > 0 ? S.hdr[lane - 1] : 0u, lo = lane < 4 ? S.hdr[lane] : 0u;
			const uint32_t w = sh ? __funnelshift_r(lo, hi, sh) : lo;  // the header bytes shifted right by s0 bytes
			if(w) atomicOr(&words[lane], w);
		}
		// subframe header fields (stream_encoder_framing.c:393-520): one field per thread, spread over the CTA so that no warp
		// carries the whole header on top of its runs. Slots per channel: 0 type byte + wasted-bits unary (+ the constant),
		// 1 precision + shift, 2 entropy method + partition order, 3.. warm-up samples, 35.. coefficients.
		for(int g = tid; g < 72 * CH; g += NT) {
			const int c = g / 72, slot = g - c * 72;
			if(c == 1 && !have1) continue;
			const SubframePlan *pc = bp + (c ? sidx1 : sidx0);
			const int ftype = __ldg(&pc->type), forder = __ldg(&pc->order), fwasted = __ldg(&pc->wasted), fsbps = __ldg(&pc->bps);
			const bool fpred = ftype == SF_FIXED || ftype == SF_LPC;
			// first bit of the subframe: the exclusive prefix of its first run = the totals of the warps in front of it
			uint32_t sf0 = bit0 + header_bits;
			for(int w = 0; w < c * (TPC >> 5); w++) sf0 += S.scan[w];
			const uint32_t warm0 = sf0 + kSubframeHeaderBits + (uint32_t)fwasted;
			const uint32_t after_warm = warm0 + (uint32_t)forder * (uint32_t)fsbps;
			BitPut bw;
			if(slot == 0) {
				uint32_t tb;
				switch(ftype) {
					case SF_CONSTANT: tb = 0x00; break;
					case SF_VERBATIM: tb = 0x02; break;
					case SF_FIXED: tb = 0x10 | ((uint32_t)forder << 1); break;
					default: tb = 0x40 | ((uint32_t)(forder - 1) << 1); break;
				}
				bw.init(words, sf0);
				bw.put(tb | (fwasted ? 1u : 0u), 8);
				if(fwasted) { bw.skip((uint32_t)fwasted - 1); bw.put(1, 1); }
				if(ftype == SF_CONSTANT) bw.put(mask_bits(S.warm[c][0], (uint32_t)fsbps), (uint32_t)fsbps);
				bw.finish();
			}
			else if(slot == 1) {
				if(ftype == SF_LPC) {
					bw.init(words, after_warm);
					bw.put((uint32_t)__ldg(&pc->precision) - 1, kQlpPrecisionLen);
					bw.put(mask_bits(__ldg(&pc->shift), kQlpShiftLen), kQlpShiftLen);
					bw.finish();
				}
			}
			else if(slot == 2) {
				if(fpred) {
					const uint32_t fprec = (uint32_t)__ldg(&pc->precision);
					bw.init(words, after_warm + (ftype == SF_LPC ? kQlpPrecisionLen + kQlpShiftLen + (uint32_t)forder * fprec : 0u));
					bw.put((uint32_t)__ldg(&pc->method), kEntropyTypeLen);
					bw.put((uint32_t)__ldg(&pc->porder), kRiceOrderLen);
					bw.finish();
				}
			}
			else if(slot < 3 + FB200_MAX_LPC_ORDER) {
				const int i = slot - 3;
				if(fpred && i < forder) {
					bw.init(words, warm0 + (uint32_t)i * (uint32_t)fsbps);
					bw.put(mask_bits(S.warm[c][i], (uint32_t)fsbps), (uint32_t)fsbps);
					bw.finish();
				}
			}
			else {
				const int i = slot - 3 - FB200_MAX_LPC_ORDER;
				if(ftype == SF_LPC && i < forder) {
					const uint32_t fprec = (uint32_t)__ldg(&pc->precision);
					bw.init(words, after_warm + kQlpPrecisionLen + kQlpShiftLen + (uint32_t)i * fprec);
					bw.put(mask_bits(__ldg(&pc->qlp[i]), fprec), fprec);
					bw.finish();
				}
			}
		}
	}

	if(PAIR) {
		// the pair's bits, from bit 0, go to its staging region; k_join splices the regions of a frame
		__syncthreads();
		const size_t region = (size_t)blk * npairs + pair;
		uint32_t *dst = A.stage + region * (size_t)A.pair_words;
		const uint32_t nw = fits ? (total + 31u) >> 5 : 0u;
		for(uint32_t i = tid; i < nw; i += NT) dst[i] = words[i];
		if(tid == 0) A.stage_bits[region] = fits ? total : 0xffffffffu;
		return;
	}
	emit3_finish(A, S, words, crc_tab, blk, ca, nbytes, s0, wend, fits);
}

// ================================================================ k_join
// Streams of more than two channels: one CTA per frame splices the channel pairs that k_emit3<PAIR> packed (each from bit 0 of
// its staging region) behind the frame header -- a funnel-shift copy into shared memory, laid out so that the frame's END is
// word aligned -- and finishes the frame like k_emit3: CRC-16, look-back offset, copy to its place in the stream.
__host__ __device__ inline size_t join_smem_bytes(int join_words)
{
	return (sizeof(Emit3Shared) + 15) / 16 * 16 + 3328 + (size_t)(join_words + 8) * 4;
}

__global__ void __launch_bounds__(256, 2) k_join(EncK P, Emit3Args A)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int tid = threadIdx.x, NT = blockDim.x, lane = tid & 31, warp = tid >> 5;
	Emit3Shared &S = *reinterpret_cast<Emit3Shared *>(smem_raw);
	uint16_t *const crc_tab = reinterpret_cast<uint16_t *>(smem_raw + (sizeof(Emit3Shared) + 15) / 16 * 16);
	uint32_t *const words = reinterpret_cast<uint32_t *>(reinterpret_cast<unsigned char *>(crc_tab) + 3328);
	const int words_cap = A.join_words + 8;

	if(tid == 0) S.blk = (int)(atomicAdd(A.ticket, 1u) - A.ticket_base);
	__syncthreads();
	const int blk = S.blk;
	const int npairs = (P.channels + 1) >> 1;  // <= 4
	const uint32_t header_bits = emit3_frame_header(P, blk, 0, warp == (NT >> 5) - 1, lane, S.hdr);

	uint32_t pb[4] = {0, 0, 0, 0};
	bool ok = true;
	uint32_t total = header_bits;
#pragma unroll
	for(int p = 0; p < 4; p++)
		if(p < npairs) {
			pb[p] = __ldg(&A.stage_bits[(size_t)blk * npairs + p]);
			if(pb[p] == 0xffffffffu) { ok = false; pb[p] = 0; }
			total += pb[p];
		}
	const uint32_t nbytes = (total + 7) >> 3;      // frame bytes without the CRC-16
	const uint32_t s0 = (4u - (nbytes & 3u)) & 3u;  // leading pad bytes: the frame's END is word aligned in `words`
	const uint32_t bit0 = s0 * 8;
	const uint32_t wend = (s0 + nbytes) >> 2;       // word index of the CRC-16
	const bool fits = ok && (int)wend + 2 <= words_cap;
	if(tid == 0) {
		st_volatile_u64(&A.lookback[blk], lb_pack(nbytes + 2, A.epoch, 1));
		if(!fits) atomicExch(A.err, 2);
	}
	if(fits) {
		for(uint32_t i = tid; i < wend + 2; i += NT) words[i] = 0;
		__syncthreads();
		if(warp == (NT >> 5) - 1 && lane < 5) {
			const uint32_t sh = 8 * s0;
			const uint32_t hi = lane > 0 ? S.hdr[lane - 1] : 0u, lo = lane < 4 ? S.hdr[lane] : 0u;
			const uint32_t w = sh ? __funnelshift_r(lo, hi, sh) : lo;  // the header bytes shifted right by s0 bytes
			if(w) atomicOr(&words[lane], w);
		}
		uint32_t D = bit0 + header_bits;  // destination bit of the current pair
#pragma unroll
		for(int p = 0; p < 4; p++)
			if(p < npairs) {
				const uint32_t *src = A.stage + ((size_t)blk * npairs + p) * (size_t)A.pair_words;
				const uint32_t sh = D & 31u, w0 = D >> 5;
				const uint32_t nsrc = (pb[p] + 31u) >> 5, nd = (sh + pb[p] + 31u) >> 5;
				// destination word w0 + t = source words t-1, t shifted right by sh bits; the first and the last one are shared with
				// the neighbours (header / other pairs): OR; the words in between belong to this pair alone: plain stores
				for(uint32_t t = tid; t < nd; t += NT) {
					const uint32_t a = t < nsrc ? __ldg(src + t) : 0u, b = (t >= 1 && t - 1 < nsrc) ? __ldg(src + t - 1) : 0u;
					const uint32_t v = __funnelshift_r(a, b, sh);
					if(t == 0 || t + 1 == nd) { if(v) atomicOr(&words[w0 + t], v); }
					else words[w0 + t] = v;
				}
				D += pb[p];
			}
	}
	__syncthreads();
	emit3_finish(A, S, words, crc_tab, blk, 0, nbytes, s0, wend, fits);
}

}  // namespace fb200
