// replaygain_synthesis.cu -- flac -d --apply-replaygain-which-is-not-lossless: the option's parse (main.c:767-790), the decision
// per file (decode.c:1775-1820, grabbag/replaygain.c:582-669) and FLAC__replaygain_synthesis__apply_gain
// (src/share/replaygain_synthesis/replaygain_synthesis.c) over every container of a fb200_decode_pcm_files_replaygain_* call in one
// launch. The decode, the plan and k_pcm_pack are decoder.cu's.
#include <locale.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "fb200_internal.h"
#include "flac_metadata.h"
#include "flac_parse.h"
#include "glibc_tanh.cuh"

namespace fb200 {

// ---------------------------------------------------------------- the dither generator (random_int_)
// Two 32-bit registers, both linear over GF(2): r1 shifts right and takes parity(r1 & 0xF5) into bit 31, r2 shifts left and takes
// parity((r2 >> 25) & 0x63) into bit 0; a draw steps both and returns r1 ^ r2. Both start at 1 when the process starts. The state
// after D draws is M1^D * 1 and M2^D * 1: c_rgs_jump[r][k] holds the rows of Mr^(2^k), so any D costs at most 64 products of a
// 32 x 32 bit matrix and a vector (32 popc each).
__constant__ uint32_t c_rgs_jump[2][64][32];

static const std::vector<uint32_t> &rgs_jump_table()
{
	static std::vector<uint32_t> tab;
	static std::once_flag once;
	std::call_once(once, [] {
		tab.assign(2 * 64 * 32, 0);
		uint32_t m[2][32];
		for(int i = 0; i < 32; i++) {
			m[0][i] = i < 31 ? 1u << (i + 1) : 0xF5u;
			m[1][i] = i > 0 ? 1u << (i - 1) : 0x63u << 25;
		}
		for(int r = 0; r < 2; r++)
			for(int k = 0; k < 64; k++) {
				memcpy(&tab[(r * 64 + k) * 32], m[r], sizeof m[r]);
				uint32_t sq[32];  // row i of A * A: the XOR of the rows of A that row i of A selects
				for(int i = 0; i < 32; i++) {
					uint32_t v = 0;
					for(int j = 0; j < 32; j++)
						if(m[r][i] >> j & 1) v ^= m[r][j];
					sq[i] = v;
				}
				memcpy(m[r], sq, sizeof sq);
			}
	});
	return tab;
}

static int rgs_upload_jump(cudaStream_t st)
{
	const std::vector<uint32_t> &t = rgs_jump_table();
	FB_CUDA(cudaMemcpyToSymbolAsync(c_rgs_jump, t.data(), t.size() * sizeof(uint32_t), 0, cudaMemcpyHostToDevice, st));
	return FB200_OK;
}

struct RgsGen { uint32_t r1, r2; };

// the state 2^k draws after g
__device__ __forceinline__ RgsGen rgs_mul(int k, RgsGen g)
{
	uint32_t a = 0, b = 0;
#pragma unroll 8
	for(int i = 0; i < 32; i++) {
		a |= (uint32_t)(__popc(c_rgs_jump[0][k][i] & g.r1) & 1) << i;
		b |= (uint32_t)(__popc(c_rgs_jump[1][k][i] & g.r2) & 1) << i;
	}
	return RgsGen{a, b};
}

// the state after d draws from the process's start
__device__ __noinline__ RgsGen rgs_jump(unsigned long long d)
{
	RgsGen g{1u, 1u};
	for(int k = 0; d; k++, d >>= 1)
		if(d & 1) g = rgs_mul(k, g);
	return g;
}

__device__ __forceinline__ int32_t rgs_draw(RgsGen &g)
{
	g.r1 = (g.r1 >> 1) | (uint32_t)(__popc(g.r1 & 0xF5u) & 1) << 31;
	g.r2 = (g.r2 << 1) | (uint32_t)(__popc((g.r2 >> 25) & 0x63u) & 1);
	return (int32_t)(g.r1 ^ g.r2);
}

// ---------------------------------------------------------------- apply_gain, value by value

// F44_1 .. F44_3 (the 48-entry tables are three copies of these 16), as the (float) casts of the reference's literals round them
__constant__ float c_rgs_coef[3][16] = {
	{0x1.b34b2ep-1f, 0x1.29e0a2p-2f, -0x1.9b642ap-5f, -0x1.e236p-3f, -0x1.2ad132p-1f, -0x1.573d54p-1f, -0x1.8aecb6p-2f, -0x1.37adap-3f,
	 -0x1.a64dfep-6f, 0x1.2129c6p-3f, 0x1.caba7ap-3f, 0x1.3b6d68p-3f, 0x1.ab4ed4p-5f, -0x1.71ef4cp-9f, -0x1.f2880ep-6f, -0x1.fd81aap-6f},
	{0x1.c9cc74p+0f, 0x1.e90086p-1f, -0x1.79ceb2p-3f, -0x1.c496bcp-2f, -0x1.c4a0f6p-1f, -0x1.6c1496p+0f, -0x1.053756p+0f, -0x1.64fcp-2f,
	 -0x1.d6a3ccp-4f, 0x1.fff476p-4f, 0x1.85cb7p-2f, 0x1.467ca8p-2f, 0x1.ad8a7ap-4f, -0x1.fcc85p-6f, -0x1.0836a8p-4f, -0x1.e18eeap-6f},
	{0x1.720328p+1f, 0x1.583be8p+1f, 0x1.afc986p-3f, -0x1.f7bb48p-1f, -0x1.1c484ep+0f, -0x1.1842ep+1f, -0x1.2eb7acp+1f, -0x1.e8e0f6p-1f,
	 -0x1.e9f6f6p-3f, -0x1.1bf5c4p-3f, 0x1.be56eap-2f, 0x1.516cb8p-1f, 0x1.f2ee14p-3f, -0x1.354c0ep-9f, 0x1.2e25f4p-6f, 0x1.1a4998p-6f}};

// (double)x * multi_scale, the hard 6 dB limiter, * 2147483647. (apply_gain :372-381). x / (1 - 0.5) is x * 2, exactly.
__device__ __noinline__ double rgs_limit(double s)
{
	if(s < -0.5) return __dsub_rn(__dmul_rn(fb_tanh(__dmul_rn(__dadd_rn(s, 0.5), 2.0)), 0.5), 0.5);
	return __dadd_rn(__dmul_rn(fb_tanh(__dmul_rn(__dsub_rn(s, 0.5), 2.0)), 0.5), 0.5);
}

__device__ __forceinline__ double rgs_sample(int32_t x, const RgsParam &P)
{
	double s = __dmul_rn((double)x, P.multi);
	if(P.hard && (s < -0.5 || s > 0.5)) s = rgs_limit(s);
	return __dmul_rn(s, 2147483647.);
}

// ROUND64: the magic-constant add, then the bits
__device__ __forceinline__ long long rgs_round64(double x, double add)
{
	return __double_as_longlong(__dadd_rn(__dadd_rn(x, add), (double)0x001FFFFD80000000ll)) - 0x433FFFFD80000000ll;
}

// >> conv_shift and the clip to the target width (:383-389)
__device__ __forceinline__ int32_t rgs_finish(long long v, const RgsParam &P)
{
	const long long val64 = v >> P.conv_shift;
	if(val64 >= -P.clip) return (int32_t)(-(P.clip + 1));
	if(val64 < P.clip) return (int32_t)P.clip;
	return (int32_t)val64;
}

// No shaping (no dither): every value on its own. One CTA per kRgsItem values of one segment.
constexpr int kRgsItem = 1024;

__global__ void __launch_bounds__(256) k_rg_synth0(int32_t *__restrict__ pcm, const RgsSeg *__restrict__ segs, int nsegs)
{
	const unsigned long long item = blockIdx.x;
	int lo = 0, hi = nsegs - 1;
	while(lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if(segs[mid].item0 <= item) lo = mid;
		else hi = mid - 1;
	}
	const RgsSeg S = segs[lo];
	for(int k = threadIdx.x; k < kRgsItem; k += 256) {
		const unsigned long long i = (item - S.item0) * kRgsItem + k;
		if(i >= S.n) break;
		int32_t *p = pcm + S.v0 + i;
		*p = rgs_finish(rgs_round64(rgs_sample(*p, S.P), S.P.add), S.P);
	}
}

// scalar16_(x, F + i): sixteen float products summed left to right in float; F + i reads coefficient (i + j) & 15
template <int SH, int I>
__device__ __forceinline__ float rgs_dot(const float (&h)[16])
{
	float acc = __fmul_rn(h[0], c_rgs_coef[SH - 1][I & 15]);
#pragma unroll
	for(int j = 1; j < 16; j++) acc = __fadd_rn(acc, __fmul_rn(h[j], c_rgs_coef[SH - 1][(I + j) & 15]));
	return acc;
}

// dither_output_ with shaping (:257-262) splits into two recurrences per (container, channel). The dither history depends only on
// the draws: d = (float)(tri - scalar16_(DitherHistory)), Sum = sample + d. The error feedback, through ROUND64 & Mask, is the
// non-linear one: val = ROUND64(Sum + scalar16_(ErrorHistory)) & Mask, ErrorHistory = (float)(Sum - val). I is the position from
// the container's start mod 32, which decides the history slot and the coefficient offset.
template <int SH, int I>
__device__ __forceinline__ double rgs_dither_step(double s, double tri, float (&dh)[16])
{
	const float d = (float)__dsub_rn(tri, (double)rgs_dot<SH, I>(dh));
	dh[(-1 - I) & 15] = d;
	return __dadd_rn(s, (double)d);
}

template <int SH, int I>
__device__ __forceinline__ long long rgs_error_step(double sum, float (&eh)[16], const RgsParam &P)
{
	const long long val = (long long)((unsigned long long)rgs_round64(__dadd_rn(sum, (double)rgs_dot<SH, I>(eh)), P.add) & P.mask);
	eh[(-1 - I) & 15] = (float)__dsub_rn(sum, (double)val);
	return val;
}

// Lane 0's part of a tile: the dither recurrence of tile k + 1 (tri, s -> sum) interleaved with the error recurrence of tile k
// (sum -> val32); the two are independent, so their latencies overlap.
template <int I, int SH>
struct RgsSerial {
	__device__ __forceinline__ static void run(const double *__restrict__ s1, const double *__restrict__ t1, double *__restrict__ u1,
	                                           const double *__restrict__ u0, int32_t *__restrict__ o, float (&dh)[16], float (&eh)[16], const RgsParam &P)
	{
		u1[I] = rgs_dither_step<SH, I>(s1[I], t1[I], dh);
		o[I] = rgs_finish(rgs_error_step<SH, I>(u0[I], eh, P), P);
		RgsSerial<I + 1, SH>::run(s1, t1, u1, u0, o, dh, eh, P);
	}
};
template <int SH>
struct RgsSerial<32, SH> {
	__device__ __forceinline__ static void run(const double *, const double *, double *, const double *, int32_t *, float (&)[16], float (&)[16], const RgsParam &) {}
};

template <int I, int SH>
struct RgsDitherOnly {
	__device__ __forceinline__ static void run(const double *__restrict__ s1, const double *__restrict__ t1, double *__restrict__ u1, float (&dh)[16])
	{
		u1[I] = rgs_dither_step<SH, I>(s1[I], t1[I], dh);
		RgsDitherOnly<I + 1, SH>::run(s1, t1, u1, dh);
	}
};
template <int SH>
struct RgsDitherOnly<32, SH> {
	__device__ __forceinline__ static void run(const double *, const double *, double *, float (&)[16]) {}
};

// With shaping: one warp per (container, channel) chain, in tiles of 32 positions aligned to the container's start. For tile k + 1
// every lane takes one position: it gathers the input, scales it, runs the limiter (fb_tanh) and makes its two draws, keeping the
// generator state of its own position (one jump-ahead at the start and at each delivered block it enters, else 64 draws on per
// tile by one matrix product). Lane 0 then runs the only serial work: the dither recurrence of tile k + 1 and the error
// recurrence of tile k, interleaved, with both histories in registers (the unrolled loop makes every index static). The warp
// stores tile k's values in place. All staging is in shared memory, double-buffered by tile.
template <int SH>
__global__ void __launch_bounds__(32) k_rg_synth(int32_t *__restrict__ pcm, const RgsChain *__restrict__ chains, const RgsBlock *__restrict__ blocks)
{
	__shared__ double sh_s[2][32], sh_t[2][32], sh_u[2][32];
	__shared__ int32_t sh_o[32];
	const int lane = threadIdx.x;
	const RgsChain K = chains[blockIdx.x];
	int32_t *p = pcm + K.v0 + K.c;
	const unsigned long long ns = K.ns, ntiles = (ns + 31) / 32;
	const uint32_t jlast = K.b0 + K.nb - 1;
	// this lane's place in the blocks and its generator state at its position; bend = ~0: not yet placed
	uint32_t j = K.b0;
	unsigned long long bend = 0;
	RgsGen g{1u, 1u};
	auto pre = [&](unsigned long long tile, int buf) {
		const unsigned long long t = tile * 32 + lane;
		double s = 0.0, tri = 0.0;
		if(t < ns) {
			if(t >= bend) {
				RgsBlock B = blocks[j];
				while(t >= B.s + B.n && j < jlast) B = blocks[++j];
				bend = B.s + B.n;
				g = rgs_jump(K.draw0 + 2ull * (K.C * B.s + K.c * B.n + (t - B.s)));
			}
			s = rgs_sample(p[t * K.C], K.P);
			RgsGen h = g;
			const int32_t a = rgs_draw(h), b = rgs_draw(h);
			tri = __dmul_rn((double)K.P.dither, __dadd_rn((double)a, (double)b));
			if(t + 32 < bend) g = rgs_mul(6, g);  // 64 draws on: the same lane's position in the next tile
			else bend = t + 1;                     // the next tile's position lies in a later block: jump there
		}
		sh_s[buf][lane] = s;
		sh_t[buf][lane] = tri;
	};
	float dh[16], eh[16];
#pragma unroll
	for(int i = 0; i < 16; i++) dh[i] = eh[i] = 0.f;
	pre(0, 0);
	__syncwarp();
	if(lane == 0) RgsDitherOnly<0, SH>::run(sh_s[0], sh_t[0], sh_u[0], dh);
	__syncwarp();
	for(unsigned long long k = 0; k < ntiles; k++) {
		const int cur = (int)(k & 1), nxt = cur ^ 1;
		pre(k + 1, nxt);
		__syncwarp();
		if(lane == 0) RgsSerial<0, SH>::run(sh_s[nxt], sh_t[nxt], sh_u[nxt], sh_u[cur], sh_o, dh, eh, K.P);
		__syncwarp();
		const unsigned long long t = k * 32 + lane;
		if(t < ns) p[t * K.C] = sh_o[lane];
		__syncwarp();
	}
}

// Dither / Add / Mask from the stream's bits (init_dither_context, :203-225), conv_shift and the clip from the target width and
// multi_scale from both (apply_gain :338-346)
RgsParam rgs_param(uint32_t bps, double scale, bool hard, uint32_t shaping)
{
	static const uint8_t kDefaultDither[] = {92, 92, 88, 84, 81, 78, 74, 67, 0, 0};
	const uint32_t target = 8 * ((bps + 7) / 8);
	int indx = (int)bps - 11 - (int)shaping;
	if(indx < 0) indx = 0;
	if(indx > 9) indx = 9;
	RgsParam P;
	memset(&P, 0, sizeof P);
	P.multi = scale / (double)(1u << (bps - 1));
	P.add = 0.5 * (double)((1ll << (32 - bps)) - 1);
	P.mask = ~0ull << (32 - bps);
	const float d = 0.01f * (float)kDefaultDither[indx];
	P.dither = d / (float)(1ll << bps);
	P.conv_shift = (int)(32 - target);
	P.clip = -(1ll << (target - 1));
	P.hard = hard ? 1 : 0;
	return P;
}

int rgs_run(const RgsPlan &plan, uint32_t shaping, int32_t *pcm, cudaStream_t st, uint8_t **work, size_t *work_cap, uint64_t *launches)
{
	const size_t o_segs = 0;
	const size_t o_chains = (o_segs + plan.segs.size() * sizeof(RgsSeg) + 15) & ~(size_t)15;
	const size_t o_blocks = (o_chains + plan.chains.size() * sizeof(RgsChain) + 15) & ~(size_t)15;
	const size_t need = o_blocks + plan.blocks.size() * sizeof(RgsBlock) + 16;
	if(plan.segs.empty() && plan.chains.empty()) return FB200_OK;
	if(need > *work_cap) {
		cudaFree(*work);
		*work = nullptr;
		*work_cap = 0;
		FB_CUDA(cudaMalloc(work, need));
		*work_cap = need;
	}
	uint8_t *w = *work;
	if(!plan.segs.empty()) {
		FB_CUDA(cudaMemcpyAsync(w + o_segs, plan.segs.data(), plan.segs.size() * sizeof(RgsSeg), cudaMemcpyHostToDevice, st));
		const RgsSeg &last = plan.segs.back();
		const unsigned long long items = last.item0 + (last.n + kRgsItem - 1) / kRgsItem;
		k_rg_synth0<<<(unsigned)items, 256, 0, st>>>(pcm, reinterpret_cast<const RgsSeg *>(w + o_segs), (int)plan.segs.size());
		++*launches;
	}
	if(!plan.chains.empty()) {
		int rc;
		if((rc = rgs_upload_jump(st)) != FB200_OK) return rc;
		FB_CUDA(cudaMemcpyAsync(w + o_chains, plan.chains.data(), plan.chains.size() * sizeof(RgsChain), cudaMemcpyHostToDevice, st));
		FB_CUDA(cudaMemcpyAsync(w + o_blocks, plan.blocks.data(), plan.blocks.size() * sizeof(RgsBlock), cudaMemcpyHostToDevice, st));
		const unsigned grid = (unsigned)plan.chains.size();  // one warp per chain
		const RgsChain *c = reinterpret_cast<const RgsChain *>(w + o_chains);
		const RgsBlock *b = reinterpret_cast<const RgsBlock *>(w + o_blocks);
		if(shaping == 1) k_rg_synth<1><<<grid, 32, 0, st>>>(pcm, c, b);
		else if(shaping == 2) k_rg_synth<2><<<grid, 32, 0, st>>>(pcm, c, b);
		else k_rg_synth<3><<<grid, 32, 0, st>>>(pcm, c, b);
		++*launches;
	}
	FB_CUDA(cudaGetLastError());
	return FB200_OK;
}

// ---------------------------------------------------------------- the decision per file (host)

namespace {

// parse_double_: strtod (C locale) over the value's first min(31, length - 1) characters, as safe_strncpy copies them
bool rgs_parse_double(const std::string &entry, double *val)
{
	static const locale_t c_locale = newlocale(LC_ALL_MASK, "C", (locale_t)0);
	const size_t eq = entry.find('=');
	if(eq == std::string::npos) return false;
	const size_t vlen = entry.size() - (eq + 1);
	char s[32];
	const size_t n = std::min<size_t>(sizeof s, vlen);
	if(n < 1) return false;
	strncpy(s, entry.c_str() + eq + 1, n - 1);
	s[n - 1] = 0;
	char *end;
	const double v = strtod_l(s, &end, c_locale);
	if(end == s) return false;
	*val = v;
	return true;
}

// FLAC__metadata_object_vorbiscomment_find_entry_from(block, 0, name): the first entry whose name before its first '=' matches
int rgs_find(const std::vector<std::string> &ent, RgField field)
{
	for(size_t i = 0; i < ent.size(); i++)
		if(vorbis_entry_matches(ent[i].data(), ent[i].size(), kRgName[field])) return (int)i;
	return -1;
}

// grabbag__replaygain_load_from_vorbiscomment
bool rgs_load(const std::vector<std::string> &ent, bool album, bool strict, double *reference, double *gain, double *peak, bool *album_used)
{
	*reference = 89.0;
	int r = rgs_find(ent, RG_REFERENCE);
	if(r >= 0) (void)rgs_parse_double(ent[r], reference);
	bool res = true;
	const int g = rgs_find(ent, album ? RG_ALBUM_GAIN : RG_TRACK_GAIN);
	const int p = rgs_find(ent, album ? RG_ALBUM_PEAK : RG_TRACK_PEAK);
	if(g < 0 || p < 0) res = false;
	if(res && !rgs_parse_double(ent[g], gain)) res = false;
	if(res && !rgs_parse_double(ent[p], peak)) res = false;
	if(res && *peak < 0.0) res = false;
	*album_used = album;
	if(!res && !strict) res = rgs_load(ent, !album, true, reference, gain, peak, album_used);
	return res;
}

}  // namespace

// The metadata callback over every VORBIS_COMMENT block of the file (the last decides), for a stream of bps bits
void rgs_decide(const uint8_t *p, size_t n, uint32_t bps, const fb200_replaygain_synthesis &rg, fb200_replaygain_synthesis_info *I)
{
	memset(I, 0, sizeof *I);
	I->status = FB200_RGS_NO_TAGS;
	for_each_vorbis_comment(p, n, [&](const uint8_t *b, uint32_t len) {
		std::vector<std::string> ent;
		if(!read_metadata_vorbiscomment(b, len, &ent)) return;  // libFLAC fails the block: the callback never sees it
		double reference = 89.0, gain = 0.0, peak = 0.0;
		bool album_used = false;
		const bool ok = rgs_load(ent, rg.album != 0, false, &reference, &gain, &peak, &album_used);
		I->reference = reference; I->gain = gain; I->peak = peak; I->album_used = album_used; I->scale = 0.0;
		if(!ok) I->status = FB200_RGS_NO_TAGS;
		else if(bps < 4 || bps > 24) I->status = FB200_RGS_BPS;
		else if(gain > 90 || gain < -90) I->status = FB200_RGS_GAIN;
		else {
			// grabbag__replaygain_compute_scale_factor, with the host's pow
			double scale = (float)pow(10.0, (gain + rg.preamp) * 0.05);
			if(rg.limiter == FB200_RGS_LIMIT_PEAK && peak > 0.0) {
				const double max_scale = (float)(1.0 / peak);
				if(scale > max_scale) scale = max_scale;
			}
			I->scale = scale;
			I->status = FB200_RGS_APPLIED;
		}
	});
}

bool rgs_spec_ok(const fb200_replaygain_synthesis *rg)
{
	if(!rg) { set_error("the ReplayGain synthesis spec is NULL"); return false; }
	if(rg->limiter > FB200_RGS_LIMIT_HARD || rg->noise_shaping > 3 || rg->album > 1 || rg->per_file > 1) {
		set_error("limiter %u, noise_shaping %u, album %u or per_file %u out of range", rg->limiter, rg->noise_shaping, rg->album, rg->per_file);
		return false;
	}
	return true;
}

}  // namespace fb200

using namespace fb200;

extern "C" {

int fb200_replaygain_synthesis_parse(const char *spec, fb200_replaygain_synthesis *rg)
{
	if(!rg) return FB200_ERR_INVALID;
	fb200_replaygain_synthesis r;
	memset(&r, 0, sizeof r);
	r.album = 1;
	r.limiter = FB200_RGS_LIMIT_HARD;
	r.noise_shaping = 1;
	if(spec) {
		static const locale_t c_locale = newlocale(LC_ALL_MASK, "C", (locale_t)0);
		r.limiter = FB200_RGS_LIMIT_NONE;
		r.noise_shaping = 0;
		char *p;
		r.preamp = strtod_l(spec, &p, c_locale);
		for(; *p; p++) {
			if(*p == 'a') r.album = 1;
			else if(*p == 't') r.album = 0;
			else if(*p == 'l') r.limiter = FB200_RGS_LIMIT_PEAK;
			else if(*p == 'L') r.limiter = FB200_RGS_LIMIT_HARD;
			else if(*p == 'n' && p[1] >= '0' && p[1] <= '3') r.noise_shaping = (uint32_t)(*++p - '0');
			else { set_error("bad specification string \"%s\"", spec); return FB200_ERR_INVALID; }
		}
	}
	*rg = r;
	return FB200_OK;
}

int fb200_replaygain_synthesis_file(const uint8_t *file, uint64_t nbytes, const fb200_replaygain_synthesis *rg, fb200_replaygain_synthesis_info *info)
{
	if(!file || !info) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	if(!rgs_spec_ok(rg)) return FB200_ERR_INVALID;
	FLAC__StreamMetadata_StreamInfo si;
	memset(&si, 0, sizeof si);
	bool has_si = false;
	uint32_t si_len = 0;
	size_t audio = 0;
	if(!walk_metadata(file, (size_t)nbytes, si, &has_si, &si_len, &audio) || !has_si) {
		set_error("not a .flac file with STREAMINFO");
		return FB200_ERR_INVALID;
	}
	rgs_decide(file, (size_t)nbytes, si.bits_per_sample, *rg, info);
	return FB200_OK;
}

// tanh on the device vs the host's own (tests/test_gpu_decode_replaygain.py)
}  // extern "C"

namespace fb200 {
__global__ void k_debug_tanh(const double *x, double *y, unsigned n)
{
	const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) y[i] = fb_tanh(x[i]);
}
}  // namespace fb200

extern "C" {

int fb200_debug_tanh(const double *x, double *y, uint32_t n, int device)
{
	if((!x || !y) && n) return FB200_ERR_INVALID;
	if(n == 0) return FB200_OK;
	FB_CUDA(cudaSetDevice(device));
	double *dx = nullptr, *dy = nullptr;
	FB_CUDA(cudaMalloc(&dx, (size_t)n * sizeof(double)));
	FB_CUDA(cudaMalloc(&dy, (size_t)n * sizeof(double)));
	FB_CUDA(cudaMemcpy(dx, x, (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
	k_debug_tanh<<<(n + 255) / 256, 256>>>(dx, dy, n);
	FB_CUDA(cudaGetLastError());
	FB_CUDA(cudaMemcpy(y, dy, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
	cudaFree(dx);
	cudaFree(dy);
	return FB200_OK;
}

int fb200_debug_replaygain_synthesis(int device, const int32_t *in, uint32_t channels, uint64_t samples, const uint32_t *blocks, uint32_t nblocks,
                                     uint32_t bps, double scale, uint32_t hard_limit, uint32_t noise_shaping, uint64_t first_draw, int32_t *out)
{
	if(!in || !out || !blocks || nblocks == 0 || samples == 0) { set_error("a required pointer is NULL or the input is empty"); return FB200_ERR_INVALID; }
	if(channels < 1 || channels > 8 || bps < 4 || bps > 24 || noise_shaping > 3) {
		set_error("%u channels, %u bits, shaping %u, first draw %llu", channels, bps, noise_shaping, (unsigned long long)first_draw);
		return FB200_ERR_INVALID;
	}
	uint64_t sum = 0;
	for(uint32_t j = 0; j < nblocks; j++) {
		if(blocks[j] == 0) { set_error("block %u is empty", j); return FB200_ERR_INVALID; }
		sum += blocks[j];
	}
	if(sum != samples) { set_error("blocks sum to %llu, not %llu samples", (unsigned long long)sum, (unsigned long long)samples); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(device));
	const uint64_t nv = samples * channels;
	RgsPlan plan;
	const RgsParam P = rgs_param(bps, scale, hard_limit != 0, noise_shaping);
	if(noise_shaping == 0) plan.segs.push_back(RgsSeg{0, nv, 0, P});
	else {
		uint64_t s = 0;
		for(uint32_t j = 0; j < nblocks; j++) {
			plan.blocks.push_back(RgsBlock{s, blocks[j]});
			s += blocks[j];
		}
		for(uint32_t c = 0; c < channels; c++) plan.chains.push_back(RgsChain{0, samples, first_draw, channels, c, 0, nblocks, P});
	}
	int32_t *d = nullptr;
	FB_CUDA(cudaMalloc(&d, (size_t)nv * sizeof(int32_t)));
	uint8_t *work = nullptr;
	size_t cap = 0;
	uint64_t launches = 0;
	int rc = FB200_OK;
	if(cudaMemcpy(d, in, (size_t)nv * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) rc = FB200_ERR_CUDA;
	if(rc == FB200_OK) rc = rgs_run(plan, noise_shaping, d, nullptr, &work, &cap, &launches);
	if(rc == FB200_OK && cudaMemcpy(out, d, (size_t)nv * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess) rc = FB200_ERR_CUDA;
	if(rc == FB200_ERR_CUDA) set_error("fb200_debug_replaygain_synthesis: %s", cudaGetErrorString(cudaGetLastError()));
	cudaFree(d);
	cudaFree(work);
	return rc;
}

}  // extern "C"
