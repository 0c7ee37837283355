// hacktv_b200 - the fused line kernel (included by htv_kernels.cu).
//
// One persistent CTA walks a run of consecutive scan lines and does, per line, everything between
// the picture in HBM and the int16 IQ in HBM - raster, chroma, video filter, sound carriers, mixers -
// without the composite signal ever leaving the SM:
//
//   R1  the line's row of the composite store: template (blank + sync pulses) + Y + the low-passed chroma on the
//       subcarrier + burst, converted once per picture and colour-frame phase (k_compose, ref video.c:2864-3040,
//       fir.c:357-375)
//   R2  VBI overlay; the finished composite line goes into a 4-row ring of byte planes in shared memory
//   M   51-tap VSB / low-pass video filter on the tensor cores (ref video.c:3235-3248, fir.c:564-615),
//       FM / AM / NICAM sound carriers (ref video.c:3261-3450, nicam728.c:342-411), IQ swap, offset
//       mixer (ref video.c:3466-3515), channel combiner, store.
//
// Thread <-> sample mapping: a warp owns one tile of 128 consecutive samples and every lane keeps its four
// samples in the layout the m16n8k32 accumulators have anyway: lane = 4g + t holds x = 128 tile + 32 t + g + 8 j,
// j = 0..3 (htv_mma_fir.h: mf_out_x). Both filters leave their results in exactly the registers the next
// stage needs - no exchange through shared memory, and all four samples of a lane fall into one 32-sample
// block: the sound carriers and mixers are htv_sound.cuh's with S = 8, fed per lane (KlFeed below). Loads and stores with a stride of 8 samples between a lane's values are still sector-exact (8 lanes x 4
// bytes = one 32-byte sector).

#define KL_LEAD   MF_LEAD   // composite row: byte i = sample i - 32 of the line (htv_mma_fir.h pitched row)
#define KL_UVLEAD MF_LP_LEAD // chroma planes: byte i = sample i - 8

__device__ __forceinline__ int kl_row_bytes(int W) { return(mf_row_bytes(W) + 16); }
__device__ __forceinline__ int kl_uv_bytes(int W) { return(MF_TILE * mf_tiles(W) + 32); }

// tap operand of the chroma low-pass (one k-step of 32): mf_lp_a_word (htv_mma_fir.h, shared with the host-side emulation)
#define kl_chroma_a_word mf_lp_a_word

// the three partial sums of a byte-split contraction back to the reference's int32 accumulator (mf_combine:
// 65536 hh + 256 mid + ll with wrap-around), as two shift-adds, then >> 15
__device__ __forceinline__ int kl_acc15(int hh, int mid, int ll)
{
	const unsigned t = (unsigned) mid + ((unsigned) hh << 8);
	return((int) ((unsigned) ll + (t << 8)) >> 15);
}
__device__ __forceinline__ int kl_fir_out(int hh, int mid, int ll) { return(sat16i(kl_acc15(hh, mid, ll))); }

// The 51-tap VSB / low-pass video filter on the tensor cores, one tile of 128 samples per warp: ph is the lane's first
// byte (mf_b_offset) of the staged row's high-byte plane, the low-byte plane RB bytes on; atab the tap operand
// ([k-step][I hi, I lo, Q hi, Q lo][lane], shared or global memory). The lane's outputs at xb + 8 j go to oi / oq.
template<bool HASQ>
__device__ __forceinline__ void kl_vfilter(const unsigned char *ph, int RB, const uint4 *atab, int lane, int (&oi)[4], int (&oq)[4])
{
	const unsigned char *plo = ph + RB;
	int ihh[4] = { 0, 0, 0, 0 }, imid[4] = { 0, 0, 0, 0 }, ill[4] = { 0, 0, 0, 0 };
	int qhh[4] = { 0, 0, 0, 0 }, qmid[4] = { 0, 0, 0, 0 }, qll[4] = { 0, 0, 0, 0 };
	#pragma unroll
	for(int s = 0; s < MF_KSTEPS; s++)
	{
		const uint2 xh = *reinterpret_cast<const uint2 *>(ph + 32 * s);
		const uint2 xl = *reinterpret_cast<const uint2 *>(plo + 32 * s);
		const uint4 aih = atab[(s * 4 + 0) * 32 + lane], ail = atab[(s * 4 + 1) * 32 + lane];
		mma_ss(ihh, aih, xh); mma_su(imid, aih, xl); mma_us(imid, ail, xh); mma_uu(ill, ail, xl);
		if(HASQ)
		{
			const uint4 aqh = atab[(s * 4 + 2) * 32 + lane], aql = atab[(s * 4 + 3) * 32 + lane];
			mma_ss(qhh, aqh, xh); mma_su(qmid, aqh, xl); mma_us(qmid, aql, xh); mma_uu(qll, aql, xl);
		}
	}
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		const int ci = mf_lane_ci(j);
		oi[j] = kl_fir_out(ihh[ci], imid[ci], ill[ci]);
		oq[j] = HASQ ? kl_fir_out(qhh[ci], qmid[ci], qll[ci]) : 0;
	}
}

// Mixers after the modulation (htv_sound.cuh), channel combiner, store in the strided layout.
// ST: the sample type the store converts to (htv_sample_type.h), -1 for dp.sample_type at run time. The channel combiner
// (`acc`, int16 in the output layout) still adds in int16 with wrap-around; the conversion is the last step, as the
// reference's file sink converts what the video stage handed it. A lane stores each of its samples on its own (1, 2,
// 4 or 8 bytes); the eight lanes g = 0..7 of a t still cover one contiguous run of the line per j.
// the mixers from the line's sound descriptor or from the lane state (FED)
template<int SND>
__device__ __forceinline__ void kl_mix8(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la, int xb, int (&oi)[4], int (&oq)[4])
{
	kl_mix<SND, 8>(dp, dt, la, xb, oi, oq);
}
template<int SND>
__device__ __forceinline__ void kl_mix8(const htv_dparams_t &dp, const DevTables &dt, const KlLane &L, int xb, int (&oi)[4], int (&oq)[4])
{
	kl_mix_lane<SND, 8>(dp, dt, L, oi, oq);
}

template<bool FULL, int SND, int ST, typename IN>
__device__ __forceinline__ void kl_post_store(const htv_dparams_t &dp, const DevTables &dt, const IN &in,
	int W, int xb, int row, int (&oi)[4], int (&oq)[4], int16_t *out, const int16_t *acc)
{
	kl_mix8<SND>(dp, dt, in, xb, oi, oq);
	const size_t lbase = (size_t) row * (size_t) W;
	if constexpr(ST != HTV_TYPE_INT16)
	{
		const int st = ST < 0 ? dp.sample_type : ST;
		const bool cpx = KL_HAS(SND, KL_CPX, dp.complex_out);
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			if(FULL || xb + 8 * j < W) st_put_sum(out, acc, lbase + xb + 8 * j, st, cpx, oi[j], oq[j]);
		}
		return;
	}
	if(KL_HAS(SND, KL_CPX, dp.complex_out))
	{
		unsigned *o = reinterpret_cast<unsigned *>(out) + lbase + xb;
		const unsigned *a = acc ? reinterpret_cast<const unsigned *>(acc) + lbase + xb : NULL;
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			if(FULL || xb + 8 * j < W)
			{
				unsigned v = ((unsigned) oi[j] & 0xFFFFu) | ((unsigned) oq[j] << 16);
				if(a) v = __vadd2(v, __ldcs(a + 8 * j));
				__stcs(o + 8 * j, v);
			}
		}
	}
	else
	{
		unsigned short *o = reinterpret_cast<unsigned short *>(out) + lbase + xb;
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			if(FULL || xb + 8 * j < W) o[8 * j] = (unsigned short) (oi[j] + (acc ? acc[lbase + xb + 8 * j] : 0));
		}
	}
}

// ---- k_line's sound feed ---------------------------------------------------------------------------------------
// A lane's samples are xb + 8 j of every line, so the audio-clock index m = L W + shift + xb of its first sample grows by
// exactly W from one line to the next. The sound state is a closed form of m: the audio index in effect
// j = floor(32000 (m + 1) / rate) - 1, the NICAM symbol in effect s = floor(m D / F), m mod 32767 and m mod nicam_cc_len.
// A CTA sets them up once by exact 64-bit division (kd_div) and then advances each quotient and remainder by the
// increments of one line (htv_dparams_t kl_w_*). What varies per audio sample or per symbol comes from the records the
// pre-pass chains write - dt.seg_rec (k_fm_scan_fix) and dt.nic_rec (k_nicam_rec) - loaded where the line's lane
// state is built (kl_lane_feed), so that no record is held in registers from one line to the next.
struct KlFeed {
	unsigned aq, ar;            // 32000 (m + 1) = aq rate + ar: aq = j + 1 (mod 2^32), the slot of j's record
	unsigned sq, sr;            // m D = sq F + sr: sq = s (mod 2^32); sr / D samples into symbol s
	int kk, cc;                 // m mod 32767, m mod nicam_cc_len
	ulonglong2 seg;             // record of audio index j: B(j), angle step ... (kl_feed_load)
	float2 rot;                 // ... and (cos, sin) of 8 steps
	unsigned nA, nB;            // records of symbols s and s + 1
};

template<int SND>
__device__ __forceinline__ void kl_feed_load(const htv_dparams_t &dp, const DevTables &dt, KlFeed &f)
{
	if(KL_HAS(SND, KL_FM, dp.have_fm))
	{
		const SegRec *r = dt.seg_rec + (f.aq & (RA - 1));
		f.seg = __ldg(&r->ba);
		f.rot = __ldg(&r->rot);
	}
	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		f.nA = __ldg(dt.nic_rec + (f.sq & (RS - 1)));
		f.nB = __ldg(dt.nic_rec + ((f.sq + 1) & (RS - 1)));
	}
}

// the feed of audio-clock index m (>= 0)
template<int SND>
__device__ __forceinline__ void kl_feed_init(const htv_dparams_t &dp, const DevTables &dt, KlFeed &f, long long m)
{
	unsigned rem;
	kd_div((unsigned long long) m, 32767u, 1.0 / 32767.0, rem);
	f.kk = (int) rem;
	if(KL_HAS(SND, KL_FM, dp.have_fm) || KL_HAS(SND, KL_AM, dp.have_am))
	{
		f.aq = (unsigned) kd_div((unsigned long long) (m + 1) * HTV_AUDIO_RATE, (unsigned) dp.rate, 1.0 / (double) dp.rate, rem);
		f.ar = rem;
	}
	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		f.sq = (unsigned) kd_div((unsigned long long) m * (unsigned) dp.nicam_D, (unsigned) dp.nicam_F, 1.0 / (double) dp.nicam_F, rem);
		f.sr = rem;
		kd_div((unsigned long long) m, (unsigned) dp.nicam_cc_len, 1.0 / (double) dp.nicam_cc_len, rem);
		f.cc = (int) rem;
	}
}

// the feed W samples on (the lane's first sample on the next line)
template<int SND>
__device__ __forceinline__ void kl_feed_next(const htv_dparams_t &dp, const DevTables &dt, KlFeed &f)
{
	f.kk += dp.kl_w_kk;
	if(f.kk >= 32767) f.kk -= 32767;
	if(KL_HAS(SND, KL_FM, dp.have_fm) || KL_HAS(SND, KL_AM, dp.have_am))
	{
		f.aq += dp.kl_w_aq; f.ar += dp.kl_w_ar;
		if(f.ar >= (unsigned) dp.rate) { f.ar -= (unsigned) dp.rate; f.aq++; }
	}
	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		f.sq += dp.kl_w_sq; f.sr += dp.kl_w_sr;
		if(f.sr >= (unsigned) dp.nicam_F) { f.sr -= (unsigned) dp.nicam_F; f.sq++; }
		f.cc += dp.kl_w_cc;
		if(f.cc >= dp.nicam_cc_len) f.cc -= dp.nicam_cc_len;
	}
}

// the sound stage's lane state from the feed at audio-clock index m (the segment start st(j) = m - floor(ar / 32000):
// the record of j = -1 is stored one step back, so that the same form holds at the stream start, where st = 0).
// PART: which of L's fields - 1 the FM and AM carriers' and kk, 2 NICAM's, 4 the offset mixer's (kl_sound)
template<int SND, int PART>
__device__ __forceinline__ void kl_lane_feed(const htv_dparams_t &dp, const DevTables &dt, KlFeed f, long long m, KlLane &L)
{
	kl_feed_load<SND>(dp, dt, f);
	if(PART & 1)
	{
		L.kk = f.kk;
		L.nb = 0x7FFFFFFF;
	}
	const bool fm = (PART & 1) && KL_HAS(SND, KL_FM, dp.have_fm), am = (PART & 1) && KL_HAS(SND, KL_AM, dp.have_am);
	if(fm || am)
	{
		const int nb = (int) (((unsigned) dp.rate - f.ar + HTV_AUDIO_RATE - 1) / HTV_AUDIO_RATE);   // first sample of j + 1
		if(nb <= 24) L.nb = nb;
		if(fm)
		{
			L.angA = f.seg.y;
			L.phA = f.seg.x + f.seg.y * (unsigned long long) (f.ar / HTV_AUDIO_RATE + 1);
			L.rot = f.rot;
			L.angB = L.angA; L.phB = L.phA;
			if(nb <= 24)
			{
				const ulonglong2 b = __ldg(&dt.seg_rec[(f.aq + 1) & (RA - 1)].ba);
				L.angB = b.y;
				L.phB = b.x - b.y * (unsigned long long) (nb - 1);
			}
		}
		if(am)
		{
			const bool neg = (unsigned long long) HTV_AUDIO_RATE * (unsigned long long) (m + 1) < (unsigned long long) dp.rate;   // j < 0
			L.amA = (pcm_mono(dt, neg ? -1 : (int64_t) (f.aq - 1), dp.volume) + 32768) / 2;
			L.amB = (pcm_mono(dt, (int64_t) f.aq, dp.volume) + 32768) / 2;
			L.phM = dp.am_ang * (unsigned long long) (m + 1);
		}
	}
	if((PART & 2) && KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		const unsigned D = (unsigned) dp.nicam_D;
		const int off = (int) (f.sr / D), dist = (int) (((unsigned) dp.nicam_F - f.sr + D - 1) / D);   // s started off samples ago, s + 1 starts at dist
		L.nbs = dist;
		L.niA = (int) (f.nA & 511u) * dp.nicam_sps + off; L.nqA = (int) ((f.nA >> 9) & 511u) * dp.nicam_sps + off;
		L.niB = (int) (f.nB & 511u) * dp.nicam_sps - dist; L.nqB = (int) ((f.nB >> 9) & 511u) * dp.nicam_sps - dist;
		L.gen = !dp.nicam_lut_ok || dp.nicam_sps - 1 < 32 || ((f.nA >> 20) & 1u) || (dist <= 24 && ((f.nB >> 20) & 1u));
		L.cc = f.cc;
	}
	if(PART & 4)
	{
		L.kk = f.kk;
		L.m = m;
		L.offph = dp.offset_phase0 + dp.offset_ang * (unsigned long long) (m + 1 - 32767);
	}
}

// the generic NICAM sum of the samples m + 8 j: the symbols whose pulse covers a sample, from the newest started at or
// before it (symbol sx, rx / D samples ago) back, their polarities from the records
__device__ __forceinline__ void kl_nic_generic_feed(const htv_dparams_t &dp, const DevTables &dt, const KlFeed &f, long long m,
	const short *ntp, int (&bi)[4], int (&bq)[4])
{
	const unsigned F = (unsigned) dp.nicam_F, D = (unsigned) dp.nicam_D;
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		unsigned rx = f.sr + 8u * j * D;
		const unsigned sx = f.sq + rx / F;
		rx %= F;
		bi[j] = 0; bq[j] = 0;
		for(int cnd = 0; cnd < NIC_CAND; cnd++)
		{
			const unsigned d = (rx + cnd * F) / D;                      // samples since symbol sx - cnd started
			if((long long) d > m + 8 * j) break;                        // before the stream start
			const int sy = (int) (__ldg(dt.nic_rec + ((sx - cnd) & (RS - 1))) >> 18) & 3;
			kl_nic_add(sy, ntp[d + NIC_TPAD], bi[j], bq[j]);            // the table is zero outside the pulse
		}
	}
}

// cp.async: 16 bytes global -> shared without passing through registers
__device__ __forceinline__ void kl_cp16(void *dst_smem, const void *src)
{
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void kl_cp_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// VF: a video filter is on; HASQ: it has Q taps (VSB); FULL: 128 | W (no
// partial tile: the x < W tests fold away); CSAT: the chroma low-pass can leave the int16 range (sum of |taps| > 32768),
// which k_compose's saturating low-pass handles when it fills the store: the CSAT forms run the same code as the others
//
// The forms with a video filter and a composite store (FS: VF, not PS, not SRC) do not filter: k_vf_rows filtered each
// line's three composite rows and overlays once, into the filtered store (a row per line of each slot and phase) or,
// for the lines whose filter window leaves one frame's rows or meets an overlay, into the call's own rows. Per
// iteration q they load line q + 1's filtered I | Q (R1), and give line q its sound carriers and store it (M). They read
// the raster descriptor's pic a line ahead of R1 by a uniform load; with the sound state fed per lane (FED, below) that
// is their only per-line value, and their warps share nothing per line and meet at no barrier.
//
// Every other form, per iteration q (one scan line), runs
//   R2(q)   VBI overlay on the values fetched earlier, composite row q mod 4                  | __syncthreads
//   R1(q+1) the composite row of the NEXT line is loaded here ...
//   M(q-1)  ... and arrive while line q - 1 (whose right-hand halo R2(q) has just written) is filtered (mma),
//           gets its sound carriers and is stored.
// The raster descriptor of line q + 1 and, unless FED, the sound descriptor of the line modulated come in by cp.async at
// the top of the iteration.
// FED: the forms with the sound stages compiled in (SND >= 0) derive each lane's sound state from its audio-clock index
// (KlFeed), set up once per CTA and advanced by W per line, instead of reading LineA2. The general forms (SND = -1)
// keep reading LineA2: with every stage a run-time flag, the feed's state and arithmetic cost them more registers and
// time than the descriptor does (at W = 1280, 320 threads: k_line 0.385 against 0.217 ms per 64 frames on an H100).
// One barrier per line, so the ring has 4 rows: a warp that is through M(q - 1) may run on into R2(q + 1), before the
// next barrier, while another warp is still reading line q - 1's row. R2(q + 1) writes line q + 1's row, the right
// halo of line q's and the left halo of line q + 2's; with 4 rows none of them is line q - 1's.
//
// SRC: the composite lines are not rastered here but read from `src` (row q + 2 = relative line q, int16): SECAM, whose
// chrominance chain (htv_secam.cuh) runs between the raster and the modulator. R2 folds away, the rest is the same.
// WC: the line width compiled in (0: dp.W), so that the shared-memory row and plane offsets become immediates
// ST: the output sample type compiled into the store (HTV_TYPE_INT16: the int16 store), -1: dp.sample_type at run time
//
// PS: encoders whose colour subcarrier does not repeat within 4 frames (htv_tables.c comp_phases = 0) have no composite
// store. Their R1 reads the converted picture store instead - template + Y and, on colour lines, U | V << 16 after the
// chroma low-pass, converted once per picture (k_picture) - and R2 adds burst and subcarrier (ref video.c:3011-3040).
//
// S-Video (KL_SV, dp.s_video; ref video.c:3031-3040, 3206-3228): the subcarrier term goes to Q instead of I, and the
// video filter runs on I only, so Q of the stored line is that line's own chroma. k_compose wrote it into the store's
// chroma plane (dt.comp_q), which M reads at the row of mrow (FS: k_vf_rows added it to Q of the filtered row); SRC: the
// chain wrote Q into its own plane, `srcq`; PS: R2
// parks it in a two-row ring in shared memory at the lane's own slots (row q & 1), which M takes back for mrow.
template<bool VF, bool HASQ, bool FULL, bool CSAT, int MAXT, int MINB, bool SRC = false, int SND = -1, int WC = 0, int ST = HTV_TYPE_INT16,
	bool PS = false>
__global__ void __launch_bounds__(MAXT, MINB)
k_line(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineR2 *lrp, const LineA2 *lap, long long mf,
	int nlines, int run, int16_t *out, const int16_t *acc, int acc_rows, const int16_t *src = nullptr, const int16_t *srcq = nullptr)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	// FS: the filtered store holds each line's filter output (k_vf_rows); RING: the filter runs here, on the ring
	constexpr bool FS = VF && !PS && !SRC, RING = VF && !FS, FED = SND >= 0;
	const int W = WC ? WC : dp.W;
	const int RB = kl_row_bytes(W);
	// lap: the sound descriptors (not FED); mf: the audio-clock index of relative line 0's first sample (line0 W + shift, FED)
	// sound descriptors x2 (not FED) | raster descriptors x2 | RING: [row 0..3][hi, lo] composite planes, FIR taps | NICAM
	// pulse | PS, S-Video: chroma [row 0..1][j][thread]
	LineA2 *sla = reinterpret_cast<LineA2 *>(smem_raw);
	LineR2 *slr = reinterpret_cast<LineR2 *>(sla + (FED ? 0 : 2));
	unsigned char *rows = reinterpret_cast<unsigned char *>(slr + 2);
	uint4 *atab = reinterpret_cast<uint4 *>(rows + (RING ? 8 * RB : 0));  // [k-step][I hi, I lo, Q hi, Q lo][lane]
	short *ntp = reinterpret_cast<short *>(atab + (RING ? MF_ATAB_WORDS / 4 : 0));
	const int tid = threadIdx.x, lane = tid & 31, nt = tid >> 5;
	const int g = lane >> 2, t = lane & 3;
	const int xb = mf_lane_x(nt, lane, 0);                                  // the lane's samples: xb + 8 j
	const bool sv = KL_HAS(SND, KL_SV, dp.s_video);
	short *const svq = ntp + ((dp.nicam_tpad_len + 7) & ~7);

	const int a = blockIdx.x * run, bnd = min(a + run, nlines);
	if(a >= nlines) return;
	// relative line q: raster lines a-1 .. bnd (descriptor lrp[q + 1]), modulate a .. bnd-1
	const int q0 = RING ? a - 1 : a, q1 = RING ? bnd : bnd - 1;

	// ---- one-time set-up -------------------------------------------------------
	if(RING) for(int i = tid; i < MF_ATAB_WORDS / 4; i += blockDim.x) atab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.mma_atab) + i);
	if(RING) for(int i = tid; i < 8 * RB / 4; i += blockDim.x) reinterpret_cast<unsigned *>(rows)[i] = 0;
	if(KL_HAS(SND, KL_NIC, dp.have_nicam)) kl_tpad_load(dp, dt, ntp);
	if(!SRC && !FS && tid < 4) reinterpret_cast<int4 *>(slr + (q0 & 1))[tid] = __ldg(reinterpret_cast<const int4 *>(lrp + q0 + 1) + tid);
	__syncthreads();
	// FS: pic of the line R1 loads next (q0, then q0 + 1 ...), and of the one after it
	long long fpic = FS ? __ldg(&lrp[q0 + 1].pic) : 0;
	long long fpn = FS && q0 + 1 <= q1 ? __ldg(&lrp[q0 + 2].pic) : 0;
	const bool snd = FED && KL_HAS(SND, KL_FM, dp.have_fm) || KL_HAS(SND, KL_AM, dp.have_am) || KL_HAS(SND, KL_NIC, dp.have_nicam) ||
		KL_HAS(SND, KL_OFF, dp.have_offset);
	const long long mx0 = mf + xb;                                          // the lane's first sample on relative line 0
	KlFeed fd;
	if(snd) kl_feed_init<SND>(dp, dt, fd, mx0 + (long long) a * W);

	// PS: the span the chroma low-pass reaches (taps <= 17: 8 samples either side of the picture); the store is zero outside
	const bool in_chroma = xb + 24 >= dp.active_left - 8 && xb < dp.active_left + dp.active_width + 8;
	const bool in_burst = xb + 24 >= dp.burst_left && xb < dp.burst_left + dp.burst_width;
	const int fo0 = mf_b_offset(nt, 0, lane);
	constexpr int NA16 = FED ? 0 : (int) (sizeof(LineA2) / 16);

	// loads of line q issued one phase early: the line's composite row (int16 x 4); FS: the line's filtered I | Q << 16
	// (x 4), from the filtered store or, for the lines k_line_desc_r listed (pic < 0), from the call's rows at the list
	// index; PS: line values (int16 x 4) and, on colour lines, filtered U | V << 16 (x 4)
	int tm[4];
	unsigned px[4];
	#define KL_R1(QQ) do { \
		if(FS) \
		{ \
			const long long pic_ = fpic; \
			const uint32_t *fp_ = (pic_ >= 0 ? dt.filt + pic_ : dt.vfx + (size_t) (-1 - pic_) * W) + xb; \
			_Pragma("unroll") for(int j = 0; j < 4; j++) px[j] = (FULL || xb + 8 * j < W) ? __ldg(fp_ + 8 * j) : 0u; \
			break; \
		} \
		if(!PS) \
		{ \
			const int16_t *tp_ = SRC ? src + (size_t) ((QQ) + 2) * W + xb : dt.comp + slr[(QQ) & 1].pic + xb; \
			_Pragma("unroll") for(int j = 0; j < 4; j++) tm[j] = (FULL || xb + 8 * j < W) ? (int) __ldg(tp_ + 8 * j) : 0; \
			break; \
		} \
		const LineR2 &ln = slr[(QQ) & 1]; \
		const long long pic_ = ln.pic; \
		const int16_t *tp_ = (pic_ >= 0 ? dt.pic_val + pic_ : dt.tmpl_out + (size_t) ln.tmpl * W) + xb; \
		_Pragma("unroll") for(int j = 0; j < 4; j++) tm[j] = (FULL || xb + 8 * j < W) ? (int) __ldg(tp_ + 8 * j) : 0; \
		if(in_chroma && ln.pal && pic_ >= 0) \
		{ \
			const uint32_t *cp_ = dt.pic_cuv + pic_ + xb; \
			_Pragma("unroll") for(int j = 0; j < 4; j++) px[j] = (FULL || xb + 8 * j < W) ? __ldg(cp_ + 8 * j) : 0u; \
		} \
		else { px[0] = px[1] = px[2] = px[3] = 0u; } \
	} while(0)
	KL_R1(q0);

	int r4 = q0 & 3;                                                        // ring row of line q
	for(int q = q0; q <= q1; q++, r4 = (r4 + 1) & 3)
	{
		const int mrow = RING ? q - 1 : q;                                  // the line modulated in this iteration
		// ---- the raster descriptor of the next line -> shared memory ------------------------------------------
		if(tid < 4) { if(!SRC && !FS && q + 1 <= q1) kl_cp16(reinterpret_cast<int4 *>(slr + ((q + 1) & 1)) + tid, reinterpret_cast<const int4 *>(lrp + q + 2) + tid); }
		else if(tid < 4 + NA16) { if(mrow >= a) kl_cp16(reinterpret_cast<int4 *>(sla + (mrow & 1)) + (tid - 4), reinterpret_cast<const int4 *>(lap + mrow) + (tid - 4)); }
		// a CTA narrower than 4 + NA16 threads (one warp: W <= 128) copies the rest of the sound descriptor in further passes
		if(!FED && (int) blockDim.x < 4 + NA16 && mrow >= a)
			for(int i = (int) blockDim.x - 4 + tid; i < NA16; i += blockDim.x)
				kl_cp16(reinterpret_cast<int4 *>(sla + (mrow & 1)) + i, reinterpret_cast<const int4 *>(lap + mrow) + i);

		// ---- R2: (PS: burst, subcarrier,) VBI overlay of line q ---------------------
		const LineR2 &li = slr[q & 1];
		int val[4] = { tm[0], tm[1], tm[2], tm[3] };
		const unsigned fv[4] = { px[0], px[1], px[2], px[3] };              // FS: the filtered line q
		const int mpic = !VF && !SRC && !PS && sv ? (int) li.pic : 0;       // S-Video: the row of the line (< 2^31, htv_dev_create)
		int cq[4] = { 0, 0, 0, 0 };                                         // PS, S-Video: the chroma of line q
		if(PS && li.pal)
		{
			const int li_pal = li.pal;
			short2 cl[4];
			{
				const htv_c16_t *cp = dt.clut + li.clut_off + xb;
				#pragma unroll
				for(int j = 0; j < 4; j++) cl[j] = (FULL || xb + 8 * j < W) ? kl_ldc16(cp + 8 * j) : make_short2(0, 0);
			}
			int cu[4], cv[4];
			#pragma unroll
			for(int j = 0; j < 4; j++) { cu[j] = (int) (short) (px[j] & 0xFFFFu); cv[j] = (int) px[j] >> 16; }
			if(in_burst)
			{
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int x = xb + 8 * j;
					if(x >= dp.burst_left && x < dp.burst_left + dp.burst_width)
					{
						const int w = dt.burst_win[x - dp.burst_left];
						cu[j] = (dp.burst_i * w) >> 15;
						cv[j] = (dp.burst_q * w) >> 15;
					}
				}
			}
			if(sv)
			{
				#pragma unroll
				for(int j = 0; j < 4; j++) cq[j] = ((int) cl[j].x * cv[j] * li_pal + (int) cl[j].y * cu[j]) >> 15;
			}
			else
			{
				#pragma unroll
				for(int j = 0; j < 4; j++) val[j] += ((int) cl[j].x * cv[j] * li_pal + (int) cl[j].y * cu[j]) >> 15;
			}
		}
		if(PS && sv)
		{
			#pragma unroll
			for(int j = 0; j < 4; j++) svq[((q & 1) * 4 + j) * blockDim.x + tid] = (short) cq[j];
		}
		if(!SRC && !FS && li.ov_any)
		{
			// VBI stages run on the finished line (ref video.c:4213-4357 register them behind the raster)
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				const int x = xb + 8 * j;
				if(x >= li.ov_from && x < li.ov_to) val[j] = li.ov_value;
				if(li.ov_add >= 0 && x < W) val[j] = wrap16i(val[j]) + dt.ov_add[(size_t) li.ov_add * W + x];
			}
		}

		const int rprev = r4 == 0 ? 3 : r4 - 1, rnext = r4 == 3 ? 0 : r4 + 1;   // ring rows of lines q - 1, q + 1
		if(RING)
		{
			// ---- composite line -> ring row q mod 4 (+ the neighbours' halos) ----------
			unsigned char *rp = rows + (2 * r4) * RB + KL_LEAD + xb;
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				if(FULL || xb + 8 * j < W) { rp[8 * j] = (unsigned char) (val[j] >> 8); rp[RB + 8 * j] = (unsigned char) val[j]; }
			}
			if(xb < KL_LEAD)
			{
				// first 32 samples: right halo of the previous line's row
				unsigned char *hp = rows + (2 * rprev) * RB + KL_LEAD + W + xb;
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					if(xb + 8 * j < KL_LEAD) { hp[8 * j] = (unsigned char) (val[j] >> 8); hp[RB + 8 * j] = (unsigned char) val[j]; }
				}
			}
			if(xb + 24 >= W - KL_LEAD && xb < W)
			{
				// last 32 samples: left halo of the next line's row
				unsigned char *hp = rows + (2 * rnext) * RB + xb - (W - KL_LEAD);
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int x = xb + 8 * j;
					if(x >= W - KL_LEAD && x < W) { hp[8 * j] = (unsigned char) (val[j] >> 8); hp[RB + 8 * j] = (unsigned char) val[j]; }
				}
			}
		}
		if(!FS || !FED)
		{
			if(tid < 4 + NA16 || (!FED && (int) blockDim.x < 4 + NA16)) kl_cp_wait();
			__syncthreads();                                                // rows of line q, the descriptors of q + 1 and of mrow
		}

		// ---- R1: the next line's values start their way here -------------------------
		if(q + 1 <= q1)
		{
			fpic = fpn;
			KL_R1(q + 1);
			if(FS && q + 2 <= q1) fpn = __ldg(&lrp[q + 3].pic);
		}
		if(mrow < a) continue;

		int oi[4], oq[4];
		if(RING) kl_vfilter<HASQ>(rows + (2 * rprev) * RB + fo0, RB, atab, lane, oi, oq);   // ---- M: video filter of line q - 1
		else if(FS)
		{
			#pragma unroll
			for(int j = 0; j < 4; j++) { oi[j] = (int) (short) (fv[j] & 0xFFFFu); oq[j] = (int) fv[j] >> 16; }
		}
		else
		{
			#pragma unroll
			for(int j = 0; j < 4; j++) { oi[j] = wrap16i(val[j]); oq[j] = 0; }
		}

		// ---- sound carriers, mixers, store ---------------------------------------
		if(FULL || xb < W)
		{
			if(sv && !FS)
			{
				// Q = the chroma of line mrow (the video filter leaves it alone; FS: k_vf_rows added it)
				const int16_t *qp = (SRC ? srcq + (size_t) (mrow + 2) * W : PS ? srcq : dt.comp_q + mpic) + xb;
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					if(PS) oq[j] += svq[((mrow & 1) * 4 + j) * blockDim.x + tid];
					else oq[j] += (FULL || xb + 8 * j < W) ? (int) __ldg(qp + 8 * j) : 0;
				}
			}
			if(!FED)
			{
				const LineA2 *la = sla + (mrow & 1);
				kl_sound<SND, 8>(dp, dt, la, ntp, xb, oi, oq);
				kl_post_store<FULL, SND, ST>(dp, dt, la, W, xb, mrow, oi, oq, out, mrow < acc_rows ? acc : NULL);
				continue;
			}
			const long long m = mx0 + (long long) mrow * W;
			// the FM and AM carriers, NICAM, the mixers: each part's state built right before it runs
			KlLane L;
			const auto gen = [&](int (&bi)[4], int (&bq)[4]) { kl_nic_generic_feed(dp, dt, fd, m, ntp, bi, bq); };
			kl_lane_feed<SND, 1>(dp, dt, fd, m, L);
			kl_sound_lane<SND, 8, false, 1>(dp, dt, L, oi, oq, gen);
			kl_lane_feed<SND, 2>(dp, dt, fd, m, L);
			kl_sound_lane<SND, 8, false, 2>(dp, dt, L, oi, oq, gen);
			kl_lane_feed<SND, 4>(dp, dt, fd, m, L);
			if(snd) kl_feed_next<SND>(dp, dt, fd);
			kl_post_store<FULL, SND, ST>(dp, dt, L, W, xb, mrow, oi, oq, out, mrow < acc_rows ? acc : NULL);
		}
	}
	#undef KL_R1
}

// ---------------------------------------------------------------------------
// k_vf_rows: the video filter of the k_line forms with a composite store (FS), once per row instead of once per line of
// every frame. A CTA filters one line, a warp one tile of 128 samples, as k_line's M stage did: the three composite rows
// of lines L - 1 .. L + 1 (32-sample halos on the neighbours) go into a row of byte planes in shared memory exactly as
// k_line's ring held them, with their VBI overlays; the output is the pair k_line holds before the sound carriers,
// I | Q << 16, with S-Video's chroma added to Q.
//   blocks [0, cv.n (lines - 2)): the filtered store's rows of lines 2 .. lines - 1 of the composite-store entries cv.e
//            (slot * comp_phases + phase) - rows of one entry, no overlays
//   the rest: row k of dt.vfx, line first + dt.vf_list[1 + k], for k < dt.vf_list[0] (vf_exception)
// ---------------------------------------------------------------------------
#define VF_CONV 64                    // composite-store entries one launch filters: all of a call's (htv_dev_create checks)
struct VfConv { int n; int e[VF_CONV]; };

template<bool HASQ>
__global__ void __launch_bounds__(384)
k_vf_rows(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const __grid_constant__ VfConv cv, int64_t first)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	__shared__ int4 som[3];                                             // the overlays of lines L - 1 .. L + 1
	__shared__ int sov[3];
	const int W = dp.W, RB = kl_row_bytes(W), N = dp.lines;
	const int tid = threadIdx.x, lane = tid & 31;
	const int ns = cv.n * (N - 2);
	long long row[3];                                                   // composite rows of lines L - 1, L, L + 1
	uint32_t *dst;
	const bool exc = (int) blockIdx.x >= ns;
	if(!exc)
	{
		const long long r = (long long) cv.e[blockIdx.x / (N - 2)] * N + blockIdx.x % (N - 2) + 1;
		row[0] = r - 1; row[1] = r; row[2] = r + 1;
		dst = dt.filt + r * W;
	}
	else
	{
		const int k = blockIdx.x - ns;
		if(k >= dt.vf_list[0]) return;
		const int64_t L = first + dt.vf_list[1 + k];
		#pragma unroll
		for(int d = 0; d < 3; d++) row[d] = comp_row(dp, dt, L - 1 + d);
		dst = dt.vfx + (size_t) k * W;
		if(tid < 3) sov[tid] = line_overlay(dt, L - 1 + tid, som[tid]);
		__syncthreads();
	}

	// ---- the composite window of line L -> [hi, lo] byte planes (byte b = sample b - KL_LEAD) --------------
	unsigned char *ph = smem_raw;
	for(int b = tid; b < RB; b += blockDim.x)
	{
		const int x = b - KL_LEAD, d = x < 0 ? 0 : x < W ? 1 : 2, xs = x - (d - 1) * W;
		int val = 0;
		if(d != 2 || x < W + KL_LEAD)
		{
			val = dt.comp[row[d] * W + xs];
			if(exc && sov[d])
			{
				const int4 m = som[d];
				if(xs >= m.x && xs < m.y) val = m.z;
				if(m.w >= 0) val = wrap16i(val) + dt.ov_add[(size_t) m.w * W + xs];
			}
		}
		ph[b] = (unsigned char) (val >> 8);
		ph[RB + b] = (unsigned char) val;
	}
	__syncthreads();

	int oi[4], oq[4];
	const int nt = tid >> 5, xb = mf_lane_x(nt, lane, 0);
	kl_vfilter<HASQ>(ph + mf_b_offset(nt, 0, lane), RB, reinterpret_cast<const uint4 *>(dt.mma_atab), lane, oi, oq);
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		const int x = xb + 8 * j;
		if(x >= W) continue;
		if(dp.s_video) oq[j] += dt.comp_q[row[1] * W + x];
		dst[x] = ((unsigned) oi[j] & 0xFFFFu) | ((unsigned) oq[j] << 16);
	}
}
