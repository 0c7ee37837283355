// hacktv_b200 - the sound carriers and the post-modulation mixers (included by htv_kernels.cu), for the fused line kernel
// (htv_line.cuh) and for the split and FM-video modulators alike, on four samples per thread, S apart:
//   S = 8: k_line's lane layout (x = xb + 8 j, the m16n8k32 accumulator layout, htv_mma_fir.h: mf_out_x);
//   S = 1: four consecutive samples (k_mod, k_mod_tma, k_mod_mma, k_fmv_base, k_fmv_mod).
// Either way all four samples fall into one 32-sample block. The arithmetic - the reference's Q31 phasor, the FM and AM
// carriers, the NICAM pulse look-up, overlap-add and carrier multiply, IQ swap and the offset mixer - is written once,
// in primitives that take plain values (kl_amp .. kl_offset). Two entries feed them: kl_sound / kl_mix read the
// per-line sound descriptor LineA2 (k_line_desc_a2), which the descriptor is indexed by; kl_sound_lane / kl_mix_lane
// read a lane state (KlLane) that the k_line forms with the sound stages compiled in derive per lane (htv_line.cuh
// KlFeed). Two entries rather than one fed two ways: built from LineA2 through a KlLane, the general forms of k_line and
// the split modulators held the state in registers instead of reading it from shared memory where they use it, and the
// 320-thread k_line forms spilled 120-340 bytes.

#define KL_BIAS   2048      // NICAM pulse-table index bias (LineA2.symb)

// one complex int16 table entry through the read-only path: x = i, y = q
__device__ __forceinline__ short2 kl_ldc16(const htv_c16_t *p) { return(__ldg(reinterpret_cast<const short2 *>(p))); }

// the zero-padded NICAM pulse table (htv_tables.c: 8 zeros, the pulse, zeros) -> shared memory, by the whole CTA
__device__ __forceinline__ void kl_tpad_load(const htv_dparams_t &dp, const DevTables &dt, short *ntp)
{
	const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
	int4 *dst = reinterpret_cast<int4 *>(ntp);
	for(int i = threadIdx.x; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
}

// one line's sound descriptor -> shared memory, by the whole CTA
__device__ __forceinline__ void kl_la_load(LineA2 *dst, const LineA2 *src)
{
	for(int i = threadIdx.x; i < (int) (sizeof(LineA2) / 16); i += blockDim.x)
		reinterpret_cast<int4 *>(dst)[i] = __ldg(reinterpret_cast<const int4 *>(src) + i);
}

// SND: the sound carriers and post-modulation stages an instantiation has compiled in, as a mask of the flags below, or
// -1 for the general form, which tests dp on every line. They are fixed for an encoder's life, so the host picks the
// instantiation from dp (kl_snd_mask). Only the mask of the PAL systems with FM mono and NICAM on a VSB carrier has its
// own instantiation, and only at W = 1024 (16 Msps), with the width compiled in too (WC); at 320 threads the fixed form
// spills.
#define KL_FM   1
#define KL_AM   2
#define KL_NIC  4
#define KL_OFF  8
#define KL_SWAP 16
#define KL_CPX  32
#define KL_SV   64      // S-Video: the colour subcarrier goes to Q (k_line only; no compiled-in mask has it)
#define KL_SND_FM_NICAM (KL_FM | KL_NIC | KL_CPX)
#define KL_HAS(SND, BIT, RT) ((SND) < 0 ? (RT) != 0 : ((SND) & (BIT)) != 0)

static inline int kl_snd_mask(const htv_dparams_t &dp)
{
	return((dp.have_fm ? KL_FM : 0) | (dp.have_am ? KL_AM : 0) | (dp.have_nicam ? KL_NIC : 0) |
		(dp.have_offset ? KL_OFF : 0) | (dp.swap_iq ? KL_SWAP : 0) | (dp.complex_out ? KL_CPX : 0) | (dp.s_video ? KL_SV : 0));
}

// ---- the arithmetic, on plain values (ref video.c:3261-3515, nicam728.c:342-411) ----------------------------------
// The reference's Q31 phasor: its amplitude kq = kk + 1 multiplications after a renormalisation (every 32 767 samples),
// and the fast sin / cos of a 0.64 phase. Its (I, Q) are __float2int_rd(amp * cs), __float2int_rd(amp * sn): the FM and
// AM carriers take them as they are, the offset mixer and the FM video modulator clamp them to 32767.
__device__ __forceinline__ float kl_amp(float kq) { return(32767.99998f - kq * 1.52587890625e-5f); }
__device__ __forceinline__ void kl_sincos(unsigned long long ph, float &sn, float &cs)
{
	__sincosf((float) (int) (ph >> 32) * 1.4629180792671596e-9f, &sn, &cs);   // pi / 2^31
}

// FM carrier, rotation form: one sin/cos for the first sample (phase ph, amplitude kf = kk + 1), the other three by
// rotating with rot, the segment's (cos, sin) of S angle steps. Only where no audio-segment boundary and no
// renormalisation falls between the samples. The carriers take their level by reference, so that it is read where it
// is used: read once ahead of the branch between the two FM forms, it changes the bench form's register allocation.
template<int S>
__device__ __forceinline__ void kl_fm_rot(unsigned long long ph, float2 rot, float kf, const int &level, int (&oi)[4], int (&oq)[4])
{
	float sn, cs;
	kl_sincos(ph, sn, cs);
	float amp = kl_amp(kf);
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		oi[j] += (__float2int_rd(amp * cs) * level) >> 15;
		oq[j] += (__float2int_rd(amp * sn) * level) >> 15;
		const float c2 = __fmaf_rn(cs, rot.x, -(sn * rot.y)), s2 = __fmaf_rn(sn, rot.x, cs * rot.y);
		cs = c2; sn = s2;
		amp -= (float) S * 1.52587890625e-5f;
	}
}

// FM carrier, per-sample form: every sample its own sin/cos. phA / angA: segment A's phase at the first sample and its
// step per sample; phB / angB segment B's, in effect from sample nb on, where x0 is the first sample (nb and x0 count from
// the same origin: the line's first sample in the descriptor entry, the thread's first in the lane entry, x0 = 0).
// phase(j, ph) gives sample j's phase from the running phase ph.
// PRECISE (FM video only): in fp64 from the full 64-bit phase. An FM modulator integrates its input, so a sound-carrier
// sample that is 1 LSB off turns everything after it; the fast fp32 evaluation loses the sign of a carrier sample that
// lands on a zero crossing (an unmodulated 6.5 MHz carrier at 20 Msps does so every 40 samples).
template<int S, bool PRECISE, typename PH>
__device__ __forceinline__ void kl_fm_each(unsigned long long phA, unsigned long long angA, unsigned long long phB,
	unsigned long long angB, int x0, int nb, float kf, const int &level, int (&oi)[4], int (&oq)[4], PH phase)
{
	const unsigned long long stA = angA * S, stB = angB * S;
	float kq = kf;
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		const unsigned long long ph = phase(j, x0 + S * j >= nb ? phB : phA);
		if(kq > 32767.0f) kq -= 32767.0f;
		if(PRECISE)
		{
			double sn, cs;
			sincospi((double) (long long) ph * 1.0842021724855044e-19, &sn, &cs);     // 2 / 2^64
			const double amp = 32767.999984741211 - (double) kq * 1.52587890625e-5;
			oi[j] += (min((int) floor(amp * cs), 32767) * level) >> 15;
			oq[j] += (min((int) floor(amp * sn), 32767) * level) >> 15;
		}
		else
		{
			const float amp = kl_amp(kq);
			float sn, cs;
			kl_sincos(ph, sn, cs);
			oi[j] += (__float2int_rd(amp * cs) * level) >> 15;
			oq[j] += (__float2int_rd(amp * sn) * level) >> 15;
		}
		phA += stA; phB += stB; kq += (float) S;
	}
}

// AM carrier: carrier phase phM and step ang per sample; amA / amB the level (sample + 32768) / 2 of the audio segment
// before / from sample nb (x0, nb as in kl_fm_each)
template<int S>
__device__ __forceinline__ void kl_am(unsigned long long phM, unsigned long long ang, int amA, int amB, int x0, int nb, float kf,
	const int &level, int (&oi)[4], int (&oq)[4])
{
	const unsigned long long stM = ang * S;
	float kq = kf;
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		if(kq > 32767.0f) kq -= 32767.0f;
		const float amp = kl_amp(kq);
		float sn, cs;
		kl_sincos(phM, sn, cs);
		const int smp = x0 + S * j >= nb ? amB : amA;
		oi[j] += (((__float2int_rd(amp * cs) * smp) >> 15) * level) >> 15;
		oq[j] += (((__float2int_rd(amp * sn) * smp) >> 15) * level) >> 15;
		phM += stM; kq += (float) S;
	}
}

// NICAM pulse-shaping table (htv_tables.c): one entry per sample and channel. (iA, qA) the index (I, Q) of the first
// sample under symbol A, (iB, qB) under symbol B, which is in effect from sample nb on (x0, nb as in kl_fm_each).
template<int S>
__device__ __forceinline__ void kl_nic_lut(const int16_t *lut, int iA, int qA, int iB, int qB, int x0, int nb, int (&bi)[4],
	int (&bq)[4])
{
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		const bool b = x0 + S * j >= nb;
		bi[j] = __ldg(lut + S * j + (b ? iB : iA));
		bq[j] = __ldg(lut + S * j + (b ? qB : qA));
	}
}

// one symbol of the generic NICAM sum (stream start, unusual rates): its pulse-table entry r with the polarities of its
// code sy; the pulse table holds the same integer sums (htv_tables.c), so the two forms agree wherever both apply
__device__ __forceinline__ void kl_nic_add(int sy, int r, int &bi, int &bq)
{
	bi += (sy & 1) ? r : -r;
	bq += (sy & 2) ? r : -r;
}

// NICAM: the pulse sums (bi, bq) times the carrier table from ccp (extended past its period, htv_tables.c: never wraps)
template<int S>
__device__ __forceinline__ void kl_nic_carrier(const htv_c16_t *ccp, const int (&bi)[4], const int (&bq)[4], int (&oi)[4], int (&oq)[4])
{
	#pragma unroll
	for(int j = 0; j < 4; j++)
	{
		const short2 cc = kl_ldc16(ccp + S * j);
		// the overlap-add ring holds at most 7 pulses of < 2^11: it never wraps an int16
		oi[j] += (bi[j] * cc.x - bq[j] * cc.y) >> 15;
		oq[j] += (bi[j] * cc.y + bq[j] * cc.x) >> 15;
	}
}

// Mixers after the modulation (ref video.c:3466-3515). Every addition before them is an int16 wrap-around addition in
// the reference. oi / oq stay unwrapped where only their low 16 bits reach the store; the mixer, which multiplies, wraps
// its inputs first.
__device__ __forceinline__ void kl_swap(int (&oi)[4], int (&oq)[4])
{
	#pragma unroll
	for(int j = 0; j < 4; j++) { const int t = oi[j]; oi[j] = oq[j]; oq[j] = t; }
}

// one sample of the frequency-offset mixer at audio-clock index m: its start-up table below m = 32767, then the phasor
// at the phase and amplitude that phasor(ph, kq) gives (evaluated only there)
template<typename P>
__device__ __forceinline__ void kl_offset(const DevTables &dt, long long m, P phasor, int &oi, int &oq)
{
	const int vi = wrap16i(oi), vq = wrap16i(oq);
	int bi, bq;
	if(m < 32767)
	{
		const unsigned char st = dt.offset_start[m];
		bi = -(st & 1); bq = -((st >> 1) & 1);
	}
	else
	{
		unsigned long long ph;
		float kq;
		phasor(ph, kq);
		const float amp = kl_amp(kq);
		float sn, cs;
		kl_sincos(ph, sn, cs);
		bi = min(__float2int_rd(amp * cs), 32767); bq = min(__float2int_rd(amp * sn), 32767);   // pi >> 16 <= 32767
	}
	oi = (vi * bi - vq * bq) >> 15;
	oq = (vi * bq + vq * bi) >> 15;
}

// ---- sound carriers for the four samples xb + S j of a thread, from the line's sound descriptor ------------------
// All four samples lie in the 32-sample block b = xb >> 5, for which the line descriptor lists the audio segment / NICAM
// symbol in effect at the block's first sample, and at most one boundary of either kind falls inside a block (an audio
// segment is rate / 32 kHz samples long; the host takes the generic NICAM sum at rates where a symbol is 32 samples or
// shorter).
// FM carrier, S = 8: the rotation form - unless an audio-segment boundary or a renormalisation of the reference's phasor
// falls between the samples; then the per-sample form. S = 1: the per-sample form, always (the rotation rounds
// differently).
template<int SND, int S, bool PRECISE = false>
__device__ __forceinline__ void kl_sound(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la,
	const short *ntp, int xb, int (&oi)[4], int (&oq)[4])
{
	const int b = xb >> 5;
	const bool fm = KL_HAS(SND, KL_FM, dp.have_fm), am = KL_HAS(SND, KL_AM, dp.have_am);
	if(fm || am)
	{
		const int sg = la->fm_blk[b];
		const int nb = la->seg_x[sg + 1];
		const int sg1 = min(sg + 1, MAX_SEGS - 1);
		int kk = la->kk0 + xb;
		if(kk >= 32767) kk -= 32767;
		const float kf = (float) (kk + 1);
		const bool mixed = S == 1 || (nb > xb && nb <= xb + 3 * S) || kk + 3 * S + 1 > 32767;
		if(fm)
		{
			if(!mixed)
			{
				const int s0 = xb >= nb ? sg1 : sg;
				kl_fm_rot<S>(la->seg_phase[s0] + la->seg_ang[s0] * (unsigned long long) xb, la->seg_rot[s0], kf, dp.fm_level, oi, oq);
			}
			else
			{
				const unsigned long long angA = la->seg_ang[sg], angB = la->seg_ang[sg1];
				kl_fm_each<S, PRECISE>(la->seg_phase[sg] + angA * (unsigned long long) xb, angA,
					la->seg_phase[sg1] + angB * (unsigned long long) xb, angB, xb, nb, kf, dp.fm_level, oi, oq,
					[&](int j, unsigned long long ph) {
						if(S > 1) return(ph);
						// the split kernels: each sample's phase straight from the descriptor, so that the two running
						// phases and their steps need no registers there
						const int sj = xb + j >= nb ? sg1 : sg;
						return(la->seg_phase[sj] + la->seg_ang[sj] * (unsigned long long) (xb + j));
					});
			}
		}
		if(am)
			kl_am<S>(la->am_phase0 + dp.am_ang * (unsigned long long) (xb + 1), dp.am_ang, (la->seg_am[sg] + 32768) / 2,
				(la->seg_am[sg1] + 32768) / 2, xb, nb, kf, dp.am_level, oi, oq);
	}

	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		int bi[4], bq[4];
		if(!la->nic_generic)
		{
			// pulse-table index = base + x
			const int ib = la->nic_blk[b];
			const uint2 cur = la->symb[ib], nxt = la->symb[ib + 1];
			kl_nic_lut<S>(dt.nicam_lut - KL_BIAS + xb, (int) (cur.x & 0xFFFFu), (int) (cur.x >> 16), (int) (nxt.x & 0xFFFFu),
				(int) (nxt.x >> 16), xb, (int) nxt.y, bi, bq);
		}
		else
		{
			// the symbols whose pulse covers the sample
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				const int x = xb + S * j;
				// the newest symbol started at or before x: from the one in effect at the block start (S = 1; k_line searches
				// from the line's first)
				int i3 = S == 1 ? la->nic_blk[b] : 0;
				const int ns = la->nsym;
				while(i3 + 1 < ns && (int) la->symb[i3 + 1].y <= x) i3++;
				bi[j] = 0; bq[j] = 0;
				for(int cnd = 0; cnd < NIC_CAND; cnd++)
				{
					const int i = i3 - cnd;
					if(i < 0) break;
					const int sy = la->symc[i];
					const int d0 = x - (int) la->symb[i].y + NIC_TPAD;      // the table is zero outside the pulse
					if(d0 < 0) continue;
					kl_nic_add(sy, ntp[d0], bi[j], bq[j]);
				}
			}
		}
		kl_nic_carrier<S>(dt.nicam_cc + la->cc0 + xb, bi, bq, oi, oq);
	}
}

// ---- the same carriers from a lane state ---------------------------------------------------------------------------
// The state of the carriers at the thread's first sample u = 0 (k_line: KlFeed, htv_line.cuh). A is the audio segment /
// NICAM symbol in effect at u = 0, B the next one; at most one boundary of either kind falls among the four samples.
struct KlLane {
	unsigned long long phA, angA, phB, angB;  // FM: phase at u = 0 in segment A / B, and per sample
	float2 rot;                               // FM: (cos, sin) of 8 angle steps of A
	int nb;                                   // B is in effect from u = nb on (> 0; > 3 S: on none of the samples)
	int kk;                                   // audio-clock index of u = 0, mod 32767
	unsigned long long phM;                   // AM: carrier phase at u = 0
	int amA, amB;                             // AM: (sample + 32768) / 2 of A and B
	int gen;                                  // NICAM: the generic sum instead of the pulse table
	int niA, nqA, niB, nqB;                   // NICAM: pulse-table index (I, Q) of u = 0 under symbol A / B
	int nbs;                                  // NICAM: B is in effect from u = nbs on
	int cc;                                   // NICAM: carrier-table index of u = 0
	long long m;                              // offset mixer: audio-clock index of u = 0 ...
	unsigned long long offph;                 // ... and the mixer's phase there
};

// the carriers from a lane state; nic_generic(bi, bq) gives the generic NICAM sum of the four samples (stream start,
// symbols without a pulse-table row, rates where a symbol is 32 samples or shorter). PART: 1 the FM and AM carriers
// (fields nb .. amB of L), 2 NICAM (gen .. cc), 3 both - k_line fills and runs the two parts one after the other, so
// that the state of only one of them is held at a time.
template<int SND, int S, bool PRECISE = false, int PART = 3, typename G>
__device__ __forceinline__ void kl_sound_lane(const htv_dparams_t &dp, const DevTables &dt, const KlLane &L, int (&oi)[4], int (&oq)[4],
	G nic_generic)
{
	const bool fm = (PART & 1) && KL_HAS(SND, KL_FM, dp.have_fm), am = (PART & 1) && KL_HAS(SND, KL_AM, dp.have_am);
	if(fm || am)
	{
		const float kf = (float) (L.kk + 1);
		const bool mixed = S == 1 || L.nb <= 3 * S || L.kk + 3 * S + 1 > 32767;
		if(fm)
		{
			if(!mixed) kl_fm_rot<S>(L.phA, L.rot, kf, dp.fm_level, oi, oq);
			else kl_fm_each<S, PRECISE>(L.phA, L.angA, L.phB, L.angB, 0, L.nb, kf, dp.fm_level, oi, oq,
				[](int, unsigned long long ph) { return(ph); });
		}
		if(am) kl_am<S>(L.phM, dp.am_ang, L.amA, L.amB, 0, L.nb, kf, dp.am_level, oi, oq);
	}

	if((PART & 2) && KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		int bi[4], bq[4];
		if(!L.gen) kl_nic_lut<S>(dt.nicam_lut, L.niA, L.nqA, L.niB, L.nqB, 0, L.nbs, bi, bq);
		else nic_generic(bi, bq);
		kl_nic_carrier<S>(dt.nicam_cc + L.cc, bi, bq, oi, oq);
	}
}

// ---- the mixers, from the line's sound descriptor or from a lane state --------------------------------------------
template<int SND, int S>
__device__ __forceinline__ void kl_mix(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la,
	int xb, int (&oi)[4], int (&oq)[4])
{
	if(KL_HAS(SND, KL_SWAP, dp.swap_iq)) kl_swap(oi, oq);
	if(KL_HAS(SND, KL_OFF, dp.have_offset))
	{
		const long long m0 = la->m0;
		const unsigned long long off0 = la->off_phase0;
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			const int x = xb + S * j;
			const long long m = m0 + x;
			kl_offset(dt, m, [&](unsigned long long &ph, float &kq) {
				kq = (float) ((int) (m % 32767) + 1);
				ph = off0 + dp.offset_ang * (unsigned long long) (x + 1);
			}, oi[j], oq[j]);
		}
	}
}

template<int SND, int S>
__device__ __forceinline__ void kl_mix_lane(const htv_dparams_t &dp, const DevTables &dt, const KlLane &L, int (&oi)[4], int (&oq)[4])
{
	if(KL_HAS(SND, KL_SWAP, dp.swap_iq)) kl_swap(oi, oq);
	if(KL_HAS(SND, KL_OFF, dp.have_offset))
	{
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			kl_offset(dt, L.m + S * j, [&](unsigned long long &ph, float &kq) {
				int kk = L.kk + S * j;
				if(kk >= 32767) kk -= 32767;
				kq = (float) (kk + 1);
				ph = L.offph + dp.offset_ang * (unsigned long long) (S * j);
			}, oi[j], oq[j]);
		}
	}
}
