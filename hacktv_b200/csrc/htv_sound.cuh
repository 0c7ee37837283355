// hacktv_b200 - the sound carriers and the post-modulation mixers (included by htv_kernels.cu), for the fused line kernel
// (htv_line.cuh) and for the split and FM-video modulators alike. Both read the per-line sound descriptor LineA2
// (k_line_desc_a2) and work on four samples per thread, S apart:
//   S = 8: k_line's lane layout (x = xb + 8 j, the m16n8k32 accumulator layout, htv_mma_fir.h: mf_out_x);
//   S = 1: four consecutive samples (k_mod, k_mod_tma, k_mod_mma, k_fmv_base, k_fmv_mod).
// Either way all four samples fall into one 32-sample block, which is what the descriptor is indexed by.

#define KL_BIAS   2048      // NICAM pulse-table index bias (LineA2.symb)

// one complex int16 table entry through the read-only path: x = i, y = q
__device__ __forceinline__ short2 kl_ldc16(const htv_c16_t *p) { return(__ldg(reinterpret_cast<const short2 *>(p))); }

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
#define KL_SND_FM_NICAM (KL_FM | KL_NIC | KL_CPX)
#define KL_HAS(SND, BIT, RT) ((SND) < 0 ? (RT) != 0 : ((SND) & (BIT)) != 0)

static inline int kl_snd_mask(const htv_dparams_t &dp)
{
	return((dp.have_fm ? KL_FM : 0) | (dp.have_am ? KL_AM : 0) | (dp.have_nicam ? KL_NIC : 0) |
		(dp.have_offset ? KL_OFF : 0) | (dp.swap_iq ? KL_SWAP : 0) | (dp.complex_out ? KL_CPX : 0));
}

// ---- sound carriers for the four samples xb + S j of a thread, added into oi / oq -------------------------------
// (ref video.c:3261-3450, nicam728.c:342-411). All four samples lie in the 32-sample block b = xb >> 5, for which the
// line descriptor lists the audio segment / NICAM symbol in effect at the block's first sample, and at most one
// boundary of either kind falls inside a block (an audio segment is rate / 32 kHz samples long; the host takes the
// generic NICAM sum at rates where a symbol is 32 samples or shorter).
// FM carrier, S = 8: one sin/cos for the first sample, the other three by rotating with the segment's (cos, sin) of 8
// angle steps - unless an audio-segment boundary or a renormalisation of the reference's phasor (every 32 767 samples)
// falls between the samples; then every sample gets its own. S = 1: every sample gets its own sin/cos, always (the
// rotation rounds differently).
// PRECISE (FM video only): the FM carrier in fp64 from the full 64-bit phase. An FM modulator integrates its input, so a
// sound-carrier sample that is 1 LSB off turns everything after it; the fast fp32 evaluation loses the sign of a carrier
// sample that lands on a zero crossing (an unmodulated 6.5 MHz carrier at 20 Msps does so every 40 samples).
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
		// amplitude of the reference's Q31 phasor kk + 1 multiplications after a renormalisation
		const float kf = (float) (kk + 1);
		const bool mixed = S == 1 || (nb > xb && nb <= xb + 3 * S) || kk + 3 * S + 1 > 32767;
		if(fm)
		{
			if(!mixed)
			{
				const int s0 = xb >= nb ? sg1 : sg;
				const unsigned long long ph = la->seg_phase[s0] + la->seg_ang[s0] * (unsigned long long) xb;
				const float2 rot = la->seg_rot[s0];
				float sn, cs;
				__sincosf((float) (int) (ph >> 32) * 1.4629180792671596e-9f, &sn, &cs);   // pi / 2^31
				float amp = 32767.99998f - kf * 1.52587890625e-5f;
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					oi[j] += (__float2int_rd(amp * cs) * dp.fm_level) >> 15;
					oq[j] += (__float2int_rd(amp * sn) * dp.fm_level) >> 15;
					const float c2 = __fmaf_rn(cs, rot.x, -(sn * rot.y)), s2 = __fmaf_rn(sn, rot.x, cs * rot.y);
					cs = c2; sn = s2;
					amp -= (float) S * 1.52587890625e-5f;
				}
			}
			else
			{
				const unsigned long long angA = la->seg_ang[sg], angB = la->seg_ang[sg1];
				unsigned long long phA = la->seg_phase[sg] + angA * (unsigned long long) xb;
				unsigned long long phB = la->seg_phase[sg1] + angB * (unsigned long long) xb;
				const unsigned long long stA = angA * S, stB = angB * S;
				float kq = kf;
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					unsigned long long ph = xb + S * j >= nb ? phB : phA;
					if(S == 1)
					{
						// the split kernels: each sample's phase straight from the descriptor, so that the two running
						// phases and their steps need no registers there
						const int sj = xb + j >= nb ? sg1 : sg;
						ph = la->seg_phase[sj] + la->seg_ang[sj] * (unsigned long long) (xb + j);
					}
					if(kq > 32767.0f) kq -= 32767.0f;
					if(PRECISE)
					{
						double sn, cs;
						sincospi((double) (long long) ph * 1.0842021724855044e-19, &sn, &cs);     // 2 / 2^64
						const double amp = 32767.999984741211 - (double) kq * 1.52587890625e-5;
						oi[j] += (min((int) floor(amp * cs), 32767) * dp.fm_level) >> 15;
						oq[j] += (min((int) floor(amp * sn), 32767) * dp.fm_level) >> 15;
					}
					else
					{
						const float amp = 32767.99998f - kq * 1.52587890625e-5f;
						float sn, cs;
						__sincosf((float) (int) (ph >> 32) * 1.4629180792671596e-9f, &sn, &cs);
						oi[j] += (__float2int_rd(amp * cs) * dp.fm_level) >> 15;
						oq[j] += (__float2int_rd(amp * sn) * dp.fm_level) >> 15;
					}
					phA += stA; phB += stB; kq += (float) S;
				}
			}
		}
		if(am)
		{
			unsigned long long phM = la->am_phase0 + dp.am_ang * (unsigned long long) (xb + 1);
			const unsigned long long stM = dp.am_ang * S;
			const int amA = (la->seg_am[sg] + 32768) / 2, amB = (la->seg_am[sg1] + 32768) / 2;
			float kq = kf;
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				if(kq > 32767.0f) kq -= 32767.0f;
				const float amp = 32767.99998f - kq * 1.52587890625e-5f;
				float sn, cs;
				__sincosf((float) (int) (phM >> 32) * 1.4629180792671596e-9f, &sn, &cs);
				const int smp = xb + S * j >= nb ? amB : amA;
				oi[j] += (((__float2int_rd(amp * cs) * smp) >> 15) * dp.am_level) >> 15;
				oq[j] += (((__float2int_rd(amp * sn) * smp) >> 15) * dp.am_level) >> 15;
				phM += stM; kq += (float) S;
			}
		}
	}

	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		int bi[4], bq[4];
		if(!la->nic_generic)
		{
			// pulse-shaping table (htv_tables.c): one entry per sample and channel, index = base + x
			const int ib = la->nic_blk[b];
			const uint2 cur = la->symb[ib], nxt = la->symb[ib + 1];
			const int nb = (int) nxt.y;
			const int16_t *lut = dt.nicam_lut - KL_BIAS + xb;
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				const unsigned w = xb + S * j >= nb ? nxt.x : cur.x;
				bi[j] = __ldg(lut + S * j + (w & 0xFFFFu));
				bq[j] = __ldg(lut + S * j + (w >> 16));
			}
		}
		else
		{
			// generic sum over the symbols whose pulse covers the sample (stream start, unusual rates); the pulse table
			// holds the same integer sums (htv_tables.c), so the two forms agree wherever both apply
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
					const int r = ntp[d0];
					bi[j] += (sy & 1) ? r : -r;
					bq[j] += (sy & 2) ? r : -r;
				}
			}
		}
		// carrier table extended past its period (htv_tables.c): cc0 + x never wraps
		const htv_c16_t *ccp = dt.nicam_cc + la->cc0 + xb;
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			const short2 cc = kl_ldc16(ccp + S * j);
			// the overlap-add ring holds at most 7 pulses of < 2^11: it never wraps an int16
			oi[j] += (bi[j] * cc.x - bq[j] * cc.y) >> 15;
			oq[j] += (bi[j] * cc.y + bq[j] * cc.x) >> 15;
		}
	}
}

// ---- mixers after the modulation (ref video.c:3466-3515): IQ swap, frequency-offset mixer --------------------------
// Every addition before them is an int16 wrap-around addition in the reference. oi / oq stay unwrapped where only their
// low 16 bits reach the store; the mixer, which multiplies, wraps its inputs first.
template<int SND, int S>
__device__ __forceinline__ void kl_mix(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la,
	int xb, int (&oi)[4], int (&oq)[4])
{
	if(KL_HAS(SND, KL_SWAP, dp.swap_iq))
	{
		#pragma unroll
		for(int j = 0; j < 4; j++) { const int t = oi[j]; oi[j] = oq[j]; oq[j] = t; }
	}
	if(KL_HAS(SND, KL_OFF, dp.have_offset))
	{
		const long long m0 = la->m0;
		const unsigned long long off0 = la->off_phase0;
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			const int x = xb + S * j;
			const long long m = m0 + x;
			const int vi = wrap16i(oi[j]), vq = wrap16i(oq[j]);
			int bi, bq;
			if(m < 32767)
			{
				const unsigned char st = dt.offset_start[m];
				bi = -(st & 1); bq = -((st >> 1) & 1);
			}
			else
			{
				const int kk = (int) (m % 32767);
				const float amp = 32767.99998f - (float) (kk + 1) * 1.52587890625e-5f;
				const unsigned long long ph = off0 + dp.offset_ang * (unsigned long long) (x + 1);
				float sn, cs;
				__sincosf((float) (int) (ph >> 32) * 1.4629180792671596e-9f, &sn, &cs);
				bi = min(__float2int_rd(amp * cs), 32767); bq = min(__float2int_rd(amp * sn), 32767);   // pi >> 16 <= 32767
			}
			oi[j] = (vi * bi - vq * bq) >> 15;
			oq[j] = (vi * bq + vq * bi) >> 15;
		}
	}
}
