// hacktv_b200 - the fused line kernel (included by htv_kernels.cu).
//
// One persistent CTA walks a run of consecutive scan lines and does, per line, everything between
// the picture in HBM and the int16 IQ in HBM - raster, chroma, video filter, sound carriers, mixers -
// without the composite signal ever leaving the SM:
//
//   R1  the line's row of the converted picture store: template (blank + sync pulses) + Y, and U, V after the chroma
//       low-pass, converted once per picture when it arrived (k_picture, ref video.c:2864-2992, fir.c:357-375)
//   R2  burst, subcarrier mix (ref video.c:3011-3040), VBI overlay; the finished composite line goes into a 4-row ring
//       of byte planes in shared memory
//   M   51-tap VSB / low-pass video filter on the tensor cores (ref video.c:3235-3248, fir.c:564-615),
//       FM / AM / NICAM sound carriers (ref video.c:3261-3450, nicam728.c:342-411), IQ swap, offset
//       mixer (ref video.c:3466-3515), channel combiner, store.
//
// Thread <-> sample mapping: a warp owns one tile of 128 consecutive samples and every lane keeps its four
// samples in the layout the m16n8k32 accumulators have anyway: lane = 4g + t holds x = 128 tile + 32 t + g + 8 j,
// j = 0..3 (htv_mma_fir.h: mf_out_x). Both filters leave their results in exactly the registers the next
// stage needs - no exchange through shared memory, and all four samples of a lane fall into one 32-sample
// block, which is what the per-line sound descriptors are indexed by: the sound carriers and mixers are htv_sound.cuh's
// with S = 8. Loads and stores with a stride of 8 samples between a lane's values are still sector-exact (8 lanes x 4
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

// Mixers after the modulation (htv_sound.cuh), channel combiner, store in the strided layout.
// ST: the sample type the store converts to (htv_sample_type.h), -1 for dp.sample_type at run time. The channel combiner
// (`acc`, int16 in the output layout) still adds in int16 with wrap-around; the conversion is the last step, as the
// reference's file sink converts what the video stage handed it. A lane stores each of its samples on its own (1, 2,
// 4 or 8 bytes); the eight lanes g = 0..7 of a t still cover one contiguous run of the line per j.
template<bool FULL, int SND, int ST>
__device__ __forceinline__ void kl_post_store(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la,
	int W, int xb, int row, int (&oi)[4], int (&oq)[4], int16_t *out, const int16_t *acc)
{
	kl_mix<SND, 8>(dp, dt, la, xb, oi, oq);
	const size_t lbase = (size_t) row * (size_t) W;
	if constexpr(ST != HTV_TYPE_INT16)
	{
		const int st = ST < 0 ? dp.sample_type : ST;
		const bool cpx = KL_HAS(SND, KL_CPX, dp.complex_out);
		#pragma unroll
		for(int j = 0; j < 4; j++)
		{
			if(FULL || xb + 8 * j < W)
			{
				const size_t s = lbase + xb + 8 * j;
				if(cpx) htv_st_put2(out, s, st, wrap16i(oi[j] + (acc ? acc[2 * s] : 0)), wrap16i(oq[j] + (acc ? acc[2 * s + 1] : 0)));
				else htv_st_put(out, s, st, wrap16i(oi[j] + (acc ? acc[s] : 0)));
			}
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

// cp.async: 16 bytes global -> shared without passing through registers
__device__ __forceinline__ void kl_cp16(void *dst_smem, const void *src)
{
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void kl_cp_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// VF: a video filter is on (composite ring + tensor-core FIR); HASQ: it has Q taps (VSB); FULL: 128 | W (no
// partial tile: the x < W tests fold away); CSAT: the chroma low-pass can leave the int16 range (sum of |taps| > 32768),
// which k_picture's saturating low-pass handles when it fills the store: the CSAT forms run the same code as the others
//
// Per iteration q (one scan line) a CTA runs
//   R2(q)   burst, subcarrier, VBI overlay on the values fetched earlier, composite row q mod 4  | __syncthreads
//   R1(q+1) the converted row of the NEXT line (values, and filtered U / V on colour lines) is loaded here ...
//   M(q-1)  ... and arrive while line q - 1 (whose right-hand halo R2(q) has just written) is filtered (mma),
//           gets its sound carriers and is stored.
// The line descriptors (LineR2 of q + 1, LineA2 of q - 1) come in by cp.async at the top of the iteration.
// One barrier per line, so the ring has 4 rows: a warp that is through M(q - 1) may run on into R2(q + 1), before the
// next barrier, while another warp is still reading line q - 1's row. R2(q + 1) writes line q + 1's row, the right
// halo of line q's and the left halo of line q + 2's; with 4 rows none of them is line q - 1's.
//
// SRC: the composite lines are not rastered here but read from `src` (row q + 2 = relative line q, int16): SECAM, whose
// chrominance chain (htv_secam.cuh) runs between the raster and the modulator. R2 folds away, the rest is the same.
// WC: the line width compiled in (0: dp.W), so that the shared-memory row and plane offsets become immediates
// ST: the output sample type compiled into the store (HTV_TYPE_INT16: the int16 store), -1: dp.sample_type at run time
//
// S-Video (KL_SV, dp.s_video; ref video.c:3031-3040, 3206-3228): the subcarrier term of R2 goes to Q instead of I, and the
// video filter runs on I only, so Q of the stored line is that line's own chroma. R2 parks it in a two-row ring in shared
// memory at the lane's own slots (row q & 1), M takes it back for mrow: no other thread touches the slots, so no barrier
// orders them, and nothing stays live in registers across the loop. SRC: the chain wrote Q into its own plane, `srcq`.
template<bool VF, bool HASQ, bool FULL, bool CSAT, int MAXT, int MINB, bool SRC = false, int SND = -1, int WC = 0, int ST = HTV_TYPE_INT16>
__global__ void __launch_bounds__(MAXT, MINB)
k_line(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineR2 *lrp, const LineA2 *lap,
	int nlines, int run, int16_t *out, const int16_t *acc, int acc_rows, const int16_t *src = nullptr, const int16_t *srcq = nullptr)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = WC ? WC : dp.W;
	const int RB = kl_row_bytes(W);
	// descriptors x2 | [row 0..3][hi, lo] composite planes | FIR taps | NICAM pulse | S-Video chroma [row 0..1][j][thread]
	LineA2 *sla = reinterpret_cast<LineA2 *>(smem_raw);
	LineR2 *slr = reinterpret_cast<LineR2 *>(sla + 2);
	unsigned char *rows = reinterpret_cast<unsigned char *>(slr + 2);
	uint4 *atab = reinterpret_cast<uint4 *>(rows + (VF ? 8 * RB : 0));    // [k-step][I hi, I lo, Q hi, Q lo][lane]
	short *ntp = reinterpret_cast<short *>(atab + (VF ? MF_ATAB_WORDS / 4 : 0));
	const int tid = threadIdx.x, lane = tid & 31, nt = tid >> 5;
	const int g = lane >> 2, t = lane & 3;
	const int xb = mf_lane_x(nt, lane, 0);                                  // the lane's samples: xb + 8 j
	const bool sv = KL_HAS(SND, KL_SV, dp.s_video);
	short *const svq = ntp + ((dp.nicam_tpad_len + 7) & ~7);

	const int a = blockIdx.x * run, bnd = min(a + run, nlines);
	if(a >= nlines) return;
	// relative line q: raster lines a-1 .. bnd (descriptor lrp[q + 1]), modulate a .. bnd-1
	const int q0 = VF ? a - 1 : a, q1 = VF ? bnd : bnd - 1;

	// ---- one-time set-up -------------------------------------------------------
	if(VF) for(int i = tid; i < MF_ATAB_WORDS / 4; i += blockDim.x) atab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.mma_atab) + i);
	if(VF) for(int i = tid; i < 8 * RB / 4; i += blockDim.x) reinterpret_cast<unsigned *>(rows)[i] = 0;
	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
		int4 *dst = reinterpret_cast<int4 *>(ntp);
		for(int i = tid; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
	}
	if(!SRC && tid < 4) reinterpret_cast<int4 *>(slr + (q0 & 1))[tid] = __ldg(reinterpret_cast<const int4 *>(lrp + q0 + 1) + tid);
	__syncthreads();

	// the span the chroma low-pass reaches (taps <= 17: 8 samples either side of the picture); the store is zero outside
	const bool in_chroma = xb + 24 >= dp.active_left - 8 && xb < dp.active_left + dp.active_width + 8;
	const bool in_burst = xb + 24 >= dp.burst_left && xb < dp.burst_left + dp.burst_width;
	const int fo0 = mf_b_offset(nt, 0, lane);
	constexpr int NA16 = (int) (sizeof(LineA2) / 16);

	// loads of line q issued one phase early: line values (int16 x 4) and, on colour lines, filtered U | V << 16 (x 4)
	int tm[4];
	unsigned px[4];
	#define KL_R1(QQ) do { \
		if(SRC) \
		{ \
			const int16_t *sp_ = src + (size_t) ((QQ) + 2) * W + xb; \
			_Pragma("unroll") for(int j = 0; j < 4; j++) tm[j] = (FULL || xb + 8 * j < W) ? (int) __ldg(sp_ + 8 * j) : 0; \
			px[0] = px[1] = px[2] = px[3] = 0u; \
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
		const int mrow = VF ? q - 1 : q;                                    // the line modulated in this iteration
		// ---- descriptors of the next raster line and of the line modulated below -> shared memory -----
		if(tid < 4) { if(!SRC && q + 1 <= q1) kl_cp16(reinterpret_cast<int4 *>(slr + ((q + 1) & 1)) + tid, reinterpret_cast<const int4 *>(lrp + q + 2) + tid); }
		else if(tid < 4 + NA16) { if(mrow >= a) kl_cp16(reinterpret_cast<int4 *>(sla + (mrow & 1)) + (tid - 4), reinterpret_cast<const int4 *>(lap + mrow) + (tid - 4)); }
		// a CTA narrower than 4 + NA16 threads (one warp: W <= 128) copies the rest of the descriptor in further passes;
		// the forms with the width compiled in have 256 threads and need none
		if(!WC && (int) blockDim.x < 4 + NA16 && mrow >= a)
			for(int i = (int) blockDim.x - 4 + tid; i < NA16; i += blockDim.x)
				kl_cp16(reinterpret_cast<int4 *>(sla + (mrow & 1)) + i, reinterpret_cast<const int4 *>(lap + mrow) + i);

		// ---- R2: burst, subcarrier, VBI overlay of line q ---------------------------
		const LineR2 &li = slr[q & 1];
		const int li_pal = SRC ? 0 : li.pal;
		int val[4] = { tm[0], tm[1], tm[2], tm[3] };
		int cq[4] = { 0, 0, 0, 0 };                                         // S-Video: the chroma of line q
		if(li_pal)
		{
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
		if(!SRC && sv)
		{
			#pragma unroll
			for(int j = 0; j < 4; j++) svq[((q & 1) * 4 + j) * blockDim.x + tid] = (short) cq[j];
		}
		if(!SRC && li.ov_any)
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
		if(VF)
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
		if(tid < 4 + NA16 || (!WC && (int) blockDim.x < 4 + NA16)) kl_cp_wait();
		__syncthreads();                                                    // rows of line q, descriptors of q + 1 and of mrow

		// ---- R1: the next line's values start their way here -------------------------
		if(q + 1 <= q1) KL_R1(q + 1);
		if(mrow < a) continue;

		int oi[4], oq[4];
		if(VF)
		{
			// ---- M: video filter of line q - 1, one tile of 128 samples per warp -------
			const unsigned char *ph = rows + (2 * rprev) * RB + fo0, *plo = ph + RB;
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
		else
		{
			#pragma unroll
			for(int j = 0; j < 4; j++) { oi[j] = wrap16i(val[j]); oq[j] = 0; }
		}

		// ---- sound carriers, mixers, store ---------------------------------------
		if(FULL || xb < W)
		{
			if(sv)
			{
				// Q = the chroma of line mrow (the video filter leaves it alone)
				const int16_t *qp = srcq + (size_t) (mrow + 2) * W + xb;
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					if(SRC) oq[j] += (FULL || xb + 8 * j < W) ? (int) __ldg(qp + 8 * j) : 0;
					else oq[j] += svq[((mrow & 1) * 4 + j) * blockDim.x + tid];
				}
			}
			const LineA2 *la = sla + (mrow & 1);
			kl_sound<SND, 8>(dp, dt, la, ntp, xb, oi, oq);
			kl_post_store<FULL, SND, ST>(dp, dt, la, W, xb, mrow, oi, oq, out, mrow < acc_rows ? acc : NULL);
		}
	}
	#undef KL_R1
}
