// hacktv_b200 - the fused line kernel (included by htv_kernels.cu).
//
// One persistent CTA walks a run of consecutive scan lines and does, per line, everything between
// the picture in HBM and the int16 IQ in HBM - raster, chroma, video filter, sound carriers, mixers -
// without the composite signal ever leaving the SM:
//
//   R1  template (blank + sync pulses) + picture: RGB -> Y,U,V by table (ref video.c:2864-2992)
//   R2  chroma low-pass on the tensor cores, burst, subcarrier mix (ref video.c:3011-3040, fir.c:357-375),
//       VBI overlay; the finished composite line goes into a 3-row ring of byte planes in shared memory
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
// partial tile: the x < W tests fold away); CSAT: the chroma low-pass can leave the int16 range (sum of |taps| > 32768)
//
// Per iteration q (one scan line) a CTA runs
//   R1b(q)  picture values by table from the pixels fetched earlier, U / V byte planes        | __syncthreads (colour lines)
//   R2(q)   chroma low-pass (mma), burst, subcarrier, VBI overlay, composite row q mod 3       | __syncthreads
//   R1a(q+1) template + pixel loads of the NEXT line are issued here ...
//   M(q-1)  ... and arrive while line q - 1 (whose right-hand halo R2(q) has just written) is filtered (mma),
//           gets its sound carriers and is stored.
// The line descriptors (LineR2 of q + 1, LineA2 of q - 1) come in by cp.async at the top of the iteration.
//
// SRC: the composite lines are not rastered here but read from `src` (row q + 2 = relative line q, int16): SECAM, whose
// chrominance chain (htv_secam.cuh) runs between the raster and the modulator. R1b / R2 fold away, the rest is the same.
// WC: the line width compiled in (0: dp.W), so that the shared-memory row and plane offsets become immediates
// ST: the output sample type compiled into the store (HTV_TYPE_INT16: the int16 store), -1: dp.sample_type at run time
template<bool VF, bool HASQ, bool FULL, bool CSAT, int MAXT, int MINB, bool SRC = false, int SND = -1, int WC = 0, int ST = HTV_TYPE_INT16>
__global__ void __launch_bounds__(MAXT, MINB)
k_line(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineR2 *lrp, const LineA2 *lap,
	int nlines, int run, int16_t *out, const int16_t *acc, int acc_rows, const int16_t *src = nullptr)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = WC ? WC : dp.W;
	const int RB = kl_row_bytes(W), UB = kl_uv_bytes(W);
	// descriptors x2 | [row 0..2][hi, lo] composite planes | [u hi, u lo, v hi, v lo] | FIR taps | chroma taps | NICAM pulse
	LineA2 *sla = reinterpret_cast<LineA2 *>(smem_raw);
	LineR2 *slr = reinterpret_cast<LineR2 *>(sla + 2);
	unsigned char *rows = reinterpret_cast<unsigned char *>(slr + 2);
	unsigned char *uvp = rows + (VF ? 6 * RB : 0);
	uint4 *atab = reinterpret_cast<uint4 *>(uvp + 4 * UB);                 // [k-step][I hi, I lo, Q hi, Q lo][lane]
	uint4 *ctab = atab + (VF ? MF_ATAB_WORDS / 4 : 0);                      // [hi, lo][lane]
	short *ntp = reinterpret_cast<short *>(ctab + 64);
	const int tid = threadIdx.x, lane = tid & 31, nt = tid >> 5;
	const int g = lane >> 2, t = lane & 3;
	const int xb = mf_lane_x(nt, lane, 0);                                  // the lane's samples: xb + 8 j

	const int a = blockIdx.x * run, bnd = min(a + run, nlines);
	if(a >= nlines) return;
	// relative line q: raster lines a-1 .. bnd (descriptor lrp[q + 1]), modulate a .. bnd-1
	const int q0 = VF ? a - 1 : a, q1 = VF ? bnd : bnd - 1;

	// ---- one-time set-up -------------------------------------------------------
	if(VF) for(int i = tid; i < MF_ATAB_WORDS / 4; i += blockDim.x) atab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.mma_atab) + i);
	if(dt.chroma_atab) for(int i = tid; i < 64; i += blockDim.x) ctab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.chroma_atab) + i);
	for(int i = tid; i < ((VF ? 6 * RB : 0) + 4 * UB) / 4; i += blockDim.x) reinterpret_cast<unsigned *>(rows)[i] = 0;
	if(KL_HAS(SND, KL_NIC, dp.have_nicam))
	{
		const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
		int4 *dst = reinterpret_cast<int4 *>(ntp);
		for(int i = tid; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
	}
	if(!SRC && tid < 4) reinterpret_cast<int4 *>(slr + (q0 & 1))[tid] = __ldg(reinterpret_cast<const int4 *>(lrp + q0 + 1) + tid);
	__syncthreads();

	const int full_l = dp.active_left, full_r = dp.active_left + dp.active_width;
	const bool in_full = xb + 24 >= full_l && xb < full_r;                  // the lane touches the picture area at all
	const bool all_full = xb >= full_l && xb + 24 < full_r;                 // ... with all four samples
	const bool in_burst = xb + 24 >= dp.burst_left && xb < dp.burst_left + dp.burst_width;
	unsigned char *const uv0 = uvp + KL_UVLEAD + xb;                        // the lane's bytes in the four chroma planes
	const unsigned char *const uvb = uvp + mf_lp_b_offset(nt, lane);        // ... and its chroma B fragment
	const int fo0 = mf_b_offset(nt, 0, lane);
	constexpr int NA16 = (int) (sizeof(LineA2) / 16);

	// loads of line q issued one phase early: template (int16 x 4) and pixels (RGBx x 4)
	int tm[4];
	unsigned px[4];
	#define KL_R1A(QQ) do { \
		if(SRC) \
		{ \
			const int16_t *sp_ = src + (size_t) ((QQ) + 2) * W + xb; \
			_Pragma("unroll") for(int j = 0; j < 4; j++) tm[j] = (FULL || xb + 8 * j < W) ? (int) __ldg(sp_ + 8 * j) : 0; \
			px[0] = px[1] = px[2] = px[3] = 0u; \
			break; \
		} \
		const LineR2 &ln = slr[(QQ) & 1]; \
		const int16_t *tp_ = dt.tmpl_out + (size_t) ln.tmpl * W + xb; \
		_Pragma("unroll") for(int j = 0; j < 4; j++) tm[j] = (FULL || xb + 8 * j < W) ? (int) __ldg(tp_ + 8 * j) : 0; \
		if(in_full && ln.al < ln.ar && ln.row_off >= 0) \
		{ \
			const uint32_t *pp_ = dt.frames + ln.row_off + (xb - dp.active_left); \
			_Pragma("unroll") for(int j = 0; j < 4; j++) \
			{ \
				const int x_ = xb + 8 * j; \
				px[j] = (x_ >= ln.al && x_ < ln.ar) ? __ldg(pp_ + 8 * j) : 0u; \
			} \
		} \
		else { px[0] = px[1] = px[2] = px[3] = 0u; } \
	} while(0)
	KL_R1A(q0);

	int r3 = (q0 + 3) % 3;                                                  // ring row of line q
	for(int q = q0; q <= q1; q++, r3 = r3 == 2 ? 0 : r3 + 1)
	{
		const int mrow = VF ? q - 1 : q;                                    // the line modulated in this iteration
		// ---- descriptors of the next raster line and of the line modulated below -> shared memory -----
		if(tid < 4) { if(!SRC && q + 1 <= q1) kl_cp16(reinterpret_cast<int4 *>(slr + ((q + 1) & 1)) + tid, reinterpret_cast<const int4 *>(lrp + q + 2) + tid); }
		else if(tid < 4 + NA16) { if(mrow >= a) kl_cp16(reinterpret_cast<int4 *>(sla + (mrow & 1)) + (tid - 4), reinterpret_cast<const int4 *>(lap + mrow) + (tid - 4)); }

		// ---- R1b: picture values of line q ---------------------------------------
		const LineR2 &li = slr[q & 1];
		const int li_al = SRC ? 0 : li.al, li_ar = SRC ? 0 : li.ar, li_pal = SRC ? 0 : li.pal;
		int val[4] = { tm[0], tm[1], tm[2], tm[3] };
		int uu[4] = { 0, 0, 0, 0 }, vv[4] = { 0, 0, 0, 0 };
		if(in_full && li_al < li_ar)
		{
			if(xb >= li_al && xb + 24 < li_ar && !li.keep)
			{
				// all four samples in the picture
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const short4 e = __ldg(dt.yuv_lut + (px[j] & 0xFFFFFFu));
					val[j] = e.x; uu[j] = e.y; vv[j] = e.z;
				}
			}
			else
			{
				const int16_t *kp = dt.tmpl_keep + (size_t) li.tmpl * W + xb;
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int x = xb + 8 * j;
					if(x >= li_al && x < li_ar)
					{
						const short4 e = __ldg(dt.yuv_lut + (px[j] & 0xFFFFFFu));
						val[j] = e.x; uu[j] = e.y; vv[j] = e.z;
						if(li.keep) val[j] += __ldg(kp + 8 * j);
					}
				}
			}
		}
		if(li_pal)
		{
			// subcarrier table entries of this line: in flight across the barrier and the chroma filter
			short2 cl[4];
			{
				const htv_c16_t *cp = dt.clut + li.clut_off + xb;
				#pragma unroll
				for(int j = 0; j < 4; j++) cl[j] = (FULL || xb + 8 * j < W) ? kl_ldc16(cp + 8 * j) : make_short2(0, 0);
			}
			// unfiltered U, V as byte planes; outside the picture the planes stay zero (the reference filters
			// each line on its own: zero history either side, ref fir.c:357-375)
			if(all_full)
			{
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					uv0[8 * j] = (unsigned char) (uu[j] >> 8); uv0[UB + 8 * j] = (unsigned char) uu[j];
					uv0[2 * UB + 8 * j] = (unsigned char) (vv[j] >> 8); uv0[3 * UB + 8 * j] = (unsigned char) vv[j];
				}
			}
			else if(in_full)
			{
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int x = xb + 8 * j;
					if(x >= full_l && x < full_r)
					{
						uv0[8 * j] = (unsigned char) (uu[j] >> 8); uv0[UB + 8 * j] = (unsigned char) uu[j];
						uv0[2 * UB + 8 * j] = (unsigned char) (vv[j] >> 8); uv0[3 * UB + 8 * j] = (unsigned char) vv[j];
					}
				}
			}
			__syncthreads();
			// ---- R2: chroma low-pass (tensor cores), burst, subcarrier ---------------
			int cu[4], cv[4];
			{
				int uhh[4] = { 0, 0, 0, 0 }, umid[4] = { 0, 0, 0, 0 }, ull[4] = { 0, 0, 0, 0 };
				int vhh[4] = { 0, 0, 0, 0 }, vmid[4] = { 0, 0, 0, 0 }, vll[4] = { 0, 0, 0, 0 };
				const uint4 ah = ctab[lane], al4 = ctab[32 + lane];
				const uint2 uh = *reinterpret_cast<const uint2 *>(uvb), ul = *reinterpret_cast<const uint2 *>(uvb + UB);
				const uint2 vh = *reinterpret_cast<const uint2 *>(uvb + 2 * UB), vl = *reinterpret_cast<const uint2 *>(uvb + 3 * UB);
				mma_ss(uhh, ah, uh); mma_su(umid, ah, ul); mma_us(umid, al4, uh); mma_uu(ull, al4, ul);
				mma_ss(vhh, ah, vh); mma_su(vmid, ah, vl); mma_us(vmid, al4, vh); mma_uu(vll, al4, vl);
				// accumulator register ci <-> sample j: ci = ((j & 1) << 1) | (j >> 1)
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int ci = mf_lane_ci(j);
					cu[j] = kl_acc15(uhh[ci], umid[ci], ull[ci]);
					cv[j] = kl_acc15(vhh[ci], vmid[ci], vll[ci]);
					if(CSAT) { cu[j] = sat16i(cu[j]); cv[j] = sat16i(cv[j]); }
				}
			}
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
			#pragma unroll
			for(int j = 0; j < 4; j++) val[j] += ((int) cl[j].x * cv[j] * li_pal + (int) cl[j].y * cu[j]) >> 15;
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

		const int rprev = r3 == 0 ? 2 : r3 - 1, rnext = r3 == 2 ? 0 : r3 + 1;
		if(VF)
		{
			// ---- composite line -> ring row q mod 3 (+ the neighbours' halos) ----------
			unsigned char *rp = rows + (2 * r3) * RB + KL_LEAD + xb;
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
		if(tid < 4 + NA16) kl_cp_wait();
		__syncthreads();                                                    // rows of line q, descriptors of q + 1 and of mrow

		// ---- R1a: the next line's template and pixels start their way here -------------
		if(q + 1 <= q1) KL_R1A(q + 1);
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
			const LineA2 *la = sla + (mrow & 1);
			kl_sound<SND, 8>(dp, dt, la, ntp, xb, oi, oq);
			kl_post_store<FULL, SND, ST>(dp, dt, la, W, xb, mrow, oi, oq, out, mrow < acc_rows ? acc : NULL);
		}
	}
	#undef KL_R1A
}
