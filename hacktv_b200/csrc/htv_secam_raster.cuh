// SECAM raster in the fused line kernel's form (included by htv_kernels.cu behind htv_line.cuh).
//
// What k_raster_secam does one CTA per line and one thread per 4 consecutive samples - luma from template + picture,
// the colour-difference baseband averaged with the line above (ref video.c:3093-3147), the 51-tap luma notch over the
// picture (ref video.c:3082-3090) and the 15-tap baseband low-pass (ref video.c:3162-3180) - a persistent CTA does here
// for a run of lines in k_line's lane layout (lane (g, t) of warp nt owns samples 128 nt + 32 t + g + 8 j): both
// filters are byte-split int8 contractions on the tensor cores whose
// accumulators land on the lane's own four samples, the next line's template and pixels are fetched while this line's
// filters run, and there is one barrier per line (byte planes double-buffered). Lines do not depend on each other.
// Outputs as before: composite rows (int16, luma only - k_sec_out adds the subcarrier), the baseband in the chain's
// transposed layout, the raw sums of the last 7 low-pass outputs. S-Video (dp.s_video) skips the notch (ref video.c:3206).

template<bool FULL, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB)
k_sec_raster(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *ls, int nrows, int run, int16_t *comp, SecScratch ss)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W;
	const int RB = kl_row_bytes(W), UB = kl_uv_bytes(W);
	// descriptors x2 | luma planes [buffer][hi, lo] | baseband planes [buffer][hi, lo] | notch taps | low-pass taps
	LineS2 *sl = reinterpret_cast<LineS2 *>(smem_raw);
	unsigned char *lum = reinterpret_cast<unsigned char *>(sl + 2);
	unsigned char *cbp = lum + 4 * RB;
	uint4 *ntab = reinterpret_cast<uint4 *>(cbp + 4 * UB);                   // [k-step][hi, lo][lane]
	uint4 *ctab = ntab + MF_KSTEPS * 2 * 32;                                // [hi, lo][lane]
	const int tid = threadIdx.x, lane = tid & 31, nt = tid >> 5;
	const int g = lane >> 2, t = lane & 3;
	const int xb = mf_lane_x(nt, lane, 0);                                  // the lane's samples: xb + 8 j

	const int a = blockIdx.x * run, bnd = min(a + run, nrows);
	if(a >= nrows) return;

	for(int i = tid; i < MF_KSTEPS * 2 * 32; i += blockDim.x) ntab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.notch_atab) + i);
	for(int i = tid; i < 64; i += blockDim.x) ctab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.sec_lpf_atab) + i);
	for(int i = tid; i < (4 * RB + 4 * UB) / 4; i += blockDim.x) reinterpret_cast<unsigned *>(lum)[i] = 0;
	if(tid < 4) reinterpret_cast<int4 *>(sl + (a & 1))[tid] = __ldg(reinterpret_cast<const int4 *>(ls + a) + tid);
	__syncthreads();

	const int a0 = dp.active_left, a1 = dp.active_left + dp.active_width;
	const bool in_pic = xb + 24 >= a0 && xb < a1;                           // the lane touches the picture area at all
	const int fo0 = mf_b_offset(nt, 0, lane);
	const int uo0 = mf_lp_b_offset(nt, lane);
	const bool notch_tile = MF_TILE * nt < a1 && MF_TILE * (nt + 1) > a0;

	// loads of a row issued one phase early: template (int16 x 4), this line's pixels and the stored line's (RGBx x 4)
	int tm[4];
	unsigned px[4], px2[4];
	#define KS_R1A(RR) do { \
		const LineS2 &ln = sl[(RR) & 1]; \
		const int16_t *tp_ = dt.tmpl_out + (size_t) ln.tmpl * W + xb; \
		_Pragma("unroll") for(int j = 0; j < 4; j++) tm[j] = (FULL || xb + 8 * j < W) ? (int) __ldg(tp_ + 8 * j) : 0; \
		px[0] = px[1] = px[2] = px[3] = 0u; px2[0] = px2[1] = px2[2] = px2[3] = 0u; \
		if(in_pic && ln.row_off >= 0 && (ln.sec_proc || ln.al < ln.ar)) \
		{ \
			const uint32_t *pp_ = dt.frames + ln.row_off + (xb - a0); \
			_Pragma("unroll") for(int j = 0; j < 4; j++) \
			{ \
				const int x_ = xb + 8 * j; \
				if(x_ >= a0 && x_ < a1) px[j] = __ldg(pp_ + 8 * j); \
			} \
		} \
		if(in_pic && ln.sec_proc && ln.sec_prev_kind == 2) \
		{ \
			const uint32_t *pp_ = dt.frames + ln.sec_prev_row + (xb - a0); \
			_Pragma("unroll") for(int j = 0; j < 4; j++) \
			{ \
				const int x_ = xb + 8 * j; \
				if(x_ >= a0 && x_ < a1) px2[j] = __ldg(pp_ + 8 * j); \
			} \
		} \
	} while(0)
	KS_R1A(a);

	for(int r = a; r < bnd; r++)
	{
		const int b = r & 1;
		if(tid < 4 && r + 1 < bnd) kl_cp16(reinterpret_cast<int4 *>(sl + ((r + 1) & 1)) + tid, reinterpret_cast<const int4 *>(ls + r + 1) + tid);
		const LineS2 &li = sl[b];
		const int li_al = li.al, li_ar = li.ar, proc = li.sec_proc;
		const int cur = li.sec_dr ? 2 : 1;                                  // 1: u, 2: v
		const int cb_black = cur == 1 ? dp.black_u : dp.black_v;

		// ---- luma and colour-difference baseband of the lane's four samples ----------
		int val[4] = { tm[0], tm[1], tm[2], tm[3] };
		int cbv[4] = { cb_black, cb_black, cb_black, cb_black };
		if(in_pic && (proc || li_al < li_ar))
		{
			const int16_t *kp = dt.tmpl_keep + (size_t) li.tmpl * W + xb;
			int st_c = 0;                                                   // the store holds zeros ...
			if(li.sec_prev_kind == 1) st_c = li.sec_prev_comp == 1 ? dp.black_u : dp.black_v;   // ... or black
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				const int x = xb + 8 * j;
				const bool inpic = x >= a0 && x < a1, act = x >= li_al && x < li_ar;
				if(!(act || (proc && inpic))) continue;
				const short4 e = __ldg(dt.yuv_lut + (px[j] & 0xFFFFFFu));
				if(act)
				{
					val[j] = e.x;
					if(li.keep) val[j] += __ldg(kp + 8 * j);
				}
				if(proc && inpic)
				{
					// average with what the previous line left in the store (C division: toward zero)
					int st = st_c;
					if(li.sec_prev_kind == 2)
					{
						const short4 e2 = __ldg(dt.yuv_lut + (px2[j] & 0xFFFFFFu));
						st = li.sec_prev_comp == 1 ? e2.y : e2.z;
					}
					cbv[j] = ((cur == 1 ? e.y : e.z) + st) / 2;
				}
			}
		}
		int lv[4];
		#pragma unroll
		for(int j = 0; j < 4; j++) lv[j] = wrap16i(val[j]);
		if(proc)
		{
			// byte planes: luma for the notch (samples left of the picture read as zero, ref fir.c:357-375), baseband for the low-pass
			unsigned char *rp = lum + (2 * b) * RB + KL_LEAD + xb;
			unsigned char *up = cbp + (2 * b) * UB + KL_UVLEAD + xb;
			#pragma unroll
			for(int j = 0; j < 4; j++)
			{
				if(FULL || xb + 8 * j < W)
				{
					const int nv = xb + 8 * j >= a0 ? lv[j] : 0;
					rp[8 * j] = (unsigned char) (nv >> 8); rp[RB + 8 * j] = (unsigned char) nv;
					up[8 * j] = (unsigned char) (cbv[j] >> 8); up[UB + 8 * j] = (unsigned char) cbv[j];
				}
			}
		}
		if(tid < 4) kl_cp_wait();
		__syncthreads();                                                    // planes of row r, descriptor of row r + 1

		if(r + 1 < bnd) KS_R1A(r + 1);

		if(proc)
		{
			if(notch_tile && !dp.s_video)
			{
				// ---- luma notch over the picture: 51 taps, three k-steps of 32 ----------
				const unsigned char *ph = lum + (2 * b) * RB + fo0, *plo = ph + RB;
				int hh[4] = { 0, 0, 0, 0 }, mid[4] = { 0, 0, 0, 0 }, ll[4] = { 0, 0, 0, 0 };
				#pragma unroll
				for(int s = 0; s < MF_KSTEPS; s++)
				{
					const uint2 xh = *reinterpret_cast<const uint2 *>(ph + 32 * s);
					const uint2 xl = *reinterpret_cast<const uint2 *>(plo + 32 * s);
					const uint4 ah = ntab[(s * 2 + 0) * 32 + lane], al = ntab[(s * 2 + 1) * 32 + lane];
					mma_ss(hh, ah, xh); mma_su(mid, ah, xl); mma_us(mid, al, xh); mma_uu(ll, al, xl);
				}
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int ci = mf_lane_ci(j), x = xb + 8 * j;
					if(x >= a0 && x < a1) lv[j] = kl_fir_out(hh[ci], mid[ci], ll[ci]);
				}
			}
			// ---- 15-tap low-pass of the baseband: one k-step; the two aliased words past the end of the line are added
			// by the chain (sec_tail), so the last 7 outputs are also kept as raw sums ----------
			{
				const unsigned char *uvb = cbp + (2 * b) * UB + uo0;
				int hh[4] = { 0, 0, 0, 0 }, mid[4] = { 0, 0, 0, 0 }, ll[4] = { 0, 0, 0, 0 };
				const uint4 ah = ctab[lane], al = ctab[32 + lane];
				const uint2 uh = *reinterpret_cast<const uint2 *>(uvb), ul = *reinterpret_cast<const uint2 *>(uvb + UB);
				mma_ss(hh, ah, uh); mma_su(mid, ah, ul); mma_us(mid, al, uh); mma_uu(ll, al, ul);
				#pragma unroll
				for(int j = 0; j < 4; j++)
				{
					const int ci = mf_lane_ci(j), x = xb + 8 * j;
					if(!FULL && x >= W) continue;
					const int raw = mf_combine(hh[ci], mid[ci], ll[ci]);
					ss.cbT[(((size_t) (x >> 3) * ss.rows + r) << 3) + (x & 7)] = (int16_t) sat16i(raw >> 15);
					if(x >= W - 7) ss.tail[(size_t) r * SEC_TAIL + (x - (W - 7))] = raw;
				}
			}
		}
		{
			int16_t *cp = comp + (size_t) r * W + xb;
			#pragma unroll
			for(int j = 0; j < 4; j++) if(FULL || xb + 8 * j < W) cp[8 * j] = (int16_t) lv[j];
		}
	}
	#undef KS_R1A
}
