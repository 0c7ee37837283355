// SECAM chrominance chain (ref video.c:3068-3233, fir.c:721-735), line-parallel. Included by htv_kernels.cu.
//
// The sample-serial parts of a line - the fp64 pre-emphasis IIR and the Q31 FM phasor recurrence - are run by ONE
// THREAD PER LINE, all lines of the launch at once, from the state their predecessor produced in the previous pass
// (pass 0: a guess); passes repeat until no line's input differs bitwise from its predecessor's output, i.e. until
// the sequential result is reached. Three things keep that to one full pass plus a sliver:
//   - only the recurrences live in the chain threads: the IIR (rounded FM input y) and the bare phasor (pi, pq). Bell
//     gain, level, burst window - everything that is a function of (y, phasor) at ONE sample - is k_sec_out, a plain
//     data-parallel kernel that runs once after the fixed point is reached;
//   - the chain's arrays are stored transposed in groups of 8 samples ([group][line][8]), so the 32 lanes of a
//     warp (32 lines) read and write 32 adjacent 16-byte pieces instead of 32 scattered rows;
//   - coupling between lines is short: the IIR forgets its start within ~400 samples (a1 = -0.905) and the two
//     aliased words A, B only enter the last 7 low-pass outputs. Pass 0 leaves checkpoints - the IIR state every 64
//     samples and the IIR state + phasor at the last group boundary before those 7 samples (`ck`) - k_sec_predict
//     walks the short A, B chain down the lines from them, and the later passes (k_sec_refine) re-run the IIR only
//     until it meets the old trajectory bit for bit, the FM recurrence only from `ck` (or, when a rounded FM input
//     before `ck` did change, in full from a work list: k_sec_fm_list).

#define SEC_IYC 64                    // IIR state checkpoint every 64 samples (8 groups)
#define SEC_WARMUP 160                // pass 0: samples of the previous subcarrier line the IIR guess is warmed up on

__device__ __forceinline__ bool sec_same(const SecState &a, const SecState &b)
{
	return(a.A == b.A && a.B == b.B && __double_as_longlong(a.ix) == __double_as_longlong(b.ix) &&
	       __double_as_longlong(a.iy) == __double_as_longlong(b.iy));
}

// last group boundary with all 8 samples clear of the aliased-tail terms (x < W - 7)
__device__ __forceinline__ int sec_ck(int W) { return(((W - 7) >> 3) << 3); }
__device__ __forceinline__ size_t sec_t(const SecScratch &ss, int c, int x) { return((((size_t) (x >> 3) * ss.rows + c) << 3) + (x & 7)); }

// state handed to row c: the outgoing state of the nearest row before it that carries a subcarrier (rows without
// one pass the state on, the two field-start lines clear A and B: ref video.c:3149-3160), or the launch's carry
__device__ __forceinline__ SecState sec_incoming(const LineS2 *lr, const SecScratch &ss, int c, const SecState *prev_out, int &from)
{
	bool clr = false;
	int p = c - 1;
	for(; p >= 0; p--)
	{
		if(lr[p].sec_proc) break;
		if(lr[p].sec_clear) clr = true;
	}
	from = p;
	SecState s = p >= 0 ? prev_out[p] : *ss.carry;
	if(clr) { s.A = 0; s.B = 0; }
	return(s);
}

// round() (half away from zero) of v, then the int16 clamp. The reference clamps the double and rounds (fir.c:729-733);
// the order does not matter (both are monotone and the bounds are integers). 2 v is exact, trunc(2 v) = m, and
// round(v) = (m + 1) >> 1 for m >= 0, m >> 1 for m < 0.
__device__ __forceinline__ int sec_round16(double v)
{
	const int m = __double2int_rz(__dadd_rn(v, v));
	const int r = (m + 1 + (m >> 31)) >> 1;
	return(max(-32768, min(32767, r)));
}

__device__ __forceinline__ double sec_iir_step(const htv_dparams_t &dp, double xin, double &ix, double &iy)
{
	iy = __dadd_rn(__dadd_rn(__dmul_rn(xin, dp.iir_b0), __dmul_rn(ix, dp.iir_b1)), -__dmul_rn(iy, dp.iir_a1));
	ix = xin;
	return(iy);
}

// 8 samples (packed shorts) through the IIR: the feed-forward half is independent of the recurrence
__device__ __forceinline__ int4 sec_iir8(const htv_dparams_t &dp, const int4 v, double &ix, double &iy)
{
	const int w[4] = { v.x, v.y, v.z, v.w };
	double xs[8], t[8];
	#pragma unroll
	for(int k = 0; k < 4; k++) { xs[2 * k] = (double) (short) (w[k] & 0xFFFF); xs[2 * k + 1] = (double) (w[k] >> 16); }
	#pragma unroll
	for(int k = 0; k < 8; k++) t[k] = __dadd_rn(__dmul_rn(xs[k], dp.iir_b0), __dmul_rn(k ? xs[k - 1] : ix, dp.iir_b1));
	int o[8];
	#pragma unroll
	for(int k = 0; k < 8; k++)
	{
		iy = __dadd_rn(t[k], -__dmul_rn(iy, dp.iir_a1));
		o[k] = sec_round16(iy);
	}
	ix = xs[7];
	return(make_int4((o[0] & 0xFFFF) | (o[1] << 16), (o[2] & 0xFFFF) | (o[3] << 16), (o[4] & 0xFFFF) | (o[5] << 16), (o[6] & 0xFFFF) | (o[7] << 16)));
}

// one step of the Q31 phasor recurrence (ref video.c:2278-2297): p <- (p * m) >> 31 on 64-bit products. Signed
// 32 x 32 -> 64 multiply-adds (one IMAD.WIDE each; the compiler's own code for the long long products is 3x longer).
// -m.q is exact: the table holds lround(sin * INT32_MAX), never INT32_MIN.
__device__ __forceinline__ void sec_fm_step(int &pi, int &pq, const htv_c32_t m)
{
	long long ni, nq;
	asm("{\n\t.reg .s64 t;\n\tmul.wide.s32 t, %1, %2;\n\tmad.wide.s32 %0, %3, %4, t;\n\t}" : "=l"(ni) : "r"(pi), "r"(m.i), "r"(pq), "r"(-m.q));
	asm("{\n\t.reg .s64 t;\n\tmul.wide.s32 t, %1, %2;\n\tmad.wide.s32 %0, %3, %4, t;\n\t}" : "=l"(nq) : "r"(pi), "r"(m.q), "r"(pq), "r"(m.i));
	pi = (int) (ni >> 31); pq = (int) (nq >> 31);
}

__device__ __forceinline__ int sec_ph(int pi, int pq) { return((int) (((unsigned) pi >> 16) | ((unsigned) pq & 0xFFFF0000u))); }

// modulator output of one sample before the burst window (ref video.c:3216-3225): phasor halves * level * bell gain
__device__ __forceinline__ int sec_out(const htv_dparams_t &dp, const DevTables &dt, int ph, int sv)
{
	const htv_c16_t g = dt.secam_bell[(unsigned short) sv];
	const int pih = (short) (ph & 0xFFFF), pqh = ph >> 16;
	return((short) (((((pih * dp.secam_level) >> 15) * g.i) >> 15) - ((((pqh * dp.secam_level) >> 15) * g.q) >> 15)));
}

__device__ __forceinline__ void sec_unpack8(const int4 v, int *s)
{
	s[0] = (short) (v.x & 0xFFFF); s[1] = v.x >> 16; s[2] = (short) (v.y & 0xFFFF); s[3] = v.y >> 16;
	s[4] = (short) (v.z & 0xFFFF); s[5] = v.z >> 16; s[6] = (short) (v.w & 0xFFFF); s[7] = v.w >> 16;
}

// the FM look-ups of one group of FM inputs (the recurrence's only memory dependence: issued a group ahead)
__device__ __forceinline__ void sec_gather8(const DevTables &dt, const int4 y8, int dmin, int dmax, htv_c32_t *m)
{
	int s[8];
	sec_unpack8(y8, s);
	#pragma unroll
	for(int k = 0; k < 8; k++) m[k] = dt.secam_fm_lut[max(dmin, min(dmax, s[k])) + 32768];
}

// one group of the FM recurrence over samples xb .. xb + 7, active range [x0, x1); phasor halves go to phT
__device__ __forceinline__ void sec_fm8(const SecScratch &ss, int c, int xb, int x0, int x1, const htv_c32_t *m, int &pi, int &pq)
{
	int ph[8];
	if(xb >= x0 && xb + 8 <= x1)
	{
		#pragma unroll
		for(int k = 0; k < 8; k++) { sec_fm_step(pi, pq, m[k]); ph[k] = sec_ph(pi, pq); }
	}
	else
	{
		#pragma unroll
		for(int k = 0; k < 8; k++)
		{
			ph[k] = 0;
			if(xb + k >= x0 && xb + k < x1) { sec_fm_step(pi, pq, m[k]); ph[k] = sec_ph(pi, pq); }
		}
	}
	int4 *p = reinterpret_cast<int4 *>(ss.phT + sec_t(ss, c, xb));
	p[0] = make_int4(ph[0], ph[1], ph[2], ph[3]);
	p[1] = make_int4(ph[4], ph[5], ph[6], ph[7]);
}

// From the checkpoint before sample ck to the end of the line: the last IIR steps (low-pass outputs finished with the
// aliased words A, B: ref video.c:3171-3180) and the last FM steps, which produce the line's own A, B when the FM
// loop overruns the line end (sr > W). 8 .. 15 + 2 samples. `store`: keep y and the phasor for k_sec_out.
// Inputs of a line's tail kept in registers (the predictor applies the tail a dozen times to the same line)
struct SecTailIn {
	int cbv[16];                      // baseband from sample ck on (8 used when 8 | W)
	int tl[8];                        // raw sums of the last 7 low-pass outputs
	int sr, dmin, dmax;
};

template<bool AL>
__device__ __forceinline__ void sec_tail_load(const htv_dparams_t &dp, const LineS2 &li, const SecScratch &ss, int c, SecTailIn &ti)
{
	const int W = dp.W, ck = AL ? W - 8 : sec_ck(W);
	sec_unpack8(*reinterpret_cast<const int4 *>(ss.cbT + sec_t(ss, c, ck)), ti.cbv);
	if(!AL && ck + 8 < W) sec_unpack8(*reinterpret_cast<const int4 *>(ss.cbT + sec_t(ss, c, ck + 8)), ti.cbv + 8);
	const int *tail = ss.tail + (size_t) c * SEC_TAIL;
	const int4 t0 = *reinterpret_cast<const int4 *>(tail), t1 = *reinterpret_cast<const int4 *>(tail + 4);
	ti.tl[0] = t0.x; ti.tl[1] = t0.y; ti.tl[2] = t0.z; ti.tl[3] = t0.w; ti.tl[4] = t1.x; ti.tl[5] = t1.y; ti.tl[6] = t1.z; ti.tl[7] = t1.w;
	ti.sr = li.sec_sr; ti.dmin = dp.secam_dmin[li.sec_dr]; ti.dmax = dp.secam_dmax[li.sec_dr];
}

// From the checkpoint before sample ck to the end of the line: the last IIR steps (low-pass outputs finished with the
// aliased words A, B: ref video.c:3171-3180) and the last FM steps, which produce the line's own A, B when the FM
// loop overruns the line end (sr > W). 8 .. 15 + 2 samples. `store`: keep y and the phasor for k_sec_out.
// AL: 8 | W, so ck = W - 8 and every index below is a compile-time constant
template<bool AL>
__device__ __forceinline__ SecState sec_tail_core(const htv_dparams_t &dp, const DevTables &dt, const SecScratch &ss,
	int c, const SecTailIn &ti, const SecState &in, const SecChk &ck4, bool store)
{
	const int W = dp.W, ck = AL ? W - 8 : sec_ck(W), sr = ti.sr, sl = dp.burst_left;
	const int dmin = ti.dmin, dmax = ti.dmax;
	double ix = ck4.ixm, iy = ck4.iym;
	int pi = ck4.pi, pq = ck4.pq;
	const bool fm = ck4.valid && sr > ck;
	SecState out = in;
	#pragma unroll
	for(int k = 0; k < (AL ? 10 : 17); k++)
	{
		const int x = ck + k;
		if(!AL && x >= W + 2) break;
		int yv;
		if(x < W)
		{
			int v = ti.cbv[k < 16 ? k : 15];
			if(AL ? k >= 1 : x >= W - 7)
			{
				int acc = 0;
				if(AL) acc = ti.tl[k >= 1 && k <= 7 ? k - 1 : 0];
				else
				{
					#pragma unroll
					for(int j = 0; j < 7; j++) if(x - (W - 7) == j) acc = ti.tl[j];
				}
				const int kA = AL ? 15 - k : W - x + 7, kB = kA + 1;
				if(kA <= 14) acc += in.A * dp.secam_lpf[kA];
				if(kB <= 14) acc += in.B * dp.secam_lpf[kB];
				v = sat16i(acc >> 15);
			}
			yv = sec_round16(sec_iir_step(dp, (double) v, ix, iy));
			if(store) ss.yT[sec_t(ss, c, x)] = (int16_t) yv;
		}
		else yv = (short) (x == W ? in.A : in.B);
		if(fm && x >= sl && x < sr)
		{
			const int sv = max(dmin, min(dmax, yv));
			sec_fm_step(pi, pq, dt.secam_fm_lut[sv + 32768]);
			if(x < W) { if(store) ss.phT[sec_t(ss, c, x)] = sec_ph(pi, pq); }
			else if(x == W) out.A = sec_out(dp, dt, sec_ph(pi, pq), sv);
			else out.B = sec_out(dp, dt, sec_ph(pi, pq), sv);
		}
		else if(x < W && store) ss.phT[sec_t(ss, c, x)] = 0;
	}
	out.ix = ix; out.iy = iy;
	return(out);
}

__device__ __forceinline__ SecState sec_tail(const htv_dparams_t &dp, const DevTables &dt, const LineS2 &li, const SecScratch &ss,
	int c, const SecState &in, const SecChk &ck4, bool store)
{
	SecTailIn ti;
	if((dp.W & 7) == 0)
	{
		sec_tail_load<true>(dp, li, ss, c, ti);
		return(sec_tail_core<true>(dp, dt, ss, c, ti, in, ck4, store));
	}
	sec_tail_load<false>(dp, li, ss, c, ti);
	return(sec_tail_core<false>(dp, dt, ss, c, ti, in, ck4, store));
}

// Pass 0: every line in full from a guessed incoming state - A = B = 0 and the IIR state the previous subcarrier
// line leaves when started from rest SEC_WARMUP samples before its end. IIR and FM recurrence run a group apart in
// the same thread: the FM look-ups of group g are in flight while the IIR does group g + 1.
__global__ void __launch_bounds__(32)
k_sec_pass0(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, SecScratch ss, int n)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if(c >= n) return;
	const int W = dp.W, ck = sec_ck(W), G0 = ck >> 3;
	const LineS2 &li = lr[c];
	SecState *cur = ss.st[0];
	int from;
	SecState in = sec_incoming(lr, ss, c, ss.st[1], from);
	if(from >= 0)
	{
		in.A = in.B = 0; in.pad0 = in.pad1 = 0;
		double ix = 0.0, iy = 0.0;
		const int gs = W > SEC_WARMUP ? (W - SEC_WARMUP) >> 3 : 0, ge = W >> 3;
		const int4 *fp = reinterpret_cast<const int4 *>(ss.cbT) + from;
		for(int g = gs; g < ge; g++) sec_iir8(dp, fp[(size_t) g * ss.rows], ix, iy);
		for(int x = ge << 3; x < W; x++) sec_iir_step(dp, (double) ss.cbT[sec_t(ss, from, x)], ix, iy);
		in.ix = ix; in.iy = iy;
	}
	if(li.sec_clear) { in.A = 0; in.B = 0; }
	if(!li.sec_proc) { cur[c] = in; return; }
	ss.used[c] = in;

	const int sl = dp.burst_left, sr = li.sec_sr, lim = min(sr, ck);
	const int dmin = dp.secam_dmin[li.sec_dr], dmax = dp.secam_dmax[li.sec_dr];
	double ix = in.ix, iy = in.iy;
	int pi = li.sec_sign > 0 ? 2147483647 : -2147483647, pq = 0;
	htv_c32_t m[8];
	const int4 *cbp = reinterpret_cast<const int4 *>(ss.cbT) + c;
	int4 *yp = reinterpret_cast<int4 *>(ss.yT) + c;
	int4 v = G0 > 0 ? cbp[0] : make_int4(0, 0, 0, 0);
	for(int g = 0; g < G0; g++)
	{
		const int4 vn = g + 1 < G0 ? cbp[(size_t) (g + 1) * ss.rows] : make_int4(0, 0, 0, 0);
		if((g & (SEC_IYC / 8 - 1)) == 0) ss.iyc[(size_t) (g >> 3) * ss.rows + c] = iy;
		const int4 y8 = sec_iir8(dp, v, ix, iy);
		yp[(size_t) g * ss.rows] = y8;
		htv_c32_t mn[8];
		const int xb = g << 3;
		const bool act = xb + 8 > sl && xb < lim;
		if(act) sec_gather8(dt, y8, dmin, dmax, mn);
		// the FM steps of the previous group, whose look-ups were issued an iteration ago
		if(g > 0) sec_fm8(ss, c, xb - 8, sl, lim, m, pi, pq);
		#pragma unroll
		for(int k = 0; k < 8; k++) m[k] = mn[k];
		v = vn;
	}
	if(G0 > 0) sec_fm8(ss, c, (G0 - 1) << 3, sl, lim, m, pi, pq);
	SecChk k4;
	k4.pi = pi; k4.pq = pq; k4.valid = ck < sr; k4.pad = 0;
	k4.ixm = ix; k4.iym = iy;
	ss.chk[c] = k4;
	cur[c] = ss.outc[c] = sec_tail(dp, dt, li, ss, c, in, k4, true);
}

// Predictor between pass 0 and pass 1. Pass 0 ran every line with A = B = 0; the true values ripple down the lines
// (line L's A, B enter the last 7 low-pass outputs of line L + 1, hence its last FM inputs, hence its own A, B) and
// the error shrinks only ~3x per line - about nine more full passes. But that coupling lives entirely behind the
// checkpoint pass 0 left: given IIR state and phasor before sample ck, a line's outgoing state follows from the
// incoming A, B in sec_tail's handful of steps. A CTA keeps the tail inputs of its rows in registers and iterates
// state[c] <- tail(c, state[c - 1]) SEC_PRED times through shared memory (the rows above the CTA's own are a halo that
// starts from pass 0's outputs), so pass 1 starts from states that are right to 3^-SEC_PRED. It only proposes states:
// the passes after it recompute whatever a changed incoming state can reach and compare bit for bit. The iteration
// count is an argument (HTV_SEC=pred=...; 0 proposes pass 0's states unchanged).
#define SEC_PRED 12                   // default iterations
#define SEC_PRED_HALO 16
#define SEC_PRED_T 256
template<bool AL>
__device__ __forceinline__ void sec_predict_body(const htv_dparams_t &dp, const DevTables &dt, const LineS2 *lr, const SecScratch &ss, int n, int iters,
	SecState (*sm)[SEC_PRED_T])
{
	const int tid = threadIdx.x;
	const int c = (int) blockIdx.x * (SEC_PRED_T - SEC_PRED_HALO) - SEC_PRED_HALO + tid;
	const SecState *src = ss.st[0];
	SecState *dst = ss.st[1];
	const bool live = c >= 0 && c < n;
	bool proc = false, clear = false;
	SecTailIn ti;
	SecChk k4;
	SecState s, above;
	s.A = s.B = s.pad0 = s.pad1 = 0; s.ix = s.iy = 0.0;
	above = s;
	if(live)
	{
		const LineS2 &li = lr[c];
		proc = li.sec_proc != 0; clear = li.sec_clear != 0;
		s = src[c];
		if(proc) { sec_tail_load<AL>(dp, li, ss, c, ti); k4 = ss.chk[c]; }
		if(tid == 0 || c == 0) above = c == 0 ? *ss.carry : src[c - 1];
	}
	sm[0][tid] = s;
	__syncthreads();
	#pragma unroll 1
	for(int it = 0; it < iters; it++)
	{
		SecState in = (tid == 0 || c == 0) ? above : sm[it & 1][tid - 1];
		if(clear) { in.A = 0; in.B = 0; }
		if(live) s = proc ? sec_tail_core<AL>(dp, dt, ss, c, ti, in, k4, false) : in;
		sm[(it + 1) & 1][tid] = s;
		__syncthreads();
	}
	if(live && tid >= SEC_PRED_HALO)
	{
		SecState out = src[c];
		if(proc) { out.A = s.A; out.B = s.B; out.ix = s.ix; out.iy = s.iy; }
		dst[c] = out;
	}
}

__global__ void __launch_bounds__(SEC_PRED_T)
k_sec_predict(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, SecScratch ss, int n, int iters)
{
	__shared__ SecState sm[2][SEC_PRED_T];
	if((dp.W & 7) == 0) sec_predict_body<true>(dp, dt, lr, ss, n, iters, sm);
	else sec_predict_body<false>(dp, dt, lr, ss, n, iters, sm);
}

// Pass >= 1: a line whose incoming state is not the one it was computed from. The IIR restarts at sample 0 and stops
// where it meets the stored trajectory bit for bit (same iy at a 64-sample checkpoint; ix there is the input sample);
// rounded outputs that differ are rewritten, the first one inside the FM range is remembered. Then the FM recurrence:
// from the checkpoint before ck when nothing ahead of it changed (the usual case), else the line goes on the list.
__global__ void __launch_bounds__(32)
k_sec_refine(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, SecScratch ss, int n, int pass)
{
	const int c = blockIdx.x * blockDim.x + threadIdx.x;
	if(c >= n) return;
	const int W = dp.W, ck = sec_ck(W), G0 = ck >> 3;
	const LineS2 &li = lr[c];
	const SecState *prev = ss.st[(pass + 1) & 1];
	SecState *cur = ss.st[pass & 1];
	int from;
	SecState in = sec_incoming(lr, ss, c, prev, from);
	if(li.sec_clear) { in.A = 0; in.B = 0; }
	if(!li.sec_proc) { cur[c] = in; return; }
	const SecState was = ss.used[c];
	if(sec_same(in, was))
	{
		// nothing new to compute: the line's output for this input is known
		const SecState o = ss.outc[c];
		cur[c] = o;
		if(!sec_same(o, prev[c])) atomicAdd(ss.flags, 1);
		return;
	}
	ss.used[c] = in;
	atomicAdd(ss.flags + 2, 1);

	const int sl = dp.burst_left, sr = li.sec_sr, lim = min(sr, ck);
	int first = 0x7FFFFFFF;
	SecChk k4 = ss.chk[c];
	if(__double_as_longlong(in.ix) != __double_as_longlong(was.ix) || __double_as_longlong(in.iy) != __double_as_longlong(was.iy))
	{
		double ix = in.ix, iy = in.iy;
		const int4 *cbp = reinterpret_cast<const int4 *>(ss.cbT) + c;
		int4 *yp = reinterpret_cast<int4 *>(ss.yT) + c;
		bool merged = false;
		// inputs and old outputs two groups ahead, the next trajectory checkpoint a block of 8 groups ahead
		const int4 z4 = make_int4(0, 0, 0, 0);
		int4 v = G0 > 0 ? cbp[0] : z4, v1 = G0 > 1 ? cbp[ss.rows] : z4;
		int4 old = G0 > 0 ? yp[0] : z4, old1 = G0 > 1 ? yp[ss.rows] : z4;
		double *qc = ss.iyc + c;
		double cknext = G0 > 8 ? qc[ss.rows] : 0.0;
		for(int g = 0; g < G0; g++)
		{
			if((g & (SEC_IYC / 8 - 1)) == 0)
			{
				const int b = g >> 3;
				if(g > 0 && __double_as_longlong(cknext) == __double_as_longlong(iy)) { merged = true; break; }
				qc[(size_t) b * ss.rows] = iy;
				if(g > 0) cknext = g + 8 < G0 ? qc[(size_t) (b + 1) * ss.rows] : 0.0;
			}
			const int4 v2 = g + 2 < G0 ? cbp[(size_t) (g + 2) * ss.rows] : z4;
			const int4 old2 = g + 2 < G0 ? yp[(size_t) (g + 2) * ss.rows] : z4;
			const int4 y8 = sec_iir8(dp, v, ix, iy);
			if(y8.x != old.x || y8.y != old.y || y8.z != old.z || y8.w != old.w)
			{
				yp[(size_t) g * ss.rows] = y8;
				if(first == 0x7FFFFFFF)
				{
					int a[8], b[8];
					sec_unpack8(y8, a); sec_unpack8(old, b);
					#pragma unroll
					for(int k = 7; k >= 0; k--) { const int x = (g << 3) + k; if(a[k] != b[k] && x >= sl && x < lim) first = x; }
				}
			}
			v = v1; v1 = v2; old = old1; old1 = old2;
		}
		if(!merged) { k4.ixm = ix; k4.iym = iy; ss.chk[c].ixm = ix; ss.chk[c].iym = iy; }
	}
	if(first < lim)
	{
		ss.list[atomicAdd(ss.flags + 3, 1)] = c;                            // k_sec_fm_list finishes the line
		return;
	}
	const SecState out = sec_tail(dp, dt, li, ss, c, in, k4, true);
	cur[c] = ss.outc[c] = out;
	if(!sec_same(out, prev[c])) atomicAdd(ss.flags, 1);
}

// Lines of the work list: the FM recurrence in full from the stored FM input, then the tail. The list is short (a
// fraction of a percent of the lines), so a thread per line would leave the run time at one line's worth of exposed
// look-up latency per group. One WARP per line instead: lane l fetches FM input and look-up of sample base + l for the
// next 32 samples while all lanes step through the current 32 (the entries arrive by shuffle), so a step costs the
// recurrence's own latency and nothing else.
#define SEC_LIST_WARPS 4
#define SEC_LIST_MANY 2048             // above this many lines a thread per line has the better throughput (k_sec_fm_list_t)
// `many`: that threshold, an argument of both list kernels (HTV_SEC=list=warp / thread moves it past either end)
__global__ void __launch_bounds__(32 * SEC_LIST_WARPS)
k_sec_fm_list(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, SecScratch ss, int pass, int many)
{
	const int lane = threadIdx.x & 31;
	const int nw = gridDim.x * SEC_LIST_WARPS, count = ss.flags[3];
	if(count > many) return;                                                // a long list: k_sec_fm_list_t
	const int W = dp.W, ck = sec_ck(W), sl = dp.burst_left;
	const SecState *prev = ss.st[(pass + 1) & 1];
	SecState *cur = ss.st[pass & 1];
	for(int i = blockIdx.x * SEC_LIST_WARPS + (threadIdx.x >> 5); i < count; i += nw)
	{
		const int c = ss.list[i];
		const LineS2 &li = lr[c];
		const int sr = li.sec_sr, lim = min(sr, ck);
		const int dmin = dp.secam_dmin[li.sec_dr], dmax = dp.secam_dmax[li.sec_dr];
		int pi = li.sec_sign > 0 ? 2147483647 : -2147483647, pq = 0;
		const int xs = sl & ~31;
		// FM inputs are fetched two chunks ahead, their look-ups one chunk ahead of the recurrence
		htv_c32_t m, mn;
		m.i = m.q = mn.i = mn.q = 0;
		int yn = 0, ynn = 0;
		if(xs + lane >= sl && xs + lane < lim) m = dt.secam_fm_lut[max(dmin, min(dmax, (int) ss.yT[sec_t(ss, c, xs + lane)])) + 32768];
		if(xs + 32 + lane < lim) yn = ss.yT[sec_t(ss, c, xs + 32 + lane)];
		for(int xb = xs; xb < lim; xb += 32)
		{
			if(xb + 64 + lane < lim) ynn = ss.yT[sec_t(ss, c, xb + 64 + lane)];
			if(xb + 32 + lane < lim) mn = dt.secam_fm_lut[max(dmin, min(dmax, yn)) + 32768];
			int ph = 0;
			if(xb >= sl && xb + 32 <= lim)
			{
				#pragma unroll
				for(int k = 0; k < 32; k++)
				{
					htv_c32_t mk;
					mk.i = __shfl_sync(0xFFFFFFFFu, m.i, k); mk.q = __shfl_sync(0xFFFFFFFFu, m.q, k);
					sec_fm_step(pi, pq, mk);
					ph = lane == k ? sec_ph(pi, pq) : ph;
				}
			}
			else
			{
				#pragma unroll 4
				for(int k = 0; k < 32; k++)
				{
					htv_c32_t mk;
					mk.i = __shfl_sync(0xFFFFFFFFu, m.i, k); mk.q = __shfl_sync(0xFFFFFFFFu, m.q, k);
					if(xb + k >= sl && xb + k < lim)
					{
						sec_fm_step(pi, pq, mk);
						if(lane == k) ph = sec_ph(pi, pq);
					}
				}
			}
			if(xb + lane < ck) ss.phT[sec_t(ss, c, xb + lane)] = ph;
			m = mn; yn = ynn;
		}
		if(lane == 0)
		{
			SecChk k4 = ss.chk[c];
			k4.pi = pi; k4.pq = pq; k4.valid = ck < sr;
			ss.chk[c] = k4;
			const SecState out = sec_tail(dp, dt, li, ss, c, ss.used[c], k4, true);
			cur[c] = ss.outc[c] = out;
			if(!sec_same(out, prev[c])) atomicAdd(ss.flags, 1);
		}
		__syncwarp();
	}
}

// A long work list (low sample rates put more FM inputs within reach of the corrected IIR state; noise pictures too):
// one THREAD per listed line, 32 listed lines per warp - pass 0's arrangement, on the compacted list. FM inputs are
// loaded two groups ahead, their look-ups issued one group ahead of the recurrence.
__global__ void __launch_bounds__(32)
k_sec_fm_list_t(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, SecScratch ss, int pass, int many)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	const int count = ss.flags[3];
	if(count <= many || i >= count) return;
	const int c = ss.list[i];
	const int W = dp.W, ck = sec_ck(W), G0 = ck >> 3;
	const LineS2 &li = lr[c];
	const SecState *prev = ss.st[(pass + 1) & 1];
	SecState *cur = ss.st[pass & 1];
	const int sl = dp.burst_left, sr = li.sec_sr, lim = min(sr, ck);
	const int dmin = dp.secam_dmin[li.sec_dr], dmax = dp.secam_dmax[li.sec_dr];
	int pi = li.sec_sign > 0 ? 2147483647 : -2147483647, pq = 0;
	const int4 *yp = reinterpret_cast<const int4 *>(ss.yT) + c;
	const int g0 = sl >> 3, ge = min((lim + 7) >> 3, G0);
	htv_c32_t m[8];
	int4 yn = make_int4(0, 0, 0, 0);
	if(g0 < ge) sec_gather8(dt, yp[(size_t) g0 * ss.rows], dmin, dmax, m);
	if(g0 + 1 < ge) yn = yp[(size_t) (g0 + 1) * ss.rows];
	for(int g = g0; g < ge; g++)
	{
		const int4 ynn = g + 2 < ge ? yp[(size_t) (g + 2) * ss.rows] : make_int4(0, 0, 0, 0);
		htv_c32_t mn[8];
		if(g + 1 < ge) sec_gather8(dt, yn, dmin, dmax, mn);
		sec_fm8(ss, c, g << 3, sl, lim, m, pi, pq);
		#pragma unroll
		for(int k = 0; k < 8; k++) m[k] = mn[k];
		yn = ynn;
	}
	SecChk k4 = ss.chk[c];
	k4.pi = pi; k4.pq = pq; k4.valid = ck < sr;
	ss.chk[c] = k4;
	const SecState out = sec_tail(dp, dt, li, ss, c, ss.used[c], k4, true);
	cur[c] = ss.outc[c] = out;
	if(!sec_same(out, prev[c])) atomicAdd(ss.flags, 1);
}

// carry for the next launch: the state after chain row `idx` of the final pass (rows without a subcarrier pass it on)
__global__ void k_sec_carry(const LineS2 *lr, SecScratch ss, int idx, int pass_final)
{
	if(threadIdx.x == 0 && blockIdx.x == 0)
	{
		int from;
		SecState s = sec_incoming(lr, ss, idx + 1, ss.st[pass_final & 1], from);
		*ss.carry = s;
	}
}

// After the fixed point: subcarrier samples from (FM input, phasor) - bell gain, level, burst window (ref
// video.c:3216-3228) - added to the composite rows in place, for 32 lines x 64 samples per CTA: read from the transposed
// arrays lane = line, exchanged through shared memory, added row-wise. S-Video: `compq` is not NULL, and every row of it
// is written instead (Q; zero where a line has no subcarrier).
__global__ void __launch_bounds__(256)
k_sec_out(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, SecScratch ss, int16_t *comp, int nchain,
	int16_t *compq)
{
	__shared__ __align__(16) short tile[32][64 + 8];
	__shared__ int any[32];
	const int W = dp.W, sl = dp.burst_left;
	const int r0 = blockIdx.y * 32, xt = blockIdx.x * 64;
	if(threadIdx.x < 32) any[threadIdx.x] = 0;
	__syncthreads();
	{
		const int l = threadIdx.x & 31, gi = threadIdx.x >> 5, c = r0 + l, xb = xt + gi * 8;
		int o[8];
		#pragma unroll
		for(int k = 0; k < 8; k++) o[k] = 0;
		if(c < nchain && xb < W)
		{
			const LineS2 &li = lr[c];
			const int top = min(li.sec_sr, W);
			if(li.sec_proc && li.valid && xb + 8 > sl && xb < top)              // fill lines are never emitted
			{
				const int dmin = dp.secam_dmin[li.sec_dr], dmax = dp.secam_dmax[li.sec_dr];
				int s[8];
				sec_unpack8(*reinterpret_cast<const int4 *>(ss.yT + sec_t(ss, c, xb)), s);
				const int4 *pp = reinterpret_cast<const int4 *>(ss.phT + sec_t(ss, c, xb));
				const int4 p0 = pp[0], p1 = pp[1];
				const int ph[8] = { p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w };
				int w[8];
				sec_unpack8(*reinterpret_cast<const int4 *>(dt.sec_win + xb), w);
				if(xb >= sl && xb + 8 <= top)
				{
					#pragma unroll
					for(int k = 0; k < 8; k++) o[k] = (short) ((sec_out(dp, dt, ph[k], max(dmin, min(dmax, s[k]))) * w[k]) >> 15);
				}
				else
				{
					#pragma unroll
					for(int k = 0; k < 8; k++)
					{
						const int x = xb + k;
						if(x >= sl && x < top) o[k] = (short) ((sec_out(dp, dt, ph[k], max(dmin, min(dmax, s[k]))) * w[k]) >> 15);
					}
				}
				any[l] = 1;
			}
		}
		*reinterpret_cast<int4 *>(&tile[l][gi * 8]) = make_int4((o[0] & 0xFFFF) | (o[1] << 16), (o[2] & 0xFFFF) | (o[3] << 16),
			(o[4] & 0xFFFF) | (o[5] << 16), (o[6] & 0xFFFF) | (o[7] << 16));
	}
	__syncthreads();
	{
		const int l = threadIdx.x >> 3, q = threadIdx.x & 7, c = r0 + l, x = xt + q * 8;
		if(compq && c < nchain && x < W)
		{
			int16_t *dst = compq + (size_t) c * W + x;
			if((W & 7) == 0) *reinterpret_cast<int4 *>(dst) = *reinterpret_cast<const int4 *>(&tile[l][q * 8]);
			else for(int k = 0; k < 8 && x + k < W; k++) dst[k] = tile[l][q * 8 + k];
		}
		else if(c < nchain && x < W && any[l])
		{
			int16_t *dst = comp + (size_t) c * W + x;
			if((W & 7) == 0)
			{
				int a[8], b[8];
				sec_unpack8(*reinterpret_cast<const int4 *>(dst), a);
				sec_unpack8(*reinterpret_cast<const int4 *>(&tile[l][q * 8]), b);
				#pragma unroll
				for(int k = 0; k < 8; k++) a[k] = (a[k] + b[k]) & 0xFFFF;      // wraps like the reference's int16 sum
				*reinterpret_cast<int4 *>(dst) = make_int4(a[0] | (a[1] << 16), a[2] | (a[3] << 16), a[4] | (a[5] << 16), a[6] | (a[7] << 16));
			}
			else for(int k = 0; k < 8 && x + k < W; k++) dst[k] = (int16_t) (dst[k] + tile[l][q * 8 + k]);
		}
	}
}
