/* hacktv_b200 - the file sink's sample types (ref rf_file.c: the twelve _rf_file_write_* writers, rf.h:31-36).
 *
 * The one definition of how an int16 output value becomes a uint8, int8, uint16, int16, int32 or float sample.
 * The line kernels' stores (kl_post_store in htv_line.cuh, mod_store in htv_kernels.cu), htv_convert's kernel,
 * the host layer (sizes) and the CPU check tests/sample_type_emu.c all include this header.
 *
 * x is always an int16 value (already wrapped): the reference converts what the video stage handed to rf_write.
 * Bit patterns per type (zero-extended to 32 bits):
 *   uint8   (x - INT16_MIN) >> 8
 *   int8    x >> 8
 *   uint16  x - INT16_MIN
 *   int16   x
 *   int32   (x << 16) + x, which gcc wraps at x = -32768 to +2147450880: computed as (unsigned) x * 65537
 *   float   (float) x * (1.0 / 32767.0): a double multiply rounded once to float. A float multiply by
 *           (float) (1 / 32767) differs on 1 536 of the 65 536 values. On the device the same expression
 *           compiles to DMUL.RN + F2F.F32.F64 (round to nearest), the same two roundings as on the host. */
#ifndef HTV_SAMPLE_TYPE_H
#define HTV_SAMPLE_TYPE_H

#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include "hacktv_b200.h"

#ifdef __CUDACC__
#define HTV_ST_FN __host__ __device__ __forceinline__
#else
#define HTV_ST_FN static inline
#endif

/* bytes of one value (one of I, Q), 0 for an unknown type */
HTV_ST_FN int htv_st_size(int type)
{
	switch(type)
	{
	case HTV_TYPE_UINT8: case HTV_TYPE_INT8: return(1);
	case HTV_TYPE_UINT16: case HTV_TYPE_INT16: return(2);
	case HTV_TYPE_INT32: case HTV_TYPE_FLOAT: return(4);
	}
	return(0);
}

/* hacktv's -t spelling, NULL for an unknown type */
HTV_ST_FN const char *htv_st_name(int type)
{
	switch(type)
	{
	case HTV_TYPE_UINT8: return("uint8");
	case HTV_TYPE_INT8: return("int8");
	case HTV_TYPE_UINT16: return("uint16");
	case HTV_TYPE_INT16: return("int16");
	case HTV_TYPE_INT32: return("int32");
	case HTV_TYPE_FLOAT: return("float");
	}
	return(NULL);
}

/* bytes per sample of a stream: both components for complex output, I only for real output */
HTV_ST_FN int htv_st_bytes(int type, int complex) { return(htv_st_size(type) * (complex ? 2 : 1)); }

HTV_ST_FN float htv_st_float(int x) { return((float) ((double) x * (1.0 / 32767.0))); }

/* the converted value's bit pattern */
HTV_ST_FN uint32_t htv_st_bits(int type, int x)
{
	switch(type)
	{
	case HTV_TYPE_UINT8: return((uint32_t) ((x - INT16_MIN) >> 8));
	case HTV_TYPE_INT8: return((uint32_t) (x >> 8) & 0xFFu);
	case HTV_TYPE_UINT16: return((uint32_t) (x - INT16_MIN));
	case HTV_TYPE_INT16: return((uint32_t) x & 0xFFFFu);
	case HTV_TYPE_INT32: return((uint32_t) x * 65537u);
	case HTV_TYPE_FLOAT:
	{
		const float f = htv_st_float(x);
#ifdef __CUDA_ARCH__
		return(__float_as_uint(f));
#else
		uint32_t u;
		memcpy(&u, &f, sizeof(u));
		return(u);
#endif
	}
	}
	return(0);
}

/* value i of a stream of `type` <- x */
HTV_ST_FN void htv_st_put(void *out, size_t i, int type, int x)
{
	const uint32_t b = htv_st_bits(type, x);
	switch(htv_st_size(type))
	{
	case 1: ((uint8_t *) out)[i] = (uint8_t) b; break;
	case 2: ((uint16_t *) out)[i] = (uint16_t) b; break;
	case 4: ((uint32_t *) out)[i] = b; break;
	}
}

/* complex sample s of a stream of `type` <- (xi, xq), as one store of both components */
HTV_ST_FN void htv_st_put2(void *out, size_t s, int type, int xi, int xq)
{
	const uint32_t bi = htv_st_bits(type, xi), bq = htv_st_bits(type, xq);
	switch(htv_st_size(type))
	{
	case 1: ((uint16_t *) out)[s] = (uint16_t) (bi | (bq << 8)); break;
	case 2: ((uint32_t *) out)[s] = bi | (bq << 16); break;
	case 4: ((uint64_t *) out)[s] = (uint64_t) bi | ((uint64_t) bq << 32); break;
	}
}

#endif
