// The PCM-16 code of a float sample, shared by the wire encodings (encode.cu) and the FLAC encoder (flac.cu):
// v = clip(rint(x * 32767), -32768, 32767) with the product in double (exact for every float) and round-half-to-even;
// NaN gives 0, +-Inf clip.  cvt.rni.s32.f64 rounds half to even and saturates +-Inf; NaN is mapped to 0 by the
// definition.  A macro, so that every kernel that quantizes compiles exactly the expression it always has.
#pragma once

#define VTTS_PCM16_OF(x) ((x) != (x) ? 0 : min(max(__double2int_rn((double)(x) * 32767.0), -32768), 32767))
