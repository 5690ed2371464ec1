// sdrplusplus_b200/csrc/iqtap.cuh -- IQ taps of the front end (included by kernels.cu): the effective stream (what
// IQFrontEnd::bindIQStream hands out, core/src/signal_path/iq_frontend.cpp:132-139) in the sample types its two shipped
// consumers write, the recorder (wav::Writer::write, core/src/utils/wav.cpp:150-183) and the IQ exporter
// (misc_modules/iq_exporter/src/main.cpp:503-514).
//
// The element rules below are the only statement of each conversion: k_export (b200_export_convert, b200_pcm_compress)
// calls them too.  k_iq_tap reads a group of 8 samples of the chunk once, in its format (cf32, or cs16 / cs8 times the
// chunk's ingest scale), and writes that group to every tap of the launch (up to IQT_MAX, parameter block by value).
// When the chunk and every output are 16-byte aligned, a group moves as 16-byte vectors: 8 cf32 samples are four loads,
// 8 cs16 samples two, 8 cs8 samples one; a group is four stores for CF32 / I32, two for I16, one for U8 / I8.  Otherwise,
// and for the last n % 8 samples, each sample is read and written on its own.
#pragma once

// wav.cpp:160-163  bufU8[i] = (samples[i] * 127.0f) + 128.0f: the float -> uint8_t conversion truncates
__device__ __forceinline__ unsigned char iq_rule_u8(float x) {
    const float v = __fadd_rn(__fmul_rn(x, 127.0f), 128.0f);
    return (unsigned char)__float2int_rz(v);
}
// volk_32f_s32f_convert_8i / _16i / _32i: r = x * scalar, clamped to the type's range, rounded to nearest even like rintf
__device__ __forceinline__ signed char iq_rule_i8(float x, float scalar) {
    const float r = fminf(fmaxf(__fmul_rn(x, scalar), -128.0f), 127.0f);
    return (signed char)__float2int_rn(r);
}
__device__ __forceinline__ short iq_rule_i16(float x, float scalar) {
    const float r = fminf(fmaxf(__fmul_rn(x, scalar), -32768.0f), 32767.0f);
    return (short)__float2int_rn(r);
}
__device__ __forceinline__ int iq_rule_i32(float x, float scalar) {
    const float r = fminf(fmaxf(__fmul_rn(x, scalar), -2147483648.0f), 2147483648.0f);
    return __float2int_rn(r);          // saturates at INT_MAX where the CPU conversion overflows
}

#define IQT_GROUP 8        // samples per thread
#define IQT_THREADS 256

// one complex sample of the chunk, index i
template <int FMT>
__device__ __forceinline__ float2 iqt_load1(const void* __restrict__ in, long long i, float sc) {
    if (FMT == FMT_CF32) { return __ldg(reinterpret_cast<const float2*>(in) + i); }
    if (FMT == FMT_CS16) {
        const short2 v = __ldg(reinterpret_cast<const short2*>(in) + i);
        return make_float2(__fmul_rn((float)v.x, sc), __fmul_rn((float)v.y, sc));
    }
    const char2 v = __ldg(reinterpret_cast<const char2*>(in) + i);
    return make_float2(__fmul_rn((float)v.x, sc), __fmul_rn((float)v.y, sc));
}

__device__ __forceinline__ void iqt_store1(const IqTapJob& j, long long i, float2 v) {
    switch (j.type) {
    case IQT_CF32: reinterpret_cast<float2*>(j.out)[i] = v; break;
    case IQT_U8: reinterpret_cast<uchar2*>(j.out)[i] = make_uchar2(iq_rule_u8(v.x), iq_rule_u8(v.y)); break;
    case IQT_I8: reinterpret_cast<char2*>(j.out)[i] = make_char2(iq_rule_i8(v.x, j.scalar), iq_rule_i8(v.y, j.scalar)); break;
    case IQT_I16: reinterpret_cast<short2*>(j.out)[i] = make_short2(iq_rule_i16(v.x, j.scalar), iq_rule_i16(v.y, j.scalar)); break;
    default: reinterpret_cast<int2*>(j.out)[i] = make_int2(iq_rule_i32(v.x, j.scalar), iq_rule_i32(v.y, j.scalar)); break;
    }
}

__device__ __forceinline__ unsigned iqt_pack4(unsigned a, unsigned b, unsigned c, unsigned d) {
    return (a & 0xffu) | ((b & 0xffu) << 8) | ((c & 0xffu) << 16) | (d << 24);
}
__device__ __forceinline__ unsigned iqt_pack2(short a, short b) { return (unsigned)(unsigned short)a | ((unsigned)(unsigned short)b << 16); }

template <int FMT>
__global__ void __launch_bounds__(IQT_THREADS) k_iq_tap(const __grid_constant__ IqTapParams p) {
    const long long g = (long long)blockIdx.x * IQT_THREADS + threadIdx.x;
    const long long base = g * IQT_GROUP;
    if (base >= p.n) { return; }
    if (!p.vec || base + IQT_GROUP > p.n) {
        const long long end = min((long long)p.n, base + IQT_GROUP);
        for (long long i = base; i < end; i++) {
            const float2 v = iqt_load1<FMT>(p.in, i, p.in_scale);
            for (int t = 0; t < p.njobs; t++) { iqt_store1(p.job[t], i, v); }
        }
        return;
    }
    float x[2 * IQT_GROUP];            // I, Q of the group's 8 samples
    if (FMT == FMT_CF32) {
        const float4* src = reinterpret_cast<const float4*>(p.in) + g * 4;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float4 v = __ldg(src + k);
            x[4 * k] = v.x; x[4 * k + 1] = v.y; x[4 * k + 2] = v.z; x[4 * k + 3] = v.w;
        }
    }
    else if (FMT == FMT_CS16) {
        const int4* src = reinterpret_cast<const int4*>(p.in) + g * 2;
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const int4 v = __ldg(src + k);
            const int w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
            for (int q = 0; q < 4; q++) {
                x[8 * k + 2 * q] = __fmul_rn((float)(short)(w[q] & 0xffff), p.in_scale);
                x[8 * k + 2 * q + 1] = __fmul_rn((float)(short)((unsigned)w[q] >> 16), p.in_scale);
            }
        }
    }
    else {
        const int4 v = __ldg(reinterpret_cast<const int4*>(p.in) + g);
        const int w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
        for (int q = 0; q < 4; q++) {
#pragma unroll
            for (int b = 0; b < 4; b++) { x[4 * q + b] = __fmul_rn((float)(signed char)((unsigned)w[q] >> (8 * b)), p.in_scale); }
        }
    }
    for (int t = 0; t < p.njobs; t++) {
        const IqTapJob& j = p.job[t];
        switch (j.type) {
        case IQT_CF32: {
            float4* dst = reinterpret_cast<float4*>(j.out) + g * 4;
#pragma unroll
            for (int k = 0; k < 4; k++) { dst[k] = make_float4(x[4 * k], x[4 * k + 1], x[4 * k + 2], x[4 * k + 3]); }
            break;
        }
        case IQT_U8: case IQT_I8: {
            unsigned b[2 * IQT_GROUP];
#pragma unroll
            for (int k = 0; k < 2 * IQT_GROUP; k++) {
                b[k] = j.type == IQT_U8 ? (unsigned)iq_rule_u8(x[k]) : (unsigned)(unsigned char)iq_rule_i8(x[k], j.scalar);
            }
            reinterpret_cast<uint4*>(j.out)[g] = make_uint4(iqt_pack4(b[0], b[1], b[2], b[3]), iqt_pack4(b[4], b[5], b[6], b[7]),
                                                            iqt_pack4(b[8], b[9], b[10], b[11]), iqt_pack4(b[12], b[13], b[14], b[15]));
            break;
        }
        case IQT_I16: {
            uint4* dst = reinterpret_cast<uint4*>(j.out) + g * 2;
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const float* y = x + 8 * k;
                dst[k] = make_uint4(iqt_pack2(iq_rule_i16(y[0], j.scalar), iq_rule_i16(y[1], j.scalar)),
                                    iqt_pack2(iq_rule_i16(y[2], j.scalar), iq_rule_i16(y[3], j.scalar)),
                                    iqt_pack2(iq_rule_i16(y[4], j.scalar), iq_rule_i16(y[5], j.scalar)),
                                    iqt_pack2(iq_rule_i16(y[6], j.scalar), iq_rule_i16(y[7], j.scalar)));
            }
            break;
        }
        default: {
            int4* dst = reinterpret_cast<int4*>(j.out) + g * 4;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                dst[k] = make_int4(iq_rule_i32(x[4 * k], j.scalar), iq_rule_i32(x[4 * k + 1], j.scalar),
                                   iq_rule_i32(x[4 * k + 2], j.scalar), iq_rule_i32(x[4 * k + 3], j.scalar));
            }
            break;
        }
        }
    }
}
