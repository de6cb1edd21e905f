// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  Exposure and tonemapping (ST_OPT_TONEMAPPING, ST_OPT_AUTO_EXPOSURE) for the CPU oracle.
//
// The oracle in oracle/ restates the reference, which stores the composed frame as Rgba8UnormSrgb by clamping linear light, and stays
// exactly as it is.  This library is that oracle (oracle.cpp compiled unchanged into this translation unit, for its deterministic
// pow_) plus the rule of DESIGN.md §2 "Exposure and tonemapping" in the oracle's own arithmetic, over a frame's `output`:
//   - orc_expo_histogram: the 256-bin log-luminance histogram;
//   - orc_expo_meter: the metering and adaptation of one frame, over its bins and the camera's state;
//   - orc_expo_display: the Rgba8 store, today's (op 0) or exposed and tonemapped (op 1..4);
//   - orc_expo_log2: log2_x, for the float64 restatement's bound.
// oracle_exposure/pyoracle_exposure.py calls these where the device meters and stores.
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

// Test-only mistakes (tests/test_exposure.py shows that the float64 bound catches each): 0 = the rule.
enum { MUT_NONE = 0, MUT_REC601 = 1, MUT_BIN_LOWER_EDGE = 2, MUT_NO_WINDOW = 3, MUT_SWAP_SPEEDS = 4, MUT_EXPOSE_AFTER_T = 5, MUT_ACES_TRANSPOSED = 6,
       MUT_AGX_ROW_MAJOR = 7, MUT_AGX_NO_POW = 8 };

const int kBins = 256;

// log2 of a finite x > 0: the exponent bits plus the Cephes logf polynomial of the mantissa, times log2(e) (st_device.cuh log2_x)
float log2_x(float x) {
    u32 bits = f2u(x);
    int e;
    if ((bits & 0x7f800000u) == 0u) { x = x * 8388608.0f; bits = f2u(x); e = (int)((bits >> 23) & 0xffu) - 126 - 23; }
    else e = (int)((bits >> 23) & 0xffu) - 126;
    float m = u2f((bits & 0x007fffffu) | 0x3f000000u);
    if (m < 0.707106781186547524f) { e -= 1; m = (m + m) - 1.0f; } else m = m - 1.0f;
    const float z = m * m;
    float y = 7.0376836292e-2f;
    y = y * m + -1.1514610310e-1f; y = y * m + 1.1676998740e-1f; y = y * m + -1.2420140846e-1f;
    y = y * m + 1.4249322787e-1f; y = y * m + -1.6668057665e-1f; y = y * m + 2.0000714765e-1f;
    y = y * m + -2.4999993993e-1f; y = y * m + 3.3333331174e-1f;
    y = (y * m) * z;
    y = y + -0.5f * z;
    const float ln_m = m + y;
    return ln_m * 1.44269504088896341f + (float)e;
}

float luminance(float r, float g, float b, int mut) {
    if (mut == MUT_REC601) return (0.299f * r + 0.587f * g) + 0.114f * b;
    return (0.2126f * r + 0.7152f * g) + 0.0722f * b;
}
int bin_of(float L) {
    if (!(L > 0.0f) || L == F32_INF) return -1;
    const float y = (log2_x(L) + 16.0f) * 8.0f;
    return y < 0.0f ? 0 : (y >= 256.0f ? 255 : (int)y);
}
float rclamp_(float x, float lo, float hi) { if (x < lo) x = lo; if (x > hi) x = hi; return x; }

// p = {ev, compensation, ev_min, ev_max, low, high, speed_up, speed_down}; state = {ev, target (f32 bits), counted, kept, frames}
void meter(const u32* bins, u32* state, const float* p, int mut) {
    unsigned long long n = 0;
    for (int b = 0; b < kBins; b++) n += bins[b];
    const double lo = mut == MUT_NO_WINDOW ? 0.0 : std::floor((double)p[4] * (double)n), hi = mut == MUT_NO_WINDOW ? (double)n : std::ceil((double)p[5] * (double)n);
    double start = 0.0, kept = 0.0, sum = 0.0;
    for (int b = 0; b < kBins; b++) {
        const double end = start + (double)bins[b];
        const double a = start > lo ? start : lo, z = end < hi ? end : hi;
        const double centre = mut == MUT_BIN_LOWER_EDGE ? -16.0 + (double)b / 8.0 : -16.0 + ((double)b + 0.5) / 8.0;
        if (z > a) { kept = kept + (z - a); sum = sum + (z - a) * centre; }
        start = end;
    }
    const bool first = state[4] == 0u;
    const float prev = u2f(state[0]);
    float target;
    if (kept > 0.0) {
        double t = sum / kept - (-2.4739311883324122);
        t = t < (double)p[2] ? (double)p[2] : t;
        t = t > (double)p[3] ? (double)p[3] : t;
        target = (float)t;
    } else if (first) target = rclamp_(0.0f, p[2], p[3]);
    else target = prev;
    const float up = mut == MUT_SWAP_SPEEDS ? p[7] : p[6], down = mut == MUT_SWAP_SPEEDS ? p[6] : p[7];
    float ev = target;
    if (!first) {
        const float d = target - prev;
        if (d > up) ev = prev + up;
        else if (d < -down) ev = prev - down;
    }
    state[0] = f2u(ev); state[1] = f2u(target); state[2] = (u32)n; state[3] = (u32)kept; state[4] = state[4] + 1u;
}

V3 mat(const float m[9], V3 v, bool transposed) {
    if (transposed) return v3((m[0] * v.x + m[3] * v.y) + m[6] * v.z, (m[1] * v.x + m[4] * v.y) + m[7] * v.z, (m[2] * v.x + m[5] * v.y) + m[8] * v.z);
    return v3((m[0] * v.x + m[1] * v.y) + m[2] * v.z, (m[3] * v.x + m[4] * v.y) + m[5] * v.z, (m[6] * v.x + m[7] * v.y) + m[8] * v.z);
}
float aces_curve(float v) { return (v * (v + 0.0245786f) - 0.000090537f) / (v * (0.983729f * v + 0.4329510f) + 0.238081f); }
float agx_curve(float v) {
    float l = v > 0.0f ? log2_x(v) : -12.47393f;
    l = l < -12.47393f ? -12.47393f : l;
    l = l > 4.026069f ? 4.026069f : l;
    const float x = (l + 12.47393f) / 16.499999f;
    const float x2 = x * x, x4 = x2 * x2;
    return (((((15.5f * x4 * x2 - 40.14f * x4 * x) + 31.96f * x4) - 6.868f * x2 * x) + 0.4298f * x2) + 0.1191f * x) - 0.00232f;
}
V3 transform(int op, V3 x, int mut) {
    if (op == 2) { const float d = 1.0f + luminance(x.x, x.y, x.z, mut); return v3(x.x / d, x.y / d, x.z / d); }
    if (op == 3) {
        const float A[9] = {0.59719f, 0.35458f, 0.04823f, 0.07600f, 0.90834f, 0.01566f, 0.02840f, 0.13383f, 0.83777f};
        const float B[9] = {1.60475f, -0.53108f, -0.07367f, -0.10208f, 1.10813f, -0.00605f, -0.00327f, -0.07276f, 1.07602f};
        const bool tr = mut == MUT_ACES_TRANSPOSED;
        const V3 v = mat(A, x, tr);
        return mat(B, v3(aces_curve(v.x), aces_curve(v.y), aces_curve(v.z)), tr);
    }
    if (op == 4) {
        const float M[9] = {0.842479062253094f, 0.0784335999999992f, 0.0792237451477643f, 0.0423282422610123f, 0.878468636469772f, 0.0791661274605434f,
                            0.0423756549057051f, 0.0784336f, 0.879142973793104f};
        const float MI[9] = {1.19687900512017f, -0.0980208811401368f, -0.0990297440797205f, -0.0528968517574562f, 1.15190312990417f, -0.0989611768448433f,
                             -0.0529716355144438f, -0.0980434501171241f, 1.15107367264116f};
        const bool tr = mut == MUT_AGX_ROW_MAJOR;
        const V3 v = mat(M, x, tr);
        const V3 u = mat(MI, v3(agx_curve(v.x), agx_curve(v.y), agx_curve(v.z)), tr);
        const V3 c = v3(u.x > 0.0f ? u.x : 0.0f, u.y > 0.0f ? u.y : 0.0f, u.z > 0.0f ? u.z : 0.0f);
        if (mut == MUT_AGX_NO_POW) return c;
        return v3(pow_(c.x, 2.2f), pow_(c.y, 2.2f), pow_(c.z, 2.2f));
    }
    return x;
}
// __float2uint_rz: truncating, saturating, NaN -> 0
u32 to_u32_sat_(float f) { if (!(f == f) || f <= 0.0f) return 0u; if (f >= 4294967296.0f) return 0xffffffffu; return (u32)f; }
// k_output_rgba8's store of one linear channel
uint8_t store(float v) {
    const float x = rclamp_(v, 0.0f, 1.0f);
    const float e = (x <= 0.0031308f) ? 12.92f * x : 1.055f * pow_(x, 1.0f / 2.4f) - 0.055f;
    return (uint8_t)to_u32_sat_(rclamp_(e, 0.0f, 1.0f) * 255.0f + 0.5f);
}

}  // namespace

extern "C" {

// bins (256) = the histogram of `output` (n float4 pixels)
int orc_expo_histogram(const float* output, long n, uint32_t* bins, int mutation) {
    for (int b = 0; b < kBins; b++) bins[b] = 0u;
    for (long i = 0; i < n; i++) {
        const float* c = output + 4 * i;
        const int b = bin_of(luminance(c[0], c[1], c[2], mutation));
        if (b >= 0) bins[b] += 1u;
    }
    return 0;
}

// one frame's metering and adaptation: state (5 words) is the camera's, updated in place; params = st_exposure's 8 floats
int orc_expo_meter(const uint32_t* bins, uint32_t* state, const float* params, int mutation) { meter(bins, state, params, mutation); return 0; }

// The Rgba8 store of `output` (n float4 pixels) into out (n x 4 bytes): op 0 is k_output_rgba8's, op 1..4 k_output_display<op>'s
// with exposure 2^(compensation - ev)
int orc_expo_display(const float* output, long n, int op, float ev, float compensation, uint8_t* out, int mutation) {
    const float s = pow_(2.0f, compensation - ev);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < n; i++) {
        const float* c = output + 4 * i;
        V3 t;
        if (op == 0) t = v3(c[0], c[1], c[2]);
        else {
            const V3 x = v3(c[0] > 0.0f ? c[0] : 0.0f, c[1] > 0.0f ? c[1] : 0.0f, c[2] > 0.0f ? c[2] : 0.0f);
            if (mutation == MUT_EXPOSE_AFTER_T) { const V3 y = transform(op, x, mutation); t = v3(y.x * s, y.y * s, y.z * s); }
            else t = transform(op, v3(x.x * s, x.y * s, x.z * s), mutation);
        }
        out[4 * i] = store(t.x); out[4 * i + 1] = store(t.y); out[4 * i + 2] = store(t.z); out[4 * i + 3] = 255;
    }
    return 0;
}

// T(x) before the store, per pixel (n float3 in, n float3 out), for the float64 restatement
int orc_expo_transform(const float* in, long n, int op, float* out, int mutation) {
    for (long i = 0; i < n; i++) {
        const V3 t = transform(op, v3(in[3 * i], in[3 * i + 1], in[3 * i + 2]), mutation);
        out[3 * i] = t.x; out[3 * i + 1] = t.y; out[3 * i + 2] = t.z;
    }
    return 0;
}

void orc_expo_log2(const float* a, float* out, long n) { for (long i = 0; i < n; i++) out[i] = log2_x(a[i]); }
float orc_expo_pow(float x, float y) { return pow_(x, y); }

}  // extern "C"
