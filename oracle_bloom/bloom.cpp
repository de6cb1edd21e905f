// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  Bloom (ST_OPT_BLOOM) for the CPU oracle.
//
// This library is the exposure extension (oracle_exposure/exposure.cpp, itself the unchanged oracle plus the display transforms,
// compiled into this translation unit) plus the rule of DESIGN.md §2 "Bloom" in the oracle's own arithmetic, over a frame's `output`:
//   - orc_bloom_pyramid: the pyramid's words (header, down levels, up levels) as st_read_buffer("bloom") returns them;
//   - orc_bloom_store: the Rgba8 store with the glow composited, through the display transform T of oracle_exposure.
// oracle_bloom/pyoracle_bloom.py calls these where the device builds the pyramid and stores.
#include "../oracle_exposure/exposure.cpp"

namespace {

// Test-only mistakes (tests/test_bloom.py shows that the float64 bound catches each): 0 = the rule.
enum { BM_NONE = 0, BM_KARIS_ALL = 1, BM_KARIS_NONE = 2, BM_TENT_111 = 3, BM_SIZES_UP = 4, BM_WRAP = 5, BM_SWAP_SCATTER = 6, BM_EXPOSE_AFTER = 7,
       BM_PREFILTER_AFTER_KARIS = 8, BM_SWAP_MODES = 9, BM_NAN_KEPT = 10 };
const int kMaxLevels = 8, kHeaderWords = 20;

struct P { float intensity, scatter, threshold, softness; int levels, mode; };
struct F4 { float x, y, z, w; };
F4 f4_(float x, float y, float z, float w) { F4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
F4 add(F4 a, F4 b) { return f4_(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
F4 mul(F4 a, float s) { return f4_(a.x * s, a.y * s, a.z * s, a.w * s); }
const float kInf = std::numeric_limits<float>::infinity();

int level_size(int n, int k, int mut) {
    int v = mut == BM_SIZES_UP ? (n + (1 << (k + 1)) - 1) >> (k + 1) : n >> (k + 1);
    return v > 1 ? v : 1;
}
int at(int v, int n, int mut) {
    if (mut == BM_WRAP) return ((v % n) + n) % n;
    return v < 0 ? 0 : (v > n - 1 ? n - 1 : v);
}
float chan_in(float c, float s, int mut) {
    if (mut == BM_NAN_KEPT && c != c) return c * s;
    return (c > 0.0f && c < kInf) ? c * s : 0.0f;
}
F4 prefilter(F4 v, const P& b) {
    if (!(b.threshold > 0.0f)) return v;
    float m = v.x > v.y ? v.x : v.y;
    m = m > v.z ? m : v.z;
    const float t = b.threshold, k = t * b.softness;
    const float q0 = rclamp_((m - t) + k, 0.0f, 2.0f * k);
    const float q = (q0 * q0) / (4.0f * k + 1e-4f);
    const float w = (q > m - t ? q : m - t) / (m > 1e-4f ? m : 1e-4f);
    return f4_(v.x * w, v.y * w, v.z * w, v.w);
}
float finite_or_0(float v, int mut) { return (mut == BM_NAN_KEPT || v < kInf) ? v : 0.0f; }
F4 input(const float* c, float s, const P& b, int mut) {
    F4 v = f4_(chan_in(c[0], s, mut), chan_in(c[1], s, mut), chan_in(c[2], s, mut), 0.0f);
    if (mut != BM_PREFILTER_AFTER_KARIS) v = prefilter(v, b);
    return f4_(finite_or_0(v.x, mut), finite_or_0(v.y, mut), finite_or_0(v.z, mut), 0.0f);
}
F4 tap(F4 a, F4 b, F4 c, F4 d, bool karis) {
    const F4 t = mul(add(add(a, b), add(c, d)), 0.25f);
    if (!karis) return f4_(t.x, t.y, t.z, 1.0f);
    const float w = 1.0f / (1.0f + luminance(t.x, t.y, t.z, 0));
    return f4_(t.x * w, t.y * w, t.z * w, w);
}
F4 group(F4 a, F4 b, F4 c, F4 d, bool karis) {
    const F4 s = add(add(a, b), add(c, d));
    if (!karis) return f4_(s.x * 0.25f, s.y * 0.25f, s.z * 0.25f, 0.0f);
    const float w = (a.w + b.w) + (c.w + d.w);
    return f4_(s.x / w, s.y / w, s.z / w, 0.0f);
}
// level texel (i, j) from src (sw x sh), the 13-tap filter
F4 down_texel(const std::vector<F4>& src, int sw, int sh, int i, int j, bool karis, int mut) {
    auto T = [&](int x, int y) { return src[(size_t)at(y, sh, mut) * sw + at(x, sw, mut)]; };
    auto tp = [&](int cx, int cy) { return tap(T(cx - 1, cy - 1), T(cx, cy - 1), T(cx - 1, cy), T(cx, cy), karis); };
    auto o = [&](int m, int n) { return tp(2 * i - 1 + 2 * m, 2 * j - 1 + 2 * n); };
    auto e = [&](int m, int n) { return tp(2 * i + 2 * m, 2 * j + 2 * n); };
    const F4 C = group(e(0, 0), e(1, 0), e(0, 1), e(1, 1), karis);
    const F4 TL = group(o(0, 0), o(1, 0), o(0, 1), o(1, 1), karis), TR = group(o(1, 0), o(2, 0), o(1, 1), o(2, 1), karis);
    const F4 BL = group(o(0, 1), o(1, 1), o(0, 2), o(1, 2), karis), BR = group(o(1, 1), o(2, 1), o(1, 2), o(2, 2), karis);
    const F4 r = add(mul(C, 0.5f), mul(add(add(TL, TR), add(BL, BR)), 0.125f));
    return f4_(r.x, r.y, r.z, 0.0f);
}
F4 tent(const F4* u, int cw, int ch, int fx, int fy, int mut) {
    const int cx = (fx >> 1) < cw - 1 ? (fx >> 1) : cw - 1, cy = (fy >> 1) < ch - 1 ? (fy >> 1) : ch - 1;
    const int x0 = at(cx - 1, cw, mut), x2 = at(cx + 1, cw, mut);
    const float mid = mut == BM_TENT_111 ? 1.0f : 2.0f;
    F4 r[3];
    for (int d = 0; d < 3; d++) {
        const F4* row = u + (size_t)at(cy - 1 + d, ch, mut) * cw;
        r[d] = add(add(row[x0], mul(row[cx], mid)), row[x2]);
    }
    const F4 s = add(add(r[0], mul(r[1], mid)), r[2]);
    if (mut == BM_TENT_111) return f4_(s.x / 9.0f, s.y / 9.0f, s.z / 9.0f, s.w / 9.0f);
    return mul(s, 0.0625f);
}

struct Pyramid { int L; int w[kMaxLevels], h[kMaxLevels]; std::vector<F4> down[kMaxLevels], up[kMaxLevels]; };

void build(const float* output, int W, int H, float s, const P& b, int mut, Pyramid* py) {
    const int L = b.levels;
    py->L = L;
    for (int k = 0; k < L; k++) { py->w[k] = level_size(W, k, mut); py->h[k] = level_size(H, k, mut); }
    std::vector<F4> x((size_t)W * H);
    for (size_t i = 0; i < x.size(); i++) x[i] = input(output + 4 * i, s, b, mut);
    for (int k = 0; k < L; k++) {
        const std::vector<F4>& src = k == 0 ? x : py->down[k - 1];
        const int sw = k == 0 ? W : py->w[k - 1], sh = k == 0 ? H : py->h[k - 1];
        const bool karis = mut == BM_KARIS_ALL ? true : (mut == BM_KARIS_NONE ? false : k == 0);
        std::vector<F4>& dst = py->down[k];
        dst.resize((size_t)py->w[k] * py->h[k]);
#pragma omp parallel for schedule(static)
        for (int j = 0; j < py->h[k]; j++)
            for (int i = 0; i < py->w[k]; i++) {
                F4 v = down_texel(src, sw, sh, i, j, karis, mut);
                if (k == 0 && mut == BM_PREFILTER_AFTER_KARIS) v = prefilter(v, b);
                dst[(size_t)j * py->w[k] + i] = v;
            }
    }
    py->up[L - 1] = py->down[L - 1];
    const float a = b.scatter, oma = 1.0f - a;
    const float wd = mut == BM_SWAP_SCATTER ? a : oma, wt = mut == BM_SWAP_SCATTER ? oma : a;
    for (int k = L - 2; k >= 0; k--) {
        py->up[k].resize((size_t)py->w[k] * py->h[k]);
        for (int j = 0; j < py->h[k]; j++)
            for (int i = 0; i < py->w[k]; i++) {
                const F4 t = tent(py->up[k + 1].data(), py->w[k + 1], py->h[k + 1], i, j, mut);
                const F4 r = add(mul(py->down[k][(size_t)j * py->w[k] + i], wd), mul(t, wt));
                py->up[k][(size_t)j * py->w[k] + i] = f4_(r.x, r.y, r.z, 0.0f);
            }
    }
}

}  // namespace

extern "C" {

// The pyramid of `output` (W x H float4) with exposure s (1 with tonemapping off) and st_bloom `b` = {intensity, scatter, threshold,
// softness} + levels, mode, as st_read_buffer("bloom") words into `words` (cap words); returns the word count
long orc_bloom_pyramid(const float* output, int W, int H, float s, const float* bf, int levels, int mode, float* words, long cap, int mutation) {
    const P b = {bf[0], bf[1], bf[2], bf[3], levels, mode};
    Pyramid py;
    build(output, W, H, s, b, mutation, &py);
    std::vector<uint32_t> head(kHeaderWords, 0u);
    head[0] = (uint32_t)py.L;
    for (int k = 0; k < py.L; k++) { head[1 + 2 * k] = (uint32_t)py.w[k]; head[2 + 2 * k] = (uint32_t)py.h[k]; }
    std::vector<float> out(kHeaderWords);
    std::memcpy(out.data(), head.data(), 4 * kHeaderWords);
    for (int pass = 0; pass < 2; pass++)
        for (int k = 0; k < (pass == 0 ? py.L : py.L - 1); k++)
            for (const F4& v : (pass == 0 ? py.down[k] : py.up[k])) { out.push_back(v.x); out.push_back(v.y); out.push_back(v.z); out.push_back(v.w); }
    if ((long)out.size() <= cap) std::memcpy(words, out.data(), 4 * out.size());
    return (long)out.size();
}

// The Rgba8 store (W x H x 4 bytes) of `output` with the glow of the pyramid `words` (as orc_bloom_pyramid made it): op 0 today's
// store, 1..4 exposed by s and through T
int orc_bloom_store(const float* output, int W, int H, int op, float s, const float* bf, int mode, const float* words, uint8_t* out, int mutation) {
    uint32_t head[kHeaderWords];
    std::memcpy(head, words, 4 * kHeaderWords);
    const int L = (int)head[0], w0 = (int)head[1], h0 = (int)head[2];
    size_t off = 0;
    for (int k = 0; k < L; k++) off += (size_t)head[1 + 2 * k] * head[2 + 2 * k];
    const F4* up0 = (const F4*)(words + kHeaderWords) + (L == 1 ? 0 : off);
    const float I = bf[0];
    const int md = mutation == BM_SWAP_MODES ? 1 - mode : mode;
#pragma omp parallel for schedule(static)
    for (long p = 0; p < (long)W * H; p++) {
        const int x = (int)(p % W), y = (int)(p / W);
        const float* c = output + 4 * p;
        V3 v = v3(c[0], c[1], c[2]);
        if (op != 0) v = v3((c[0] > 0.0f ? c[0] : 0.0f) * s, (c[1] > 0.0f ? c[1] : 0.0f) * s, (c[2] > 0.0f ? c[2] : 0.0f) * s);
        F4 B = tent(up0, w0, h0, x, y, mutation);
        if (mutation == BM_EXPOSE_AFTER) B = mul(B, s);
        if (md == 0) { const float k = 1.0f - I; v = v3(v.x * k + B.x * I, v.y * k + B.y * I, v.z * k + B.z * I); }
        else v = v3(v.x + B.x * I, v.y + B.y * I, v.z + B.z * I);
        const V3 t = transform(op, v, 0);
        out[4 * p] = store(t.x); out[4 * p + 1] = store(t.y); out[4 * p + 2] = store(t.z); out[4 * p + 3] = 255;
    }
    return 0;
}

}  // extern "C"
