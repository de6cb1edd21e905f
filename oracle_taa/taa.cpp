// ORACLE EXTENSION — TEST INFRASTRUCTURE ONLY.  Temporal anti-aliasing (ST_OPT_TEMPORAL_AA) for the CPU oracle.
//
// The oracle in oracle/ restates the reference, which renders one ray through each pixel centre and composes the frame, and stays
// exactly as it is.  This library is that oracle (oracle.cpp compiled unchanged into this translation unit) plus the rule of
// DESIGN.md §2 "Temporal anti-aliasing" in the oracle's own arithmetic:
//   - orc_taa_jitter / orc_taa_set_cameras: J(f) and the jittered cameras of a frame (the projection jittered before the camera is
//     serialised), put in place of the camera state's unjittered ones for the frame;
//   - orc_taa_resolve: the resolve over the composed frame the unchanged composition pass left in `output`, against the camera's
//     history, writing the new history and the resolved `output`;
//   - orc_taa_resolve_arrays: the same resolve over caller-supplied inputs (a device's own G-buffer, signals and history).
// oracle_taa/pyoracle_taa.py steps a frame pass by pass and calls these where the device jitters and resolves.
#include "../oracle/oracle.cpp"

namespace {
using namespace orc;

// Test-only mistakes (tests/test_temporal_aa.py shows that the float64 bound catches each): 0 = the rule.
enum { MUT_NONE = 0, MUT_NO_JDIFF = 1, MUT_Y_SIGN = 2, MUT_CLAMP = 3, MUT_NO_TONEMAP = 4, MUT_FIXED_ALPHA = 5, MUT_BILINEAR = 6, MUT_SKY_POINT = 7 };

const float kClipEps = 1e-8f;

double radical_inverse(u32 k, u32 base) {
    const double inv = 1.0 / (double)base;
    double r = 0.0, f = inv;
    for (; k > 0u; k /= base) { r += f * (double)(k % base); f *= inv; }
    return r;
}
V2 jitter(u32 frame) {
    const u32 k = ((frame - 1u) % 16u) + 1u;
    return v2((float)radical_inverse(k, 2u) - 0.5f, (float)radical_inverse(k, 3u) - 0.5f);
}
Camera jittered(const M4& transform, const M4& projection, u32 w, u32 h, V2 j, int mutation) {
    M4 p = projection;
    const float dx = (-2.0f * j.x) / (float)w, dy = (mutation == MUT_Y_SIGN ? -2.0f : 2.0f) * j.y / (float)h;
    for (int c = 0; c < 4; c++) { p.c[c].x = p.c[c].x + dx * p.c[c].w; p.c[c].y = p.c[c].y + dy * p.c[c].w; }
    return camera_serialize(transform, p, w, h);
}

float tmax(float a, float b) { return a > b ? a : b; }
float tmin(float a, float b) { return a < b ? a : b; }
V3 tonemap(V3 c, int mutation) { if (mutation == MUT_NO_TONEMAP) return c; const float d = 1.0f + tmax(tmax(c.x, c.y), c.z); return v3(c.x / d, c.y / d, c.z / d); }
V3 untonemap(V3 t, int mutation) { if (mutation == MUT_NO_TONEMAP) return t; const float d = 1.0f - tmax(tmax(t.x, t.y), t.z); return v3(t.x / d, t.y / d, t.z / d); }
V3 ycocg(V3 c) { return v3((0.25f * c.x + 0.5f * c.y) + 0.25f * c.z, 0.5f * c.x - 0.5f * c.z, (-0.25f * c.x + 0.5f * c.y) - 0.25f * c.z); }
V3 rgb(V3 v) { const float t = v.x - v.z; return v3(t + v.y, v.x + v.z, t - v.y); }
void cr_weights(float f, float w[4], int mutation) {
    if (mutation == MUT_BILINEAR) { w[0] = 0.0f; w[1] = 1.0f - f; w[2] = f; w[3] = 0.0f; return; }
    w[0] = f * (-0.5f + f * (1.0f - 0.5f * f));
    w[1] = 1.0f + (f * f) * (-2.5f + 1.5f * f);
    w[2] = f * (0.5f + f * (2.0f - 1.5f * f));
    w[3] = (f * f) * (-0.5f + 0.5f * f);
}
int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Per-pixel record of the resolve's discrete choices and intermediate values, for the float64 restatement (tests/ref64_taa.py):
// q.x, q.y, valid (0/1), n, clip engaged (0/1), clip factor m, h (3), t (3), box lo (3), box hi (3), composed colour c (3), 0
const int kProbeWords = 24;

// The resolve (kernels.cu k_taa_resolve), over the composed frame `comp` (linear HDR) with G-buffer depth d0[i].x
void resolve(int w, int h, const V4* comp, const V4* d0, const V4* vel, const Camera& curr, const Camera& prev, V4 jit,
             const V4* hist_in, V4* hist_out, V4* out, int mutation, float* probe) {
#pragma omp parallel for schedule(dynamic, 4)
    for (int py = 0; py < h; py++) for (int px = 0; px < w; px++) {
        const size_t i = (size_t)py * w + px;
        auto tap = [&](int dx, int dy) { return tonemap(xyz(comp[(size_t)clampi(py + dy, 0, h - 1) * w + clampi(px + dx, 0, w - 1)]), mutation); };
        const V3 t = tap(0, 0);
        V3 lo = ycocg(tap(-1, -1)), hi = lo;
        for (int k = 1; k < 9; k++) {
            const V3 v = ycocg(tap(k % 3 - 1, k / 3 - 1));
            lo = v3(tmin(lo.x, v.x), tmin(lo.y, v.y), tmin(lo.z, v.z)); hi = v3(tmax(hi.x, v.x), tmax(hi.y, v.y), tmax(hi.z, v.z));
        }
        const float W = curr.screen.x, H = curr.screen.y;
        V2 q; bool ok = true;
        const float djx = mutation == MUT_NO_JDIFF ? 0.0f : jit.x - jit.z, djy = mutation == MUT_NO_JDIFF ? 0.0f : jit.y - jit.w;
        if (d0[i].x != 0.0f) {
            q = v2((((float)px + 0.5f) - vel[i].x) - djx, (((float)py + 0.5f) - vel[i].y) - djy);
        } else {
            const float sx = ((float)px + 0.5f) - jit.x, sy = ((float)py + 0.5f) - jit.y;
            const float nx = sx * 2.0f / W - 1.0f, ny = -(sy * 2.0f / H - 1.0f);
            const V3 far_plane = project_point3(curr.ndc_to_world, v3(nx, ny, F32_EPSILON)), near_plane = project_point3(curr.ndc_to_world, v3(nx, ny, 1.0f));
            const V3 d = normalize(far_plane - near_plane);
            const V4 clip = mul(prev.projection_view, mutation == MUT_SKY_POINT ? v4(near_plane + d, 1.0f) : v4(d, 0.0f));
            const V2 s = camera_clip_to_screen(prev, clip);
            q = v2(s.x + jit.z, s.y + jit.w);
            ok = clip.w > 0.0f;
        }
        ok = ok && q.x >= 0.0f && q.y >= 0.0f && q.x < W && q.y < H;
        float n = 0.0f;
        if (ok) n = hist_in[(size_t)(u32)floor_(q.y) * w + (u32)floor_(q.x)].w;
        V3 hh = t; bool engaged = false; float m = 0.0f;
        if (n > 0.0f) {
            const float ux = q.x - 0.5f, uy = q.y - 0.5f, fx0 = floor_(ux), fy0 = floor_(uy);
            float wx[4], wy[4];
            cr_weights(ux - fx0, wx, mutation); cr_weights(uy - fy0, wy, mutation);
            const int ix = (int)fx0 - 1, iy = (int)fy0 - 1;
            hh = v3s(0.0f);
            for (int j = 0; j < 4; j++) {
                const size_t yy = (size_t)clampi(iy + j, 0, h - 1);
                V3 row = v3s(0.0f);
                for (int k = 0; k < 4; k++) row = row + wx[k] * xyz(hist_in[yy * w + clampi(ix + k, 0, w - 1)]);
                hh = hh + wy[j] * row;
            }
            if (mutation == MUT_CLAMP) {
                const V3 y = ycocg(hh);
                const V3 c = v3(tmin(tmax(y.x, lo.x), hi.x), tmin(tmax(y.y, lo.y), hi.y), tmin(tmax(y.z, lo.z), hi.z));
                engaged = c.x != y.x || c.y != y.y || c.z != y.z;
                if (engaged) hh = rgb(c);
            } else {
                const V3 c = 0.5f * (hi + lo), e = 0.5f * (hi - lo) + v3s(kClipEps);
                const V3 d = ycocg(hh) - c;
                m = tmax(tmax(abs_(d.x / e.x), abs_(d.y / e.y)), abs_(d.z / e.z));
                engaged = m > 1.0f;
                if (engaged) hh = rgb(c + d / m);
            }
        } else n = 0.0f;
        const float a = 1.0f / (n + 1.0f), alpha = mutation == MUT_FIXED_ALPHA ? (n > 0.0f ? 0.1f : 1.0f) : (a > 0.1f ? a : 0.1f);
        const V3 r = (1.0f - alpha) * hh + alpha * t;
        const float n1 = n + 1.0f;
        hist_out[i] = v4(r, n1 < 16.0f ? n1 : 16.0f);
        out[i] = v4(untonemap(r, mutation), 1.0f);
        if (probe) {
            float* pr = probe + i * kProbeWords;
            const float v[kProbeWords] = {q.x, q.y, ok ? 1.0f : 0.0f, n, engaged ? 1.0f : 0.0f, m, hh.x, hh.y, hh.z, t.x, t.y, t.z, lo.x, lo.y, lo.z, hi.x, hi.y, hi.z, comp[i].x, comp[i].y, comp[i].z, 0.0f, 0.0f, 0.0f};
            for (int k = 0; k < kProbeWords; k++) pr[k] = v[k];
        }
    }
}

M4 m4(const float* f) { M4 m; std::memcpy(&m, f, 64); return m; }

}  // namespace

extern "C" {

void orc_taa_jitter(unsigned frame, float* out2) { const V2 j = jitter(frame); out2[0] = j.x; out2[1] = j.y; }

// Puts the jittered cameras of the camera's current frame in place: curr = the camera's own matrices jittered with J(f), prev =
// (prev_transform, prev_projection) jittered with J(f - 1); jitter = 0 restores the unjittered ones.  Returns the frame id.
int orc_taa_set_cameras(void* e, int cam, const float* prev_transform16, const float* prev_projection16, int jitter_on, int mutation) {
    Engine* en = (Engine*)e;
    Engine::Cam* c = en->cameras[cam];
    const HostCamera& hc = c->cam;
    if (!jitter_on) {
        c->st.curr_camera = camera_serialize(hc.transform, hc.projection, hc.w, hc.h);
        c->st.prev_camera = camera_serialize(m4(prev_transform16), m4(prev_projection16), hc.w, hc.h);
    } else {
        c->st.curr_camera = jittered(hc.transform, hc.projection, hc.w, hc.h, jitter(c->frame), mutation);
        c->st.prev_camera = jittered(m4(prev_transform16), m4(prev_projection16), hc.w, hc.h, jitter(c->frame - 1u), mutation);
    }
    return (int)c->frame;
}

// The resolve of the camera's current frame: `output` holds the composed frame (the composition step ran), hist = the camera's two
// history buffers (w * h * 4 floats each), a / b by frame parity as on the device.  probe (optional): kProbeWords floats per pixel.
int orc_taa_resolve(void* e, int cam, float* hist_a, float* hist_b, int mutation, float* probe) {
    Engine* en = (Engine*)e;
    Engine::Cam* c = en->cameras[cam];
    CamState& cs = c->st;
    const int cur = (c->frame % 2u) == 1u ? 1 : 0;
    V4* hist[2] = {(V4*)hist_a, (V4*)hist_b};
    const V2 j = jitter(c->frame), pj = jitter(c->frame - 1u);
    std::vector<V4> comp = cs.output;
    resolve(cs.w, cs.h, comp.data(), cs.prim_gbuffer_d0[cur].data(), cs.velocity_map.data(), cs.curr_camera, cs.prev_camera, v4(j.x, j.y, pj.x, pj.y),
            hist[cur ^ 1], hist[cur], cs.output.data(), mutation, probe);
    return 0;
}

// The resolve over caller-supplied inputs: the frame is composed by the unchanged composition pass from d0 / d1 (the current G-buffer),
// the final DI and GI diffuse signals, the specular samples and the reference colours; cameras are 40-float GpuCamera records (the
// jittered ones), jit = (J(f), J(f - 1)).  Writes hist_out and out (w * h * 4 floats each).
int orc_taa_resolve_arrays(int w, int h, int mode, int cur, const float* d0, const float* d1, const float* di_diff, const float* di_spec, const float* gi_diff,
                           const float* gi_spec, const float* ref_colors, const float* vel, const float* cam_curr, const float* cam_prev, const float* jit4,
                           const float* hist_in, float* hist_out, float* out) {
    CamState cs; cs.init(w, h);
    const size_t n = (size_t)w * h;
    auto put = [&](Buf& b, const float* src) { std::memcpy(b.data(), src, n * 16); };
    put(cs.prim_gbuffer_d0[cur], d0); put(cs.prim_gbuffer_d1[cur], d1);
    put(cs.di_diff_curr_colors, di_diff); put(cs.di_spec_samples, di_spec); put(cs.gi_diff_curr_colors, gi_diff); put(cs.gi_spec_samples, gi_spec);
    put(cs.ref_colors, ref_colors); put(cs.velocity_map, vel);
    std::memcpy(&cs.curr_camera, cam_curr, 160); std::memcpy(&cs.prev_camera, cam_prev, 160);
    pass_frame_composition(cs, cur == 1, (u32)mode, true, true);
    resolve(w, h, cs.output.data(), cs.prim_gbuffer_d0[cur].data(), cs.velocity_map.data(), cs.curr_camera, cs.prev_camera, v4(jit4[0], jit4[1], jit4[2], jit4[3]),
            (const V4*)hist_in, (V4*)hist_out, (V4*)out, MUT_NONE, nullptr);
    return 0;
}

}  // extern "C"
