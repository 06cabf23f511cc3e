/* rt_oracle_temporal.cpp — rtDenoiseTemporal (include/rt_b200.h) for the oracle, built around it rather than inside it.
 * Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with rtDenoise
 * (rt_oracle_denoise.cpp, which includes the rest) and adds the temporal denoiser, restated from the header's statement with orc::
 * arithmetic, one pixel and one tap at a time in the stated order, with its own history per context.
 *
 * orTemporalImages is one temporal step on caller-supplied arrays (the current colour and features, both cameras, the history in and
 * out), so that synthetic images and cameras (NaN depths, points behind the previous camera, singular matrices, ...) can be compared
 * with the product, whose input images the tests write through rtGetDevicePointer.
 *
 * Three entry points the denoise layer already wraps have to reach the temporal state as well: rtDestroy, rtResize (a new size zeroes
 * TemporalFrame and discards the history) and rtReadback (one new name).  As that layer does with the layers below it, the three
 * wrappers it defines are declared here first with an assembler name of their own (orDen_*), and the wrappers at the end of this file
 * get the plain symbols the ABI exports; the warning about the denoise layer's own labels is silenced around the include. */
struct RtContext;
extern "C" {
int orDenoise_rtDestroy(RtContext* c) __asm__("orDen_rtDestroy");
int orDenoise_rtResize(RtContext* c, int w, int h) __asm__("orDen_rtResize");
int orDenoise_rtReadback(RtContext* c, const char* tex, float* dst, unsigned long bytes) __asm__("orDen_rtReadback");
}
#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wpragmas"
#include "rt_oracle_denoise.cpp"
#pragma GCC diagnostic pop

namespace {

// A camera as the temporal denoiser sees it: CamLocalToWorldMatrix (column-major) and ViewParams
struct TemporalCamera { float m[16]; float vp[3]; };

// History planes, W*H float4 each: guide (n, z; z = NaN: no record), moments (m1, m2, len, object bits), colour history
struct TemporalHistory { std::vector<float> guide, mom, colour; };

struct TemporalState
{
    std::vector<float> frame;                // "TemporalFrame"; empty until the first rtDenoiseTemporal
    TemporalHistory hist;
    bool history = false;
    TemporalCamera cam;
};

std::mutex g_tmpMutex;
std::map<const RtContext*, TemporalState> g_temporal;

struct TemporalArgs { int iterations; float sigmaL, sigmaN, sigmaZ, alpha; float invN, invZ, invL; };

int temporalArgs(int iterations, const float sigma[3], float alpha, TemporalArgs& a)
{
    if (iterations < 1 || iterations > RT_DENOISE_MAX_ITERATIONS) return RT_E_INVALID;
    for (int i = 0; i < 3; i++)
        if (!(sigma[i] > 0.0f) || !finite1(sigma[i])) return RT_E_INVALID;
    if (!(alpha > 0.0f && alpha <= 1.0f)) return RT_E_INVALID;
    a.iterations = iterations; a.sigmaL = sigma[0]; a.sigmaN = sigma[1]; a.sigmaZ = sigma[2]; a.alpha = alpha;
    a.invN = 1.0f / (sigma[1] * sigma[1]);
    a.invZ = 1.0f / sigma[2];
    a.invL = 1.0f / sigma[0];
    if (!finite1(a.invN) || !finite1(a.invZ) || !finite1(a.invL)) return RT_E_INVALID;
    return RT_OK;
}

float lum(float3 v) { return (0.2126f * v.x + 0.7152f * v.y) + 0.0722f * v.z; }
int asInt(float v) { int i; memcpy(&i, &v, 4); return i; }
float asFloat(int i) { float v; memcpy(&v, &i, 4); return v; }

// One call: colour = W*H float4 (FrameRender), feats = FeatureFrame, prev = NULL (or histIn NULL) for no history.  Writes histOut,
// out (DenoisedRender) and frame (TemporalFrame).
void temporalStep(int W, int H, const float* colour, const RtPixelFeatures* feats, const TemporalCamera& cur, const TemporalCamera* prev,
                  const TemporalHistory* histIn, TemporalHistory& histOut, const TemporalArgs& A, float* out, float* frame)
{
    const size_t n = (size_t)W * H;
    const float NaN = orc::u2f(0x7fc00000u);
    histOut.guide.assign(n * 4, 0.0f); histOut.mom.assign(n * 4, 0.0f); histOut.colour.assign(n * 4, 0.0f);
    std::vector<float3> e(n), m(n), nrm(n);
    std::vector<float> z(n), var(n, 0.0f);
    std::vector<char> bg(n);

    // the mode: no history, a still camera, or a reprojection through the previous camera's inverse
    int mode = 0;
    float inv[12] = {}, kx = 0.0f, ky = 0.0f;
    if (prev && histIn)
    {
        if (memcmp(prev->m, cur.m, 64) == 0 && memcmp(prev->vp, cur.vp, 12) == 0) mode = 2;
        else
        {
            mode = 1;
            const float* M = prev->m;
            const double a00 = M[0], a01 = M[4], a02 = M[8], a10 = M[1], a11 = M[5], a12 = M[9], a20 = M[2], a21 = M[6], a22 = M[10];
            const double c[3][3] = {{a11 * a22 - a12 * a21, a12 * a20 - a10 * a22, a10 * a21 - a11 * a20},
                                    {a02 * a21 - a01 * a22, a00 * a22 - a02 * a20, a01 * a20 - a00 * a21},
                                    {a01 * a12 - a02 * a11, a02 * a10 - a00 * a12, a00 * a11 - a01 * a10}};
            const double det = (a00 * c[0][0] + a01 * c[0][1]) + a02 * c[0][2];
            const double t[3] = {M[12], M[13], M[14]};
            for (int r = 0; r < 3; r++)
            {
                double R[3];
                for (int k = 0; k < 3; k++) { R[k] = c[k][r] / det; inv[4 * r + k] = (float)R[k]; }
                inv[4 * r + 3] = (float)-((R[0] * t[0] + R[1] * t[1]) + R[2] * t[2]);
            }
            kx = prev->vp[2] / prev->vp[0]; ky = prev->vp[2] / prev->vp[1];
        }
    }
    orc::float4x4 cam;
    memcpy(cam.m, cur.m, 64);
    const float3 VP = mk3(cur.vp);

    // 1-3: demodulation, reprojection, history, integration
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            const size_t p = (size_t)y * W + x;
            const RtPixelFeatures& f = feats[p];
            const float3 cc = mk3(colour + 4 * p), a = mk3(f.albedo);
            nrm[p] = mk3(f.normal); z[p] = f.dst;
            m[p] = mk3(orc::max(a.x, 0.00390625f), orc::max(a.y, 0.00390625f), orc::max(a.z, 0.00390625f));
            e[p] = mk3(cc.x / m[p].x, cc.y / m[p].y, cc.z / m[p].z);
            bool b = f.object == -1;
            const float vals[13] = {cc.x, cc.y, cc.z, a.x, a.y, a.z, nrm[p].x, nrm[p].y, nrm[p].z, z[p], e[p].x, e[p].y, e[p].z};
            for (float v : vals) b = b || !finite1(v);
            bg[p] = b;
            float* o = out + 4 * p; float* fr = frame + 4 * p;
            if (b)
            {
                o[0] = cc.x; o[1] = cc.y; o[2] = cc.z; o[3] = 1.0f;
                histOut.guide[4 * p + 3] = NaN;
                fr[0] = NaN; fr[1] = NaN; fr[2] = 0.0f; fr[3] = 0.0f;
                continue;
            }
            const float l = lum(e[p]);
            float px = NaN, py = NaN, zexp = 0.0f;
            if (mode == 2) { px = (float)x; py = (float)y; zexp = z[p]; }
            else if (mode == 1)
            {
                const float2 uv = mk2((float)(uint)x / ((float)(uint)W - 1.0f), (float)(uint)y / ((float)(uint)H - 1.0f));
                const float3 camOrigin = mul_xyz(cam, mk4(mk3(0.0f, 0.0f, 0.0f), 1.0f));
                const float3 focusPoint = mul_xyz(cam, mk4(mk3(uv.x - 0.5f, uv.y - 0.5f, 1.0f) * VP, 1.0f));
                const float3 d = normalize(focusPoint - camOrigin);
                const float3 X = mk3(camOrigin.x + d.x * z[p], camOrigin.y + d.y * z[p], camOrigin.z + d.z * z[p]);
                float L[3];
                for (int r = 0; r < 3; r++) L[r] = ((inv[4 * r] * X.x + inv[4 * r + 1] * X.y) + inv[4 * r + 2] * X.z) + inv[4 * r + 3];
                if (L[2] > 0.0f)
                {
                    const float u = (L[0] / L[2]) * kx + 0.5f, v = (L[1] / L[2]) * ky + 0.5f;
                    const float qx = u * (float)(W - 1), qy = v * (float)(H - 1);
                    const float dx = X.x - prev->m[12], dy = X.y - prev->m[13], dz = X.z - prev->m[14];
                    const float ze = sqrtf((dx * dx + dy * dy) + dz * dz);
                    const float all[11] = {X.x, X.y, X.z, L[0], L[1], L[2], u, v, qx, qy, ze};
                    bool ok = true;
                    for (float v2 : all) ok = ok && finite1(v2);
                    if (ok) { px = qx; py = qy; zexp = ze; }
                }
            }
            float sw = 0.0f, sc[3] = {0.0f, 0.0f, 0.0f}, s1 = 0.0f, s2 = 0.0f, lenH = 0.0f;
            if (px > -1.0f && px < (float)W && py > -1.0f && py < (float)H)
            {
                const float fx0 = floorf(px), fy0 = floorf(py);
                const int ix = (int)fx0, iy = (int)fy0;
                const float fx = px - fx0, fy = py - fy0;
                const float wx[2] = {1.0f - fx, fx}, wy[2] = {1.0f - fy, fy};
                for (int t = 0; t < 4; t++)
                {
                    const int qx = ix + (t & 1), qy = iy + (t >> 1);
                    const float w = wx[t & 1] * wy[t >> 1];
                    if (w == 0.0f || qx < 0 || qy < 0 || qx >= W || qy >= H) continue;
                    const size_t q = (size_t)qy * W + qx;
                    const float* g = &histIn->guide[4 * q];
                    const float* Mq = &histIn->mom[4 * q];
                    if (g[3] != g[3]) continue;
                    if (asInt(Mq[3]) != f.object) continue;
                    if (!(fabsf(g[3] - zexp) <= RT_TEMPORAL_TAU_Z * zexp)) continue;
                    if (!(((nrm[p].x * g[0] + nrm[p].y * g[1]) + nrm[p].z * g[2]) >= RT_TEMPORAL_TAU_N)) continue;
                    const float* h = &histIn->colour[4 * q];
                    sw = sw + w;
                    for (int k = 0; k < 3; k++) sc[k] = sc[k] + w * h[k];
                    s1 = s1 + w * Mq[0]; s2 = s2 + w * Mq[1];
                    lenH = orc::max(lenH, Mq[2]);
                }
            }
            float3 col = e[p];
            float m1 = l, m2 = l * l, len = 1.0f;
            if (sw > 0.0f)
            {
                len = orc::min(lenH + 1.0f, (float)RT_TEMPORAL_MAX_HISTORY);
                const float al = orc::max(A.alpha, 1.0f / len);
                const float h[3] = {sc[0] / sw, sc[1] / sw, sc[2] / sw}, h1 = s1 / sw, h2 = s2 / sw;
                col = mk3(h[0] + al * (e[p].x - h[0]), h[1] + al * (e[p].y - h[1]), h[2] + al * (e[p].z - h[2]));
                m1 = h1 + al * (l - h1);
                m2 = h2 + al * (l * l - h2);
            }
            e[p] = col;
            float* g = &histOut.guide[4 * p]; g[0] = nrm[p].x; g[1] = nrm[p].y; g[2] = nrm[p].z; g[3] = z[p];
            float* Mo = &histOut.mom[4 * p]; Mo[0] = m1; Mo[1] = m2; Mo[2] = len; Mo[3] = asFloat(f.object);
            fr[0] = px; fr[1] = py; fr[2] = len;
            o[0] = m[p].x; o[1] = m[p].y; o[2] = m[p].z; o[3] = 1.0f;
        }

    // 4: the variance
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            const size_t p = (size_t)y * W + x;
            if (bg[p]) continue;
            const float* Mp = &histOut.mom[4 * p];
            float v;
            if (Mp[2] >= 4.0f) v = orc::max(Mp[1] - Mp[0] * Mp[0], 0.0f);
            else
            {
                const float rz = A.invZ / z[p];
                float sw = 0.0f, s1 = 0.0f, s2 = 0.0f;
                for (int j = -3; j <= 3; j++)
                    for (int i = -3; i <= 3; i++)
                    {
                        const int qx = x + i, qy = y + j;
                        if (qx < 0 || qy < 0 || qx >= W || qy >= H) continue;
                        const size_t q = (size_t)qy * W + qx;
                        if (bg[q]) continue;
                        const float* Mq = &histOut.mom[4 * q];
                        float w = 1.0f;
                        if (i != 0 || j != 0)
                        {
                            const float3 dn = nrm[p] - nrm[q];
                            const float t = (z[p] - z[q]) * rz;
                            const float D = (fabsf(Mp[0] - Mq[0]) * A.invL + ((dn.x * dn.x + dn.y * dn.y) + dn.z * dn.z) * A.invN) + t * t;
                            w = D <= 103.972076416015625f ? orc::exp(-D) : 0.0f;
                            if (w == 0.0f) continue;
                        }
                        sw = sw + w;
                        s1 = s1 + w * Mq[0]; s2 = s2 + w * Mq[1];
                    }
                const float a1 = s1 / sw, a2 = s2 / sw;
                v = orc::max(a2 - a1 * a1, 0.0f) * (4.0f / Mp[2]);
            }
            var[p] = v;
            frame[4 * p + 3] = v;
        }

    // 5: the variance-guided a-trous passes
    static const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    static const float k1[3] = {0.25f, 0.5f, 0.25f};
    for (int k = 0; k < A.iterations; k++)
    {
        const int s = 1 << k;
        const float rd[3] = {0.0f, 1.0f / (float)s, 1.0f / (float)(2 * s)};
        std::vector<float3> next(e);
        std::vector<float> nextVar(var);
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++)
            {
                const size_t p = (size_t)y * W + x;
                if (bg[p]) continue;
                auto inside = [&](long long qx, long long qy) { return qx >= 0 && qy >= 0 && qx < W && qy < H && !bg[(size_t)qy * W + (size_t)qx]; };
                float sk = 0.0f, sg = 0.0f;
                for (int j = -1; j <= 1; j++)
                    for (int i = -1; i <= 1; i++)
                    {
                        const long long qx = x + i, qy = y + j;                  // immediate neighbours at every step
                        if (!inside(qx, qy)) continue;
                        const float kk = k1[i + 1] * k1[j + 1];
                        sk = sk + kk; sg = sg + kk * var[(size_t)qy * W + (size_t)qx];
                    }
                const float kL = 1.0f / (A.sigmaL * sqrtf(sg / sk) + RT_TEMPORAL_EPSILON);
                const float lp = lum(e[p]);
                const float rz = A.invZ / z[p];
                float sw = 0.0f, sr = 0.0f, sgr = 0.0f, sb = 0.0f, sv = 0.0f;
                for (int j = -2; j <= 2; j++)
                    for (int i = -2; i <= 2; i++)
                    {
                        const long long qx = x + (long long)s * i, qy = y + (long long)s * j;
                        if (!inside(qx, qy)) continue;
                        const size_t q = (size_t)qy * W + (size_t)qx;
                        float w;
                        if (i == 0 && j == 0) w = 0.140625f;
                        else
                        {
                            const float3 dn = nrm[p] - nrm[q];
                            const int d = std::max(std::abs(i), std::abs(j));
                            const float t = ((z[p] - z[q]) * rz) * rd[d];
                            const float D = (fabsf(lp - lum(e[q])) * kL + ((dn.x * dn.x + dn.y * dn.y) + dn.z * dn.z) * A.invN) + t * t;
                            w = D <= 103.972076416015625f ? (h[i + 2] * h[j + 2]) * orc::exp(-D) : 0.0f;
                            if (w == 0.0f) continue;
                        }
                        sw = sw + w;
                        sr = sr + w * e[q].x; sgr = sgr + w * e[q].y; sb = sb + w * e[q].z;
                        sv = sv + (w * w) * var[q];
                    }
                next[p] = mk3(sr / sw, sgr / sw, sb / sw);
                nextVar[p] = sv / (sw * sw);
                if (k == 0) { float* hc = &histOut.colour[4 * p]; hc[0] = next[p].x; hc[1] = next[p].y; hc[2] = next[p].z; }
            }
        e.swap(next);
        var.swap(nextVar);
    }
    for (size_t p = 0; p < n; p++)
        if (!bg[p]) { out[4 * p] = e[p].x * m[p].x; out[4 * p + 1] = e[p].y * m[p].y; out[4 * p + 2] = e[p].z * m[p].z; out[4 * p + 3] = 1.0f; }
}

} // namespace

extern "C" {

/* One temporal step on caller arrays.  colour = W*H float4 (FrameRender), features = W*H RtPixelFeatures, cur / prev = 19 floats each
 * (CamLocalToWorldMatrix column-major, ViewParams); prev and histIn NULL: no history (the first call, resetHistory = 1, a resize).
 * histIn / histOut = W*H*12 floats: the guide, moments and colour-history planes of W*H float4 each (histOut of one step is histIn of
 * the next).  params = (sigmaLuminance, sigmaNormal, sigmaDepth, alpha).  out = W*H float4 (DenoisedRender), frame = W*H float4
 * (TemporalFrame).  RT_E_INVALID for the arguments rtDenoiseTemporal refuses. */
int orTemporalImages(int W, int H, const float* colour, const void* features, const float* cur, const float* prev, const float* histIn,
                     float* histOut, int iterations, const float params[4], float* out, float* frame)
{
    if (W <= 0 || H <= 0 || !colour || !features || !cur || !histOut || !params || !out || !frame || (!prev) != (!histIn)) return RT_E_INVALID;
    TemporalArgs A;
    if (temporalArgs(iterations, params, params[3], A) != RT_OK) return RT_E_INVALID;
    const size_t n = (size_t)W * H;
    TemporalCamera c, pc;
    memcpy(c.m, cur, 64); memcpy(c.vp, cur + 16, 12);
    TemporalHistory in, hout;
    if (prev)
    {
        memcpy(pc.m, prev, 64); memcpy(pc.vp, prev + 16, 12);
        in.guide.assign(histIn, histIn + 4 * n); in.mom.assign(histIn + 4 * n, histIn + 8 * n); in.colour.assign(histIn + 8 * n, histIn + 12 * n);
    }
    temporalStep(W, H, colour, (const RtPixelFeatures*)features, c, prev ? &pc : nullptr, prev ? &in : nullptr, hout, A, out, frame);
    memcpy(histOut, hout.guide.data(), n * 16); memcpy(histOut + 4 * n, hout.mom.data(), n * 16); memcpy(histOut + 8 * n, hout.colour.data(), n * 16);
    return RT_OK;
}

int rtDenoiseTemporal(RtContext* c, int iterations, float sigmaLuminance, float sigmaNormal, float sigmaDepth, float alpha, int resetHistory)
{
    if (!c) return RT_E_INVALID;
    const float sigma[3] = {sigmaLuminance, sigmaNormal, sigmaDepth};
    TemporalArgs A;
    if (temporalArgs(iterations, sigma, alpha, A) != RT_OK || (resetHistory != 0 && resetHistory != 1))
        return fail(c, RT_E_INVALID, "rtDenoiseTemporal: bad argument");
    int rc = cameraImage(c, "rtDenoiseTemporal"); if (rc != RT_OK) return rc;
    const FeatureState& fs = featureState(c);
    if (fs.frame.empty()) return fail(c, RT_E_STATE, "rtDenoiseTemporal: no rtDispatchFeatures yet");
    if (c->tileWorld > 1) return fail(c, RT_E_STATE, "rtDenoiseTemporal: the images of a context with rtSetTile world > 1 hold its own bands only");
    const size_t n = (size_t)c->width * c->height;
    TemporalCamera cam;
    memcpy(cam.m, c->sh.CamLocalToWorldMatrix.m, 64);
    cam.vp[0] = c->sh.ViewParams.x; cam.vp[1] = c->sh.ViewParams.y; cam.vp[2] = c->sh.ViewParams.z;
    std::vector<float> out(n * 4), frame(n * 4);
    std::lock_guard<std::mutex> lock(g_tmpMutex);
    TemporalState& ts = g_temporal[c];
    const bool use = ts.history && !resetHistory;
    TemporalHistory next;
    temporalStep(c->width, c->height, c->frame.data(), fs.frame.data(), cam, use ? &ts.cam : nullptr, use ? &ts.hist : nullptr, next, A,
                 out.data(), frame.data());
    ts.hist.guide.swap(next.guide); ts.hist.mom.swap(next.mom); ts.hist.colour.swap(next.colour);
    ts.history = true; ts.cam = cam;
    ts.frame.swap(frame);
    std::lock_guard<std::mutex> lock2(g_denMutex);
    g_denoised[c].swap(out);
    return RT_OK;
}

/* ---- the three wrapped entry points: defined under a name of their own, exported under the ABI's ------------------------------------ */
int orTemporal_rtDestroy(RtContext* c) __asm__("rtDestroy");
int orTemporal_rtResize(RtContext* c, int w, int h) __asm__("rtResize");
int orTemporal_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes) __asm__("rtReadback");

int orTemporal_rtDestroy(RtContext* c)
{
    { std::lock_guard<std::mutex> lock(g_tmpMutex); g_temporal.erase(c); }
    return orDenoise_rtDestroy(c);
}

int orTemporal_rtResize(RtContext* c, int w, int h)
{
    const bool newSize = c && (w != c->width || h != c->height);
    const int rc = orDenoise_rtResize(c, w, h);
    if (rc == RT_OK && newSize)
    {
        std::lock_guard<std::mutex> lock(g_tmpMutex);
        auto it = g_temporal.find(c);
        if (it != g_temporal.end())
        {
            it->second.frame.assign((size_t)w * h * 4, 0.0f);
            it->second.history = false;
            it->second.hist = TemporalHistory();
        }
    }
    return rc;
}

int orTemporal_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    if (!(c && tex && dst && std::string(tex) == "TemporalFrame")) return orDenoise_rtReadback(c, tex, dst, bytes);
    std::lock_guard<std::mutex> lock(g_tmpMutex);
    auto it = g_temporal.find(c);
    if (it == g_temporal.end() || it->second.frame.empty()) return fail(c, RT_E_STATE, "rtReadback: no rtDenoiseTemporal yet");
    if (bytes != it->second.frame.size() * 4) return fail(c, RT_E_INVALID, "rtReadback: bytes must equal W*H*16");
    memcpy(dst, it->second.frame.data(), bytes);
    return RT_OK;
}

} // extern "C"
