/* rt_oracle_frames.cpp — rtDispatchFrames (include/rt_b200.h) for the oracle, built around it rather than inside it.  Test
 * infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with its per-pixel
 * counters (rt_oracle_pixel_stats.cpp, which includes oracle/rt_oracle.cpp unchanged) and adds the batch call as the loop the header
 * defines it by, over the wrapped rtDispatch: images, RtStats and PixelStats follow from the n single-frame dispatches. */
#include "rt_oracle_pixel_stats.cpp"

extern "C" int rtDispatchFrames(RtContext* c, int gx, int gy, int gz, int frameCount)
{
    if (!c) return RT_E_INVALID;
    const long long chain = (long long)frameCount * (c->sh.NumRaysPerPixel > 1 ? c->sh.NumRaysPerPixel : 1);
    if (frameCount < 1 || chain > RT_MAX_BATCH_SAMPLES)
        return fail(c, RT_E_INVALID, "rtDispatchFrames: frameCount must be >= 1 and frameCount * max(1, NumRaysPerPixel) at most RT_MAX_BATCH_SAMPLES");
    if (!c->sh.accumulate) return fail(c, RT_E_STATE, "rtDispatchFrames: needs accumulate = 1");
    const int F = c->sh.Frame;
    int rc = RT_OK;
    for (int k = 0; k < frameCount && rc == RT_OK; k++)
    {
        c->sh.Frame = (int)((unsigned)F + (unsigned)k);
        rc = rtDispatch(c, RT_KERNEL_RAYTRACE, gx, gy, gz);
    }
    c->sh.Frame = F;
    return rc;
}
