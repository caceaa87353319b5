/*
 * JNI binding of libkspecmc.so (include/kspecmc.h).
 *
 * NOT COMPILED IN THIS REPOSITORY'S ENVIRONMENT: the build image has no JDK (no javac, no jni.h)
 * and no tla2tools.jar.  The sources are the reference-side binding a TLC maintainer would add;
 * the tested boundary is the C ABI itself (tests/test_cabi.py, tests/test_gpu_parity.py).
 * Build (with a JDK): see java/README.md.
 */
package tlc2.gpu;

public final class Native {
    static {
        System.loadLibrary("kspecmc_jni"); // java/jni/kspecmc_jni.c, links libkspecmc.so
    }

    private Native() {}

    /** kmc_create: returns an opaque context handle, throws RuntimeException with kmc_strerror on failure. */
    public static native long create(String modelLibrary, String optionsJson);

    /** kmc_destroy */
    public static native void destroy(long ctx);

    /** kmc_run: blocking full BFS; returns the KMC_* status code. */
    public static native int run(long ctx);

    /** kmc_stats: {distinct, generated, queue, depth, deadlocks, outOfModel, probes, levels, complete, initGenerated,
     *  initCandidates}. */
    public static native long[] stats(long ctx);

    /** kmc_violation: {kind, invariantIndex, level, traceLength, fingerprint} or null when kind == 0. */
    public static native long[] violation(long ctx);

    /** kmc_trace_state: packed state words of the i-th trace state; actionOut[0] receives the action id. */
    public static native long[] traceState(long ctx, int i, int[] actionOut);

    /** kmc_fpset_put: seen[i] = fingerprint was already present (FPSet.put contract). */
    public static native boolean[] fpsetPut(long ctx, long[] fingerprints);

    /** kmc_fpset_contains */
    public static native boolean[] fpsetContains(long ctx, long[] fingerprints);

    /** kmc_fpset_size */
    public static native long fpsetSize(long ctx);

    /** kmc_strerror */
    public static native String strerror(long ctx, int code);
}
