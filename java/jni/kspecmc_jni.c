/* JNI shim: Java_tlc2_gpu_Native_* -> kmc_* (include/kspecmc.h).
 * NOT COMPILED HERE: this image has no JDK (jni.h).  With a JDK:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude \
 *       java/jni/kspecmc_jni.c -Lbuild -lkspecmc -o build/libkspecmc_jni.so
 * No callbacks into the JVM are made from engine threads; every call copies plain arrays. */
#include <jni.h>
#include <stdlib.h>
#include <string.h>

#include "kspecmc.h"

static void throw_rt(JNIEnv* env, const char* msg) {
  jclass c = (*env)->FindClass(env, "java/lang/RuntimeException");
  if (c) (*env)->ThrowNew(env, c, msg);
}

JNIEXPORT jlong JNICALL Java_tlc2_gpu_Native_create(JNIEnv* env, jclass cls, jstring lib, jstring opts) {
  const char* l = (*env)->GetStringUTFChars(env, lib, NULL);
  const char* o = opts ? (*env)->GetStringUTFChars(env, opts, NULL) : NULL;
  kmc_ctx* ctx = NULL;
  int rc = kmc_create(l, o, &ctx);
  (*env)->ReleaseStringUTFChars(env, lib, l);
  if (o) (*env)->ReleaseStringUTFChars(env, opts, o);
  if (rc != KMC_OK) {
    throw_rt(env, kmc_strerror(ctx, rc));
    if (ctx) kmc_destroy(ctx);
    return 0;
  }
  return (jlong)(intptr_t)ctx;
}

JNIEXPORT void JNICALL Java_tlc2_gpu_Native_destroy(JNIEnv* env, jclass cls, jlong ctx) {
  kmc_destroy((kmc_ctx*)(intptr_t)ctx);
}

JNIEXPORT jint JNICALL Java_tlc2_gpu_Native_run(JNIEnv* env, jclass cls, jlong ctx) {
  return kmc_run((kmc_ctx*)(intptr_t)ctx);
}

JNIEXPORT jlongArray JNICALL Java_tlc2_gpu_Native_stats(JNIEnv* env, jclass cls, jlong ctx) {
  kmc_stats_t s;
  if (kmc_stats((kmc_ctx*)(intptr_t)ctx, &s) != KMC_OK) return NULL;
  jlong v[11] = {(jlong)s.distinct, (jlong)s.generated, (jlong)s.queue, (jlong)s.depth, (jlong)s.deadlocks,
                 (jlong)s.out_of_model, (jlong)s.probes, (jlong)s.levels, (jlong)s.complete,
                 (jlong)s.init_generated, (jlong)s.init_candidates};
  jlongArray a = (*env)->NewLongArray(env, 11);
  (*env)->SetLongArrayRegion(env, a, 0, 11, v);
  return a;
}

JNIEXPORT jlongArray JNICALL Java_tlc2_gpu_Native_violation(JNIEnv* env, jclass cls, jlong ctx) {
  kmc_violation_t v;
  if (kmc_violation((kmc_ctx*)(intptr_t)ctx, &v) != KMC_OK || v.kind == KMC_RESULT_OK) return NULL;
  jlong out[5] = {v.kind, v.invariant, (jlong)v.level, (jlong)v.trace_len, (jlong)v.fingerprint};
  jlongArray a = (*env)->NewLongArray(env, 5);
  (*env)->SetLongArrayRegion(env, a, 0, 5, out);
  return a;
}

JNIEXPORT jlongArray JNICALL Java_tlc2_gpu_Native_traceState(JNIEnv* env, jclass cls, jlong ctx, jint i, jintArray act) {
  kmc_model_info_t info;
  if (kmc_model_info((kmc_ctx*)(intptr_t)ctx, &info) != KMC_OK) return NULL;
  uint64_t buf[64];
  uint32_t action = 0;
  if (info.words > 64 || kmc_trace_state((kmc_ctx*)(intptr_t)ctx, (uint32_t)i, buf, 64, &action) != KMC_OK) return NULL;
  jlongArray a = (*env)->NewLongArray(env, info.words);
  (*env)->SetLongArrayRegion(env, a, 0, info.words, (const jlong*)buf);
  if (act) {
    jint av = (jint)action;
    (*env)->SetIntArrayRegion(env, act, 0, 1, &av);
  }
  return a;
}

static jbooleanArray fp_call(JNIEnv* env, jlong ctx, jlongArray fps, int put) {
  jsize n = (*env)->GetArrayLength(env, fps);
  jlong* p = (*env)->GetLongArrayElements(env, fps, NULL);
  uint8_t* out = (uint8_t*)malloc((size_t)n + 1);
  int rc = put ? kmc_fpset_put((kmc_ctx*)(intptr_t)ctx, (const uint64_t*)p, (size_t)n, out)
               : kmc_fpset_contains((kmc_ctx*)(intptr_t)ctx, (const uint64_t*)p, (size_t)n, out);
  (*env)->ReleaseLongArrayElements(env, fps, p, JNI_ABORT);
  if (rc != KMC_OK) {
    free(out);
    throw_rt(env, kmc_strerror((kmc_ctx*)(intptr_t)ctx, rc));   /* FPSet.put throws IOException in TLC */
    return NULL;
  }
  jbooleanArray a = (*env)->NewBooleanArray(env, n);
  (*env)->SetBooleanArrayRegion(env, a, 0, n, (const jboolean*)out);
  free(out);
  return a;
}

JNIEXPORT jbooleanArray JNICALL Java_tlc2_gpu_Native_fpsetPut(JNIEnv* env, jclass cls, jlong ctx, jlongArray fps) {
  return fp_call(env, ctx, fps, 1);
}
JNIEXPORT jbooleanArray JNICALL Java_tlc2_gpu_Native_fpsetContains(JNIEnv* env, jclass cls, jlong ctx, jlongArray fps) {
  return fp_call(env, ctx, fps, 0);
}
JNIEXPORT jlong JNICALL Java_tlc2_gpu_Native_fpsetSize(JNIEnv* env, jclass cls, jlong ctx) {
  uint64_t n = 0;
  kmc_fpset_size((kmc_ctx*)(intptr_t)ctx, &n);
  return (jlong)n;
}
JNIEXPORT jstring JNICALL Java_tlc2_gpu_Native_strerror(JNIEnv* env, jclass cls, jlong ctx, jint code) {
  return (*env)->NewStringUTF(env, kmc_strerror((kmc_ctx*)(intptr_t)ctx, code));
}
