/* JNI shim between ch.sqooba.kao.KaoNative and include/kao.h.  UNCOMPILED here (no jni.h in the
 * image).  No JNI critical section is held across kao_solve (it blocks for the whole search). */
#include <jni.h>
#include <stdlib.h>
#include "kao.h"

JNIEXPORT jint JNICALL Java_ch_sqooba_kao_KaoNative_version(JNIEnv *env, jclass cls)
{
    (void)env; (void)cls;
    return kao_version();
}

static void kao_jni_throw(JNIEnv *env, int rc)
{
    jclass ex = (*env)->FindClass(env, "ch/sqooba/kao/KaoNative$KaoException");
    jmethodID ctor = (*env)->GetMethodID(env, ex, "<init>", "(ILjava/lang/String;)V");
    jstring msg = (*env)->NewStringUTF(env, kao_last_error());
    (*env)->Throw(env, (jthrowable)(*env)->NewObject(env, ex, ctor, rc, msg));
}

JNIEXPORT jint JNICALL Java_ch_sqooba_kao_KaoNative_solve(
    JNIEnv *env, jclass cls, jint P, jint B, jint R, jint RF, jint RFcur, jbyteArray rackOf,
    jshortArray wF, jshortArray wL, jintArray bounds, jintArray cur, jlong seed, jint rounds,
    jint roundSize, jint device, jint nGpus, jint flags, jintArray replicasOut, jlongArray statsOut)
{
    (void)cls;
    jbyte *rk = (*env)->GetByteArrayElements(env, rackOf, NULL);
    jshort *f = (*env)->GetShortArrayElements(env, wF, NULL);
    jshort *l = (*env)->GetShortArrayElements(env, wL, NULL);
    jint *bd = (*env)->GetIntArrayElements(env, bounds, NULL);
    jint *cu = (*env)->GetIntArrayElements(env, cur, NULL);
    jint *out = (*env)->GetIntArrayElements(env, replicasOut, NULL);

    kao_problem pb;
    pb.P = P; pb.B = B; pb.R = R; pb.RF = RF; pb.RFcur = RFcur;
    pb.rack_of = (const uint8_t *)rk;
    pb.wF = (const uint16_t *)f;
    pb.wL = (const uint16_t *)l;
    pb.rep_lo = (const int32_t *)bd;          pb.rep_hi = (const int32_t *)bd + B;
    pb.ldr_lo = (const int32_t *)bd + 2 * B;  pb.ldr_hi = (const int32_t *)bd + 3 * B;
    pb.rack_lo = (const int32_t *)bd + 4 * B; pb.rack_hi = (const int32_t *)bd + 4 * B + R;
    pb.ppr_lo = bd[4 * B + 2 * R];            pb.ppr_hi = bd[4 * B + 2 * R + 1];
    pb.cur = (const int32_t *)cu;
    /* nGpus > 1: the rounds are sharded over that many GPUs of this process (include/kao.h, kao_options) */
    kao_options opt = {(uint64_t)seed, (uint32_t)rounds, (uint32_t)roundSize, device, (uint32_t)flags, nGpus, 0u};
    kao_result res;
    res.replicas = (int32_t *)out;
    const int rc = kao_solve(&pb, &opt, &res);

    (*env)->ReleaseByteArrayElements(env, rackOf, rk, JNI_ABORT);
    (*env)->ReleaseShortArrayElements(env, wF, f, JNI_ABORT);
    (*env)->ReleaseShortArrayElements(env, wL, l, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, bounds, bd, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, cur, cu, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, replicasOut, out, rc < 0 ? JNI_ABORT : 0);
    if (rc < 0) {
        kao_jni_throw(env, rc);
        return rc;
    }
    jlong st[8] = {res.objective, res.violation, res.moves, (jlong)res.n_candidates,
                   res.objective_bound, res.optimal, res.rounds_run, res.n_gpus};
    (*env)->SetLongArrayRegion(env, statsOut, 0, 8, st);
    return rc;
}

/* leader-only rebalancing (kao_solve_leaders): host-side, no GPU; topicOf / fixed may be null */
JNIEXPORT jint JNICALL Java_ch_sqooba_kao_KaoNative_solveLeaders(
    JNIEnv *env, jclass cls, jint P, jint B, jint R, jint RF, jint RFcur, jbyteArray rackOf, jshortArray wF,
    jshortArray wL, jintArray bounds, jintArray cur, jintArray topicOf, jintArray topicBounds, jbyteArray fixed,
    jintArray replicasOut, jlongArray statsOut)
{
    (void)cls;
    jbyte *rk = (*env)->GetByteArrayElements(env, rackOf, NULL);
    jshort *f = (*env)->GetShortArrayElements(env, wF, NULL);
    jshort *l = (*env)->GetShortArrayElements(env, wL, NULL);
    jint *bd = (*env)->GetIntArrayElements(env, bounds, NULL);
    jint *cu = (*env)->GetIntArrayElements(env, cur, NULL);
    jint *to = topicOf ? (*env)->GetIntArrayElements(env, topicOf, NULL) : NULL;
    jint *tb = topicOf ? (*env)->GetIntArrayElements(env, topicBounds, NULL) : NULL;
    jbyte *fx = fixed ? (*env)->GetByteArrayElements(env, fixed, NULL) : NULL;
    jint *out = (*env)->GetIntArrayElements(env, replicasOut, NULL);

    kao_problem pb;
    pb.P = P; pb.B = B; pb.R = R; pb.RF = RF; pb.RFcur = RFcur;
    pb.rack_of = (const uint8_t *)rk;
    pb.wF = (const uint16_t *)f;
    pb.wL = (const uint16_t *)l;
    pb.rep_lo = (const int32_t *)bd;          pb.rep_hi = (const int32_t *)bd + B;
    pb.ldr_lo = (const int32_t *)bd + 2 * B;  pb.ldr_hi = (const int32_t *)bd + 3 * B;
    pb.rack_lo = (const int32_t *)bd + 4 * B; pb.rack_hi = (const int32_t *)bd + 4 * B + R;
    pb.ppr_lo = bd[4 * B + 2 * R];            pb.ppr_hi = bd[4 * B + 2 * R + 1];
    pb.cur = (const int32_t *)cu;
    int32_t T = 0;
    for (jint p = 0; to && p < P; ++p) T = to[p] + 1 > T ? to[p] + 1 : T;
    kao_topics tp = {T, (const int32_t *)to, (const int32_t *)tb, (const int32_t *)tb + T, (const int32_t *)tb + 2 * T,
                     (const int32_t *)tb + 3 * T};
    kao_result res;
    res.replicas = (int32_t *)out;
    int64_t fixed_violation = 0;
    const int rc = kao_solve_leaders(&pb, to ? &tp : NULL, (const uint8_t *)fx, &res, &fixed_violation);

    (*env)->ReleaseByteArrayElements(env, rackOf, rk, JNI_ABORT);
    (*env)->ReleaseShortArrayElements(env, wF, f, JNI_ABORT);
    (*env)->ReleaseShortArrayElements(env, wL, l, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, bounds, bd, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, cur, cu, JNI_ABORT);
    if (to) (*env)->ReleaseIntArrayElements(env, topicOf, to, JNI_ABORT);
    if (tb) (*env)->ReleaseIntArrayElements(env, topicBounds, tb, JNI_ABORT);
    if (fx) (*env)->ReleaseByteArrayElements(env, fixed, fx, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, replicasOut, out, rc < 0 ? JNI_ABORT : 0);
    if (rc < 0) {
        kao_jni_throw(env, rc);
        return rc;
    }
    jlong st[3] = {res.objective, res.violation, fixed_violation};
    (*env)->SetLongArrayRegion(env, statsOut, 0, 3, st);
    return rc;
}
