/* Minimal STAND-IN for the JDK's jni.h, used only by tests/test_abi_surface.py to type-check
 * distributed_sgd_b200/jni/dsgd_jni.c on a box without a JDK, and by tests/test_gpu_jni.py to run it through the stand-in
 * JNIEnv of jni_env.c.  It declares just the JNI names that shim uses, with
 * the JDK's types on LP64 Linux; the layout of the function table is NOT the real one -- never load a library built
 * against this header into a JVM. */
#ifndef DSGD_JNI_MOCK_H
#define DSGD_JNI_MOCK_H
#include <stdint.h>
typedef int32_t jint;
typedef int64_t jlong;
typedef int8_t jbyte;
typedef float jfloat;
typedef double jdouble;
typedef jint jsize;
typedef struct _jobject *jobject;
typedef jobject jstring, jarray, jintArray, jlongArray, jfloatArray, jdoubleArray, jbyteArray;
#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL
struct JNINativeInterface_;
typedef const struct JNINativeInterface_ *JNIEnv;
#define DSGD_MOCK_REGION(Name, JT)                                                                   \
  void (*Get##Name##ArrayRegion)(JNIEnv *env, JT##Array array, jsize start, jsize len, JT *buf);     \
  void (*Set##Name##ArrayRegion)(JNIEnv *env, JT##Array array, jsize start, jsize len, const JT *buf);
struct JNINativeInterface_ {
  jstring (*NewStringUTF)(JNIEnv *env, const char *utf);
  jsize (*GetArrayLength)(JNIEnv *env, jarray array);
  DSGD_MOCK_REGION(Int, jint)
  DSGD_MOCK_REGION(Long, jlong)
  DSGD_MOCK_REGION(Float, jfloat)
  DSGD_MOCK_REGION(Double, jdouble)
  DSGD_MOCK_REGION(Byte, jbyte)
};
#endif
