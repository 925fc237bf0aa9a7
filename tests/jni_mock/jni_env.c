/* A stand-in JNIEnv over the stand-in jni.h, for tests/test_gpu_jni.py: it runs distributed_sgd_b200/jni/dsgd_jni.c
 * without a JVM.  A Java array is a (element type, length, data) record over memory the test owns; a Get / Set region
 * call of another element type, or outside the array, copies nothing and counts an error the test reads. */
#include <string.h>
#include "jni.h"

enum { J_INT, J_LONG, J_FLOAT, J_DOUBLE, J_BYTE };
struct _jobject { int32_t type; jsize n; void *data; };

static int region_errors;

static int region_ok(jarray a, int type, jsize start, jsize len) {
  if (a && a->type == type && start >= 0 && len >= 0 && start <= a->n - len) return 1;
  ++region_errors;
  return 0;
}
#define MOCK_REGION(Name, JT, T)                                                                         \
  static void get_##Name(JNIEnv *env, JT##Array a, jsize start, jsize len, JT *buf) {                    \
    if (region_ok(a, T, start, len)) memcpy(buf, (JT *)a->data + start, sizeof(JT) * (size_t)len);        \
  }                                                                                                      \
  static void set_##Name(JNIEnv *env, JT##Array a, jsize start, jsize len, const JT *buf) {              \
    if (region_ok(a, T, start, len)) memcpy((JT *)a->data + start, buf, sizeof(JT) * (size_t)len);        \
  }
MOCK_REGION(Int, jint, J_INT)
MOCK_REGION(Long, jlong, J_LONG)
MOCK_REGION(Float, jfloat, J_FLOAT)
MOCK_REGION(Double, jdouble, J_DOUBLE)
MOCK_REGION(Byte, jbyte, J_BYTE)

static jstring new_string(JNIEnv *env, const char *utf) { return NULL; }
static jsize array_length(JNIEnv *env, jarray a) { return a->n; }

static const struct JNINativeInterface_ table = {
    .NewStringUTF = new_string,          .GetArrayLength = array_length,
    .GetIntArrayRegion = get_Int,        .SetIntArrayRegion = set_Int,
    .GetLongArrayRegion = get_Long,      .SetLongArrayRegion = set_Long,
    .GetFloatArrayRegion = get_Float,    .SetFloatArrayRegion = set_Float,
    .GetDoubleArrayRegion = get_Double,  .SetDoubleArrayRegion = set_Double,
    .GetByteArrayRegion = get_Byte,      .SetByteArrayRegion = set_Byte,
};
static JNIEnv env = &table;

JNIEnv *mock_env(void) { return &env; }
int mock_region_errors(void) { return region_errors; }
