/*
 * Minimal jni.h SUBSET for compile-checking jni/b200shuffle_jni.c where no JDK exists (this image and the GPU box have
 * neither a JVM nor jni.h).  Test infrastructure only: a real build uses $JAVA_HOME/include/jni.h, whose declarations
 * these mirror (types, JNIEXPORT/JNICALL, and the JNIEnv function-table members the shim calls).  The function table
 * of a real JVM has ~230 slots in a fixed order; this struct only lists the members used and MUST NOT be linked
 * against a JVM.
 */
#ifndef B2S_STUB_JNI_H
#define B2S_STUB_JNI_H
#include <stdint.h>

#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL
#define JNI_ABORT 2

typedef int32_t jint;
typedef int64_t jlong;
typedef int8_t jbyte;
typedef uint8_t jboolean;
typedef jint jsize;
typedef struct _jobject* jobject;
typedef jobject jclass;
typedef jobject jstring;
typedef jobject jarray;
typedef jarray jlongArray;
typedef jarray jintArray;

struct JNINativeInterface_;
typedef const struct JNINativeInterface_* JNIEnv;

struct JNINativeInterface_ {
  jobject (*NewDirectByteBuffer)(JNIEnv* env, void* address, jlong capacity);
  void* (*GetDirectBufferAddress)(JNIEnv* env, jobject buf);
  jlong (*GetDirectBufferCapacity)(JNIEnv* env, jobject buf);
  void* (*GetPrimitiveArrayCritical)(JNIEnv* env, jarray array, jboolean* isCopy);
  void (*ReleasePrimitiveArrayCritical)(JNIEnv* env, jarray array, void* carray, jint mode);
  jsize (*GetArrayLength)(JNIEnv* env, jarray array);
  jstring (*NewStringUTF)(JNIEnv* env, const char* utf);
  void (*SetLongArrayRegion)(JNIEnv* env, jlongArray array, jsize start, jsize len, const jlong* buf);
  void (*SetIntArrayRegion)(JNIEnv* env, jintArray array, jsize start, jsize len, const jint* buf);
  void (*GetLongArrayRegion)(JNIEnv* env, jlongArray array, jsize start, jsize len, jlong* buf);
  void (*GetIntArrayRegion)(JNIEnv* env, jintArray array, jsize start, jsize len, jint* buf);
};
#endif
