/*
 * A stand-in JNIEnv for running jni/b200shuffle_jni.c without a JVM (tests/jni_shim.py drives it).
 *
 * Compiled against jni/stub/jni.h only, so its function table has the shim's layout; it is a test fixture and is never
 * linked against a JVM.  It behaves like a JVM running with -Xcheck:jni: every misuse of the interface is recorded as
 * a violation, and the test that made the call fails.
 *
 *   arrays           typed long[] / int[] / byte[] objects with a length; the storage has canary guard zones on both
 *                    sides.  NULL is a valid handle.
 *   critical regions mode direct: GetPrimitiveArrayCritical returns a pointer into the array's storage (as HotSpot
 *                    does); mode copy: a fresh guarded copy, copied back by a Release with mode 0 and discarded by
 *                    JNI_ABORT.
 *   violations       a region call out of bounds or of the wrong element type; GetArrayLength, a region call or
 *                    NewStringUTF given NULL; any call but a critical Get / Release while a critical region is open;
 *                    a Release of a pointer no Get returned (or released twice); a Get still open when the native
 *                    returns; a changed guard zone; a changed input array; NewStringUTF given invalid modified UTF-8;
 *                    GetDirectBufferAddress / Capacity of an object that is not a direct buffer.
 *
 * One env per thread, as a JVM gives: an env owns the objects made through it and keeps its own violation log, so
 * natives can run on several threads at once.
 */
#include <jni.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define GUARD 64
#define CANARY 0xA5

enum { K_LONG = 'J', K_INT = 'I', K_BYTE = 'B', K_DIRECT = 'D', K_STRING = 'S' };

struct _jobject {
  int kind;
  jsize length;    /* elements of an array, bytes of a string */
  size_t elem;     /* bytes per element */
  uint8_t* block;  /* GUARD | storage | GUARD */
  uint8_t* input;  /* a snapshot of an input array's elements (NULL for an output) */
  void* address;   /* direct buffer */
  jlong capacity;  /* direct buffer */
  struct _jobject* next;
};

typedef struct region {
  struct _jobject* obj;
  void* ptr;
  uint8_t* copy; /* copy mode: the guarded block ptr lies in */
  struct region* next;
} region;

typedef struct host_env {
  const struct JNINativeInterface_* functions; /* JNIEnv* points here */
  int copy_mode;
  struct _jobject* objects;
  region* open;
  char* log;
  size_t log_len, log_cap;
} host_env;

static host_env* H(JNIEnv* e) { return (host_env*)e; }

static void violation(JNIEnv* e, const char* fmt, ...) {
  host_env* h = H(e);
  char line[256];
  va_list ap;
  va_start(ap, fmt);
  int k = vsnprintf(line, sizeof line - 1, fmt, ap);
  va_end(ap);
  if (k < 0) return;
  if (k > (int)sizeof line - 2) k = (int)sizeof line - 2;
  line[k++] = '\n';
  line[k] = 0;
  if (h->log_len + (size_t)k + 1 > h->log_cap) {
    size_t cap = (h->log_cap + (size_t)k + 1) * 2;
    char* p = realloc(h->log, cap);
    if (!p) return;
    h->log = p;
    h->log_cap = cap;
  }
  memcpy(h->log + h->log_len, line, (size_t)k + 1);
  h->log_len += (size_t)k;
}

static int is_array(const struct _jobject* o) { return o->kind == K_LONG || o->kind == K_INT || o->kind == K_BYTE; }

/* every call but a critical Get / Release checks that no critical region is open */
static void not_critical(JNIEnv* e, const char* call) {
  if (H(e)->open) violation(e, "%s called inside a critical region", call);
}

static uint8_t* new_block(size_t bytes) {
  uint8_t* b = malloc(bytes + 2 * GUARD);
  if (b) {
    memset(b, CANARY, GUARD);
    memset(b + GUARD + bytes, CANARY, GUARD);
  }
  return b;
}

static int guards_intact(const uint8_t* b, size_t bytes) {
  for (size_t i = 0; i < GUARD; i++)
    if (b[i] != CANARY || b[GUARD + bytes + i] != CANARY) return 0;
  return 1;
}

static size_t bytes_of(const struct _jobject* o) { return (size_t)o->length * o->elem; }

/* ---- the JNIEnv members the stub declares ---- */
static jobject NewDirectByteBuffer(JNIEnv* e, void* address, jlong capacity) {
  not_critical(e, "NewDirectByteBuffer");
  struct _jobject* o = calloc(1, sizeof *o);
  if (!o) return 0;
  o->kind = K_DIRECT;
  o->address = address;
  o->capacity = capacity;
  o->next = H(e)->objects;
  H(e)->objects = o;
  return o;
}

static void* GetDirectBufferAddress(JNIEnv* e, jobject buf) {
  not_critical(e, "GetDirectBufferAddress");
  if (!buf || buf->kind != K_DIRECT) {
    violation(e, "GetDirectBufferAddress of an object that is not a direct buffer");
    return 0;
  }
  return buf->address;
}

static jlong GetDirectBufferCapacity(JNIEnv* e, jobject buf) {
  not_critical(e, "GetDirectBufferCapacity");
  if (!buf || buf->kind != K_DIRECT) {
    violation(e, "GetDirectBufferCapacity of an object that is not a direct buffer");
    return -1;
  }
  return buf->capacity;
}

static void* GetPrimitiveArrayCritical(JNIEnv* e, jarray a, jboolean* isCopy) {
  if (!a || !is_array(a)) {
    violation(e, "GetPrimitiveArrayCritical of %s", a ? "an object that is not an array" : "NULL");
    return 0;
  }
  region* r = calloc(1, sizeof *r);
  if (!r) return 0;
  r->obj = a;
  const size_t n = bytes_of(a);
  if (H(e)->copy_mode) {
    r->copy = new_block(n);
    if (!r->copy) {
      free(r);
      return 0;
    }
    memcpy(r->copy + GUARD, a->block + GUARD, n);
    r->ptr = r->copy + GUARD;
  } else {
    r->ptr = a->block + GUARD;
  }
  r->next = H(e)->open;
  H(e)->open = r;
  if (isCopy) *isCopy = (jboolean)(r->copy != 0);
  return r->ptr;
}

static void ReleasePrimitiveArrayCritical(JNIEnv* e, jarray a, void* carray, jint mode) {
  region** p = &H(e)->open;
  while (*p && ((*p)->ptr != carray || (*p)->obj != a)) p = &(*p)->next;
  if (!*p) {
    violation(e, "ReleasePrimitiveArrayCritical of a pointer no open Get returned");
    return;
  }
  region* r = *p;
  *p = r->next;
  if (r->copy) {
    const size_t n = bytes_of(a);
    if (!guards_intact(r->copy, n)) violation(e, "a guard zone of a critical copy was overwritten");
    if (mode != JNI_ABORT) memcpy(a->block + GUARD, r->copy + GUARD, n);
    free(r->copy);
  }
  free(r);
}

static jsize GetArrayLength(JNIEnv* e, jarray a) {
  not_critical(e, "GetArrayLength");
  if (!a || !is_array(a)) {
    violation(e, "GetArrayLength of %s", a ? "an object that is not an array" : "NULL");
    return 0;
  }
  return a->length;
}

/* the region calls: element type, bounds, NULL */
static uint8_t* region_at(JNIEnv* e, const char* call, jarray a, int kind, jsize start, jsize len, const void* buf) {
  not_critical(e, call);
  if (!a) {
    violation(e, "%s of NULL", call);
    return 0;
  }
  if (a->kind != kind) {
    violation(e, "%s of an array of the wrong element type", call);
    return 0;
  }
  if (start < 0 || len < 0 || (int64_t)start + len > a->length) {
    violation(e, "%s [%d, %d + %d) out of bounds of an array of %d", call, start, start, len, a->length);
    return 0;
  }
  if (len > 0 && !buf) {
    violation(e, "%s with a NULL buffer", call);
    return 0;
  }
  return a->block + GUARD + (size_t)start * a->elem;
}

static void SetLongArrayRegion(JNIEnv* e, jlongArray a, jsize start, jsize len, const jlong* buf) {
  uint8_t* p = region_at(e, "SetLongArrayRegion", a, K_LONG, start, len, buf);
  if (p && len) memcpy(p, buf, (size_t)len * sizeof(jlong));
}
static void SetIntArrayRegion(JNIEnv* e, jintArray a, jsize start, jsize len, const jint* buf) {
  uint8_t* p = region_at(e, "SetIntArrayRegion", a, K_INT, start, len, buf);
  if (p && len) memcpy(p, buf, (size_t)len * sizeof(jint));
}
static void GetLongArrayRegion(JNIEnv* e, jlongArray a, jsize start, jsize len, jlong* buf) {
  uint8_t* p = region_at(e, "GetLongArrayRegion", a, K_LONG, start, len, buf);
  if (p && len) memcpy(buf, p, (size_t)len * sizeof(jlong));
}
static void GetIntArrayRegion(JNIEnv* e, jintArray a, jsize start, jsize len, jint* buf) {
  uint8_t* p = region_at(e, "GetIntArrayRegion", a, K_INT, start, len, buf);
  if (p && len) memcpy(buf, p, (size_t)len * sizeof(jint));
}
static void GetByteArrayRegion(JNIEnv* e, jbyteArray a, jsize start, jsize len, jbyte* buf) {
  uint8_t* p = region_at(e, "GetByteArrayRegion", a, K_BYTE, start, len, buf);
  if (p && len) memcpy(buf, p, (size_t)len);
}

/* modified UTF-8: no NUL byte, no four-byte form (supplementary characters are surrogate pairs), NUL as C0 80 */
static int modified_utf8(const uint8_t* s) {
  while (*s) {
    const uint8_t c = *s;
    int more;
    if (c < 0x80) more = 0;
    else if ((c & 0xE0) == 0xC0) more = 1;
    else if ((c & 0xF0) == 0xE0) more = 2;
    else return 0;
    for (int i = 1; i <= more; i++)
      if ((s[i] & 0xC0) != 0x80) return 0;
    if (more == 1 && c < 0xC2 && !(c == 0xC0 && s[1] == 0x80)) return 0; /* overlong, C0 80 aside */
    if (more == 2 && c == 0xE0 && s[1] < 0xA0) return 0;                   /* overlong */
    s += 1 + more;
  }
  return 1;
}

static jstring NewStringUTF(JNIEnv* e, const char* utf) {
  not_critical(e, "NewStringUTF");
  if (!utf) {
    violation(e, "NewStringUTF of NULL");
    return 0;
  }
  if (!modified_utf8((const uint8_t*)utf)) {
    violation(e, "NewStringUTF of invalid modified UTF-8");
    return 0;
  }
  struct _jobject* o = calloc(1, sizeof *o);
  const size_t n = strlen(utf);
  if (!o || !(o->block = new_block(n + 1))) {
    free(o);
    return 0;
  }
  o->kind = K_STRING;
  o->length = (jsize)n;
  o->elem = 1;
  memcpy(o->block + GUARD, utf, n + 1);
  o->next = H(e)->objects;
  H(e)->objects = o;
  return o;
}

static const struct JNINativeInterface_ kTable = {
    NewDirectByteBuffer, GetDirectBufferAddress, GetDirectBufferCapacity, GetPrimitiveArrayCritical,
    ReleasePrimitiveArrayCritical, GetArrayLength, NewStringUTF, SetLongArrayRegion, SetIntArrayRegion,
    GetLongArrayRegion, GetIntArrayRegion, GetByteArrayRegion,
};

/* ---- the driver's side ---- */
host_env* jenv_new(int copy_mode) {
  host_env* h = calloc(1, sizeof *h);
  if (h) {
    h->functions = &kTable;
    h->copy_mode = copy_mode;
  }
  return h;
}

/* a new array of kind 'J' / 'I' / 'B' holding length elements from data (zeros when data is NULL); input: its
 * elements must not change */
jobject jenv_array(host_env* h, int kind, jsize length, const void* data, int input) {
  struct _jobject* o = calloc(1, sizeof *o);
  if (!o) return 0;
  o->kind = kind;
  o->length = length;
  o->elem = kind == K_LONG ? 8 : kind == K_INT ? 4 : 1;
  const size_t n = bytes_of(o);
  o->block = new_block(n);
  if (!o->block || (input && !(o->input = malloc(n + 1)))) {
    free(o->block);
    free(o);
    return 0;
  }
  if (data) memcpy(o->block + GUARD, data, n);
  else memset(o->block + GUARD, 0, n);
  if (input) memcpy(o->input, o->block + GUARD, n);
  o->next = h->objects;
  h->objects = o;
  return o;
}

jobject jenv_direct_buffer(host_env* h, void* address, jlong capacity) {
  return NewDirectByteBuffer((JNIEnv*)h, address, capacity);
}

/* the elements of an array (bytes of a string, NUL-terminated), and their count */
const void* jenv_data(jobject o) { return o ? o->block + GUARD : 0; }
jsize jenv_length(jobject o) { return o ? o->length : -1; }
void* jenv_buffer_address(jobject o) { return o && o->kind == K_DIRECT ? o->address : 0; }
jlong jenv_buffer_capacity(jobject o) { return o && o->kind == K_DIRECT ? o->capacity : -1; }

/* after a native returned: no region left open, every guard intact, no input changed.  -> the violations logged since
 * the last call (empty when none); the log is cleared */
const char* jenv_check(host_env* h) {
  JNIEnv* e = (JNIEnv*)h;
  for (region* r = h->open; r; r = h->open) {
    violation(e, "a critical region still open when the native returned");
    h->open = r->next;
    free(r->copy);
    free(r);
  }
  for (struct _jobject* o = h->objects; o; o = o->next) {
    if (!o->block) continue;
    const size_t n = o->kind == K_STRING ? (size_t)o->length + 1 : bytes_of(o);
    if (!guards_intact(o->block, n)) violation(e, "a guard zone of a %c array of %d was overwritten", o->kind, o->length);
    if (o->input && memcmp(o->input, o->block + GUARD, n))
      violation(e, "input %c array of %d was changed", o->kind, o->length);
  }
  static _Thread_local char out[8192];
  const size_t k = h->log_len < sizeof out - 1 ? h->log_len : sizeof out - 1;
  if (k) memcpy(out, h->log, k);
  out[k] = 0;
  h->log_len = 0;
  return out;
}

/* frees every object made through the env */
void jenv_free_objects(host_env* h) {
  while (h->objects) {
    struct _jobject* o = h->objects;
    h->objects = o->next;
    free(o->block);
    free(o->input);
    free(o);
  }
}

void jenv_free(host_env* h) {
  if (!h) return;
  jenv_check(h);
  jenv_free_objects(h);
  free(h->log);
  free(h);
}
