// jni/rainier_jni.cpp -- the thin JNI shim between Rainier's Scala host code and the C ABI of librainier_cuda.so
// (include/rainier_cuda.h).  Binds the static native methods of scala/com/stripe/rainier/cuda/Native.java.
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no JDK (no <jni.h>, no javac/scalac).  It is written
// against the JNI specification and guarded by __has_include so that `make -C jni` is a no-op where <jni.h> is
// missing.  Build where a JDK exists:
//   g++ -O2 -std=c++17 -fPIC -shared -I$JAVA_HOME/include -I$JAVA_HOME/include/linux jni/rainier_jni.cpp \
//       -Lrainier_b200 -lrainier_cuda -Wl,-rpath,'$ORIGIN' -o librainier_jni.so
//
// Every function is a 1:1 forward.  The natives are the STATIC methods of the Java class
// scala/com/stripe/rainier/cuda/Native.java (hence the `jclass` receiver and the unmangled `..._Native_<method>` names).
// Java arrays cross by REGION COPIES (Get/Set<Type>ArrayRegion) around the native call: rn_sample / rn_density_batch /
// rn_function_eval / rn_optimize can run for seconds to minutes (NVRTC compile, warmup, a blocking stream sync, worker
// threads), and JNI forbids blocking inside a Get/ReleasePrimitiveArrayCritical region (it would also stall the GC of
// every JVM thread).  The bulk path (`sampleDirect`) takes a direct, page-locked ByteBuffer and copies nothing.
// The RIR container and the rn_config POD travel as direct ByteBuffers filled by the Scala side
// (scala/com/stripe/rainier/cuda/RIR.scala, CudaConfig.scala).  A non-zero return code becomes a RuntimeException
// carrying rn_last_error() -- mirroring the reference, where failures on this path are exceptions thrown from
// generated code (ir/MethodGenerator.scala:164-167).
#if defined(__has_include)
#if __has_include(<jni.h>)
#define RN_HAVE_JNI 1
#endif
#endif

#ifdef RN_HAVE_JNI
#include <jni.h>

#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "../include/rainier_cuda.h"

namespace {
void throw_last(JNIEnv* env) {
  jclass c = env->FindClass("java/lang/RuntimeException");
  if (c) env->ThrowNew(c, rn_last_error());
}
// region copies: Java array -> native vector before the call, native vector -> Java array after it
std::vector<double> in_doubles(JNIEnv* env, jdoubleArray a) {
  std::vector<double> v(a ? (size_t)env->GetArrayLength(a) : 0);
  if (!v.empty()) env->GetDoubleArrayRegion(a, 0, (jsize)v.size(), v.data());
  return v;
}
std::vector<int64_t> in_longs(JNIEnv* env, jlongArray a) {
  static_assert(sizeof(jlong) == sizeof(int64_t), "jlong is 64 bits");
  std::vector<int64_t> v(a ? (size_t)env->GetArrayLength(a) : 0);
  if (!v.empty()) env->GetLongArrayRegion(a, 0, (jsize)v.size(), (jlong*)v.data());
  return v;
}
void out_doubles(JNIEnv* env, jdoubleArray a, const double* src, size_t n) {
  if (a && n) env->SetDoubleArrayRegion(a, 0, (jsize)n, src);
}
}  // namespace

extern "C" {

// def create(rir: ByteBuffer, cols: Array[Array[Double]], device: Int): Long
JNIEXPORT jlong JNICALL Java_com_stripe_rainier_cuda_Native_create(JNIEnv* env, jclass, jobject rir, jobjectArray cols,
                                                                  jint device) {
  const void* rp = env->GetDirectBufferAddress(rir);
  const jlong rlen = env->GetDirectBufferCapacity(rir);
  const jsize n = cols ? env->GetArrayLength(cols) : 0;
  // columns are copied to the device inside rn_model_create, so pin them one at a time via Get<>ArrayElements
  std::vector<jdoubleArray> arrs(n);
  std::vector<jdouble*> ptrs(n);
  std::vector<int64_t> rows(n);
  for (jsize i = 0; i < n; i++) {
    arrs[i] = (jdoubleArray)env->GetObjectArrayElement(cols, i);
    rows[i] = env->GetArrayLength(arrs[i]);
    ptrs[i] = env->GetDoubleArrayElements(arrs[i], nullptr);
  }
  rn_model* m = nullptr;
  const int rc = rn_model_create(rp, (size_t)rlen, (const double* const*)ptrs.data(), rows.data(), (int)n, device, &m);
  for (jsize i = 0; i < n; i++) env->ReleaseDoubleArrayElements(arrs[i], ptrs[i], JNI_ABORT);
  if (rc != RN_OK) {
    throw_last(env);
    return 0;
  }
  return (jlong)(intptr_t)m;
}

JNIEXPORT jint JNICALL Java_com_stripe_rainier_cuda_Native_nvars(JNIEnv*, jclass, jlong h) {
  return rn_model_nvars((const rn_model*)(intptr_t)h);
}

// def densityBatch(h: Long, q: Array[Double], chains: Int, out: Array[Double]): Unit
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_densityBatch(JNIEnv* env, jclass, jlong h, jdoubleArray q,
                                                                       jint chains, jdoubleArray out) {
  const std::vector<double> vq = in_doubles(env, q);
  std::vector<double> vo((size_t)env->GetArrayLength(out));
  const int rc = rn_density_batch((rn_model*)(intptr_t)h, vq.data(), chains, vo.data());
  if (rc != RN_OK) return throw_last(env);
  out_doubles(env, out, vo.data(), vo.size());
}

// def sample(h: Long, config: ByteBuffer, seeds: Array[Long], samples: Array[Double], mass: Array[Double],
//            stats: ByteBuffer): Unit          (config = rn_config bytes, stats = chains * sizeof(rn_chain_stats))
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_sample(JNIEnv* env, jclass, jlong h, jobject config,
                                                                 jlongArray seeds, jdoubleArray samples, jdoubleArray mass,
                                                                 jobject stats) {
  const rn_config* cfg = (const rn_config*)env->GetDirectBufferAddress(config);
  rn_chain_stats* st = stats ? (rn_chain_stats*)env->GetDirectBufferAddress(stats) : nullptr;
  const std::vector<int64_t> vs = in_longs(env, seeds);
  const size_t ns = samples ? (size_t)env->GetArrayLength(samples) : 0, nm = mass ? (size_t)env->GetArrayLength(mass) : 0;
  std::unique_ptr<double[]> vo(ns ? new double[ns] : nullptr);  // uninitialised: rn_sample writes every element
  std::vector<double> vm(nm);
  const int rc = rn_sample((rn_model*)(intptr_t)h, cfg, vs.data(), (int)vs.size(), vo.get(), nm ? vm.data() : nullptr, st);
  if (rc != RN_OK) return throw_last(env);
  out_doubles(env, samples, vo.get(), ns);
  out_doubles(env, mass, vm.data(), nm);
}

// def hostAlloc(device: Int, bytes: Long): ByteBuffer   -- page-locked memory as a direct buffer (rn_host_alloc)
JNIEXPORT jobject JNICALL Java_com_stripe_rainier_cuda_Native_hostAlloc(JNIEnv* env, jclass, jint device, jlong bytes) {
  void* p = nullptr;
  if (rn_host_alloc(device, (size_t)bytes, &p) != RN_OK) {
    throw_last(env);
    return nullptr;
  }
  return env->NewDirectByteBuffer(p, bytes);
}
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_hostFree(JNIEnv* env, jclass, jint device, jobject buf) {
  if (rn_host_free(device, env->GetDirectBufferAddress(buf)) != RN_OK) throw_last(env);
}

// def sampleDirect(h: Long, config: ByteBuffer, seeds: Array[Long], samples: ByteBuffer, mass: Array[Double],
//                  stats: ByteBuffer): Unit    -- samples is a direct buffer (ideally from hostAlloc: the device->host
// copy of chains*iterations*n doubles then is one DMA into the buffer the JVM reads, with no staging copy)
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_sampleDirect(JNIEnv* env, jclass, jlong h, jobject config,
                                                                       jlongArray seeds, jobject samples, jdoubleArray mass,
                                                                       jobject stats) {
  const rn_config* cfg = (const rn_config*)env->GetDirectBufferAddress(config);
  rn_chain_stats* st = stats ? (rn_chain_stats*)env->GetDirectBufferAddress(stats) : nullptr;
  double* out = (double*)env->GetDirectBufferAddress(samples);
  const std::vector<int64_t> vs = in_longs(env, seeds);
  std::vector<double> vm(mass ? (size_t)env->GetArrayLength(mass) : 0);
  const int rc = rn_sample((rn_model*)(intptr_t)h, cfg, vs.data(), (int)vs.size(), out, vm.empty() ? nullptr : vm.data(), st);
  if (rc != RN_OK) return throw_last(env);
  out_doubles(env, mass, vm.data(), vm.size());
}

JNIEXPORT jstring JNICALL Java_com_stripe_rainier_cuda_Native_emitSource(JNIEnv* env, jclass, jlong h, jobject config) {
  const rn_config* cfg = config ? (const rn_config*)env->GetDirectBufferAddress(config) : nullptr;
  size_t need = 0;
  if (rn_emit_source((rn_model*)(intptr_t)h, cfg, nullptr, 0, &need) != RN_OK) {
    throw_last(env);
    return nullptr;
  }
  std::vector<char> buf(need);
  rn_emit_source((rn_model*)(intptr_t)h, cfg, buf.data(), buf.size(), &need);
  return env->NewStringUTF(buf.data());
}

JNIEXPORT jint JNICALL Java_com_stripe_rainier_cuda_Native_configSize(JNIEnv*, jclass) { return (jint)sizeof(rn_config); }
JNIEXPORT jint JNICALL Java_com_stripe_rainier_cuda_Native_statsSize(JNIEnv*, jclass) { return (jint)sizeof(rn_chain_stats); }
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_defaultConfig(JNIEnv* env, jclass, jobject config) {
  rn_config_default((rn_config*)env->GetDirectBufferAddress(config));
}
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_destroy(JNIEnv*, jclass, jlong h) {
  rn_model_destroy((rn_model*)(intptr_t)h);
}
// ---- compiled functions: Generator.prepare's Compiler.compile + CompiledFunction.output loop (core/Generator.scala:59-94) ----
// def functionCreate(rir: ByteBuffer, device: Int): Long
JNIEXPORT jlong JNICALL Java_com_stripe_rainier_cuda_Native_functionCreate(JNIEnv* env, jclass, jobject rir, jint device) {
  rn_function* f = nullptr;
  if (rn_function_create(env->GetDirectBufferAddress(rir), (size_t)env->GetDirectBufferCapacity(rir), device, RN_MATH_PARITY, &f) != RN_OK) {
    throw_last(env);
    return 0;
  }
  return (jlong)(intptr_t)f;
}
// def functionEval(handle: Long, draws: Array[Double], count: Long, out: Array[Double]): Unit   draws [count][n] -> out [count][m]
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_functionEval(JNIEnv* env, jclass, jlong h, jdoubleArray draws, jlong count,
                                                                        jdoubleArray out) {
  const std::vector<double> vx = in_doubles(env, draws);
  std::vector<double> vo((size_t)env->GetArrayLength(out));
  const int rc = rn_function_eval((rn_function*)(intptr_t)h, vx.data(), (int64_t)count, vo.data());
  if (rc != RN_OK) return throw_last(env);
  out_doubles(env, out, vo.data(), vo.size());
}
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_functionDestroy(JNIEnv*, jclass, jlong h) {
  rn_function_destroy((rn_function*)(intptr_t)h);
}
// ---- posterior-predictive draws: Trace.predict's Generator.get on the device (core/Trace.scala:34-41) ----
// rng states cross as long[3 * chains] = (seed48, doubleToRawLongBits(nextNextGaussian), haveNextNextGaussian) per chain
static void rng_in(JNIEnv* env, jlongArray a, std::vector<rn_rng_state>& st) {
  const jsize k = env->GetArrayLength(a) / 3;
  std::vector<jlong> v((size_t)k * 3);
  env->GetLongArrayRegion(a, 0, k * 3, v.data());
  st.assign((size_t)k, rn_rng_state{});
  for (jsize c = 0; c < k; c++) {
    st[c].seed48 = v[3 * c];
    std::memcpy(&st[c].next_gaussian, &v[3 * c + 1], 8);
    st[c].have_next = (int32_t)v[3 * c + 2];
  }
}
static void rng_out(JNIEnv* env, jlongArray a, const std::vector<rn_rng_state>& st) {
  std::vector<jlong> v(st.size() * 3);
  for (size_t c = 0; c < st.size(); c++) {
    v[3 * c] = st[c].seed48;
    std::memcpy(&v[3 * c + 1], &st[c].next_gaussian, 8);
    v[3 * c + 2] = st[c].have_next;
  }
  env->SetLongArrayRegion(a, 0, (jsize)v.size(), v.data());
}
// def generatorCreate(rir: ByteBuffer, device: Int): Long    (a RIR_FLAG_GENERATOR container)
JNIEXPORT jlong JNICALL Java_com_stripe_rainier_cuda_Native_generatorCreate(JNIEnv* env, jclass, jobject rir, jint device) {
  rn_generator* g = nullptr;
  if (rn_generator_create(env->GetDirectBufferAddress(rir), (size_t)env->GetDirectBufferCapacity(rir), device, &g) != RN_OK) {
    throw_last(env);
    return 0;
  }
  return (jlong)(intptr_t)g;
}
JNIEXPORT jint JNICALL Java_com_stripe_rainier_cuda_Native_generatorOutputs(JNIEnv*, jclass, jlong h) {
  return rn_generator_noutputs((rn_generator*)(intptr_t)h);
}
// def generatorEval(handle: Long, draws: Array[Double] /* [chains][iterations][n] */, iterations: Long, chains: Long,
//                   rng: Array[Long] /* in/out */, out: Array[Double] /* [chains][iterations][m_out] */): Unit
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_generatorEval(JNIEnv* env, jclass, jlong h, jdoubleArray draws, jlong iterations,
                                                                         jlong chains, jlongArray rng, jdoubleArray out) {
  const std::vector<double> vx = in_doubles(env, draws);
  std::vector<double> vo((size_t)env->GetArrayLength(out));
  std::vector<rn_rng_state> st;
  rng_in(env, rng, st);
  const int rc = rn_generator_eval((rn_generator*)(intptr_t)h, vx.data(), (int64_t)iterations, (int64_t)chains, st.data(), vo.data());
  if (rc != RN_OK) return throw_last(env);
  rng_out(env, rng, st);
  out_doubles(env, out, vo.data(), vo.size());
}
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_generatorDestroy(JNIEnv*, jclass, jlong h) {
  rn_generator_destroy((rn_generator*)(intptr_t)h);
}
// def sampleGenerate(model: Long, config: ByteBuffer, generator: Long, seeds: Array[Long], out: Array[Double], rngOut: Array[Long]): Unit
//   model.sample(config).predict(gen) with the draws on the device; rngOut: the states after the predictive draws
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_sampleGenerate(JNIEnv* env, jclass, jlong m, jobject config, jlong g,
                                                                          jlongArray seeds, jdoubleArray out, jlongArray rngOut) {
  const jsize chains = env->GetArrayLength(seeds);
  std::vector<jlong> vs((size_t)chains);
  env->GetLongArrayRegion(seeds, 0, chains, vs.data());
  std::vector<int64_t> s64(vs.begin(), vs.end());
  std::vector<double> vo((size_t)env->GetArrayLength(out));
  std::vector<rn_chain_stats> stats((size_t)chains);
  const int rc = rn_sample_generate((rn_model*)(intptr_t)m, (const rn_config*)env->GetDirectBufferAddress(config), (rn_generator*)(intptr_t)g,
                                    s64.data(), (int)chains, vo.data(), nullptr, stats.data());
  if (rc != RN_OK) return throw_last(env);
  std::vector<rn_rng_state> st((size_t)chains);
  for (jsize c = 0; c < chains; c++) st[c] = stats[c].rng;
  rng_out(env, rngOut, st);
  out_doubles(env, out, vo.data(), vo.size());
}
// ---- Optimizer.lbfgs for a batch of starts (optimizer/Optimizer.scala:6-24) ----
// def optimize(handle: Long, x0: Array[Double] /* [starts][n] or null */, starts: Int, m: Int, eps: Double, maxEvals: Int,
//              x: Array[Double] /* [starts][n] */, info: Array[Int]): Unit
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_optimize(JNIEnv* env, jclass, jlong h, jdoubleArray x0, jint starts, jint m,
                                                                    jdouble eps, jint maxEvals, jdoubleArray x, jintArray info) {
  rn_optimize_config oc;
  rn_optimize_config_default(&oc);
  oc.history = m;
  oc.eps = eps;
  oc.max_evaluations = maxEvals;
  const std::vector<double> v0 = in_doubles(env, x0);
  std::vector<double> vx((size_t)env->GetArrayLength(x));
  std::vector<int32_t> vi(info ? (size_t)env->GetArrayLength(info) : 0);
  const int rc = rn_optimize((rn_model*)(intptr_t)h, &oc, x0 ? v0.data() : nullptr, starts, vx.data(), nullptr, vi.empty() ? nullptr : vi.data(), nullptr);
  if (rc != RN_OK) return throw_last(env);
  out_doubles(env, x, vx.data(), vx.size());
  if (info) env->SetIntArrayRegion(info, 0, (jsize)vi.size(), (const jint*)vi.data());
}
// ---- Trace.thin(thin).diagnostics tracked while a staged sampler runs (rn_sampler_track_diagnostics) ----
// def samplerTrackDiagnostics(sampler: Long, thin: Int): Unit
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_samplerTrackDiagnostics(JNIEnv* env, jclass, jlong s, jint thin) {
  if (rn_sampler_track_diagnostics((rn_sampler*)(intptr_t)s, thin) != RN_OK) throw_last(env);
}
// def samplerTrackedDiagnostics(sampler: Long, out: Array[Double] /* [n][2] = rHat, ess */): Unit   (a collective with a communicator)
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_samplerTrackedDiagnostics(JNIEnv* env, jclass, jlong s, jdoubleArray out) {
  std::vector<double> vo((size_t)env->GetArrayLength(out));
  if (rn_sampler_tracked_diagnostics((rn_sampler*)(intptr_t)s, vo.data()) != RN_OK) return throw_last(env);
  out_doubles(env, out, vo.data(), vo.size());
}
// def samplerTrajectoryLengths(sampler: Long, counts: Array[Long] /* or null: size only */): Int   (bins = maxSteps + 1)
JNIEXPORT jint JNICALL Java_com_stripe_rainier_cuda_Native_samplerTrajectoryLengths(JNIEnv* env, jclass, jlong s, jlongArray counts) {
  int n = 0;
  if (rn_sampler_trajectory_lengths((rn_sampler*)(intptr_t)s, nullptr, 0, &n) != RN_OK) return throw_last(env), 0;
  if (counts) {
    std::vector<int64_t> v((size_t)n);
    if (rn_sampler_trajectory_lengths((rn_sampler*)(intptr_t)s, v.data(), n, &n) != RN_OK) return throw_last(env), 0;
    env->SetLongArrayRegion(counts, 0, std::min<jsize>(env->GetArrayLength(counts), (jsize)n), (const jlong*)v.data());
  }
  return (jint)n;
}
// ---- checkpoints of a staged sampler (rn_sampler_save / rn_sampler_restore); blobs travel in direct ByteBuffers ----
// def samplerSave(sampler: Long, out: ByteBuffer /* direct, or null: size only */): Long   (bytes of the checkpoint)
JNIEXPORT jlong JNICALL Java_com_stripe_rainier_cuda_Native_samplerSave(JNIEnv* env, jclass, jlong s, jobject out) {
  size_t need = 0;
  void* p = out ? env->GetDirectBufferAddress(out) : nullptr;
  const size_t cap = out ? (size_t)env->GetDirectBufferCapacity(out) : 0;
  if (rn_sampler_save((rn_sampler*)(intptr_t)s, p, cap, &need) != RN_OK) throw_last(env);
  return (jlong)need;
}
// def samplerRestore(model: Long, config: ByteBuffer, blobs: Array[ByteBuffer], lens: Array[Long]): Long   (an rn_sampler handle)
JNIEXPORT jlong JNICALL Java_com_stripe_rainier_cuda_Native_samplerRestore(JNIEnv* env, jclass, jlong m, jobject config, jobjectArray blobs,
                                                                           jlongArray lens) {
  const jsize k = env->GetArrayLength(blobs);
  std::vector<const void*> ptrs((size_t)k);
  for (jsize i = 0; i < k; i++) ptrs[i] = env->GetDirectBufferAddress(env->GetObjectArrayElement(blobs, i));
  const std::vector<int64_t> l64 = in_longs(env, lens);
  const std::vector<size_t> ls(l64.begin(), l64.end());
  rn_sampler* s = nullptr;
  if (rn_sampler_restore((rn_model*)(intptr_t)m, (const rn_config*)env->GetDirectBufferAddress(config), ptrs.data(), ls.data(), (int)k,
                         &s) != RN_OK) {
    throw_last(env);
    return 0;
  }
  return (jlong)(intptr_t)s;
}
// def checkpointInfo(blob: ByteBuffer, len: Long, out: Array[Long]): Unit
//   out = [version, phase, n, chains, chainOffset, warmDone, trackKept, totalBytes]
JNIEXPORT void JNICALL Java_com_stripe_rainier_cuda_Native_checkpointInfo(JNIEnv* env, jclass, jobject blob, jlong len, jlongArray out) {
  struct rn_checkpoint_info i;
  if (rn_checkpoint_info(env->GetDirectBufferAddress(blob), (size_t)len, &i) != RN_OK) return throw_last(env);
  const jlong v[8] = {i.version, i.phase, i.n, i.chains, i.chain_offset, i.warm_done, i.track_kept, (jlong)i.total_bytes};
  env->SetLongArrayRegion(out, 0, 8, v);
}
// def checkpointSlice(blob: ByteBuffer, len: Long, begin: Long, end: Long, out: ByteBuffer /* or null: size only */): Long
JNIEXPORT jlong JNICALL Java_com_stripe_rainier_cuda_Native_checkpointSlice(JNIEnv* env, jclass, jobject blob, jlong len, jlong begin,
                                                                            jlong end, jobject out) {
  size_t need = 0;
  void* p = out ? env->GetDirectBufferAddress(out) : nullptr;
  const size_t cap = out ? (size_t)env->GetDirectBufferCapacity(out) : 0;
  if (rn_checkpoint_slice(env->GetDirectBufferAddress(blob), (size_t)len, begin, end, p, cap, &need) != RN_OK) throw_last(env);
  return (jlong)need;
}
JNIEXPORT jstring JNICALL Java_com_stripe_rainier_cuda_Native_lastError(JNIEnv* env, jclass) {
  return env->NewStringUTF(rn_last_error());
}

}  // extern "C"
#endif  // RN_HAVE_JNI
