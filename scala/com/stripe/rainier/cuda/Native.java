package com.stripe.rainier.cuda;

import java.nio.ByteBuffer;

/**
 * JNI surface of librainier_jni.so (jni/rainier_jni.cpp), a 1:1 forward to the C ABI in include/rainier_cuda.h.
 *
 * A Java class with STATIC natives on purpose: `@native def` inside a Scala `object Native` compiles to instance
 * methods of class `Native$`, for which the JVM looks up `Java_com_stripe_rainier_cuda_Native_00024_create(JNIEnv*,
 * jobject, ...)`; static natives of this class resolve to `Java_com_stripe_rainier_cuda_Native_create(JNIEnv*, jclass,
 * ...)`, which is what the shim exports.  Scala calls them as `Native.create(...)` unchanged (sbt compiles mixed
 * Java/Scala sources).
 *
 * NOT COMPILED in the rainier_b200 repository (no JVM toolchain in its build image); see INTEGRATION.md.
 */
public final class Native {
  static {
    System.loadLibrary("rainier_jni"); // which links librainier_cuda.so
  }

  private Native() {}

  public static native long create(ByteBuffer rir, double[][] cols, int device);

  public static native int nvars(long handle);

  public static native void densityBatch(long handle, double[] q, int chains, double[] out);

  /** samples / mass are filled by region copies after the call returns (no JNI critical section spans the run) */
  public static native void sample(long handle, ByteBuffer config, long[] seeds, double[] samples, double[] mass, ByteBuffer stats);

  /** page-locked host memory (rn_host_alloc) as a direct buffer; rn_sample DMAs straight into it */
  public static native ByteBuffer hostAlloc(int device, long bytes);

  public static native void hostFree(int device, ByteBuffer buf);

  public static native void sampleDirect(long handle, ByteBuffer config, long[] seeds, ByteBuffer samples, double[] mass, ByteBuffer stats);

  public static native String emitSource(long handle, ByteBuffer config);

  public static native int configSize();

  public static native int statsSize();

  public static native void defaultConfig(ByteBuffer config);

  public static native void destroy(long handle);

  /** rn_function_*: Compiler.compile(inputs, outputs) + the CompiledFunction.output loop of Generator.prepare, batched */
  public static native long functionCreate(ByteBuffer rir, int device);

  public static native void functionEval(long handle, double[] draws, long count, double[] out);

  public static native void functionDestroy(long handle);

  /** rn_generator_*: Trace.predict's Generator.get on the device for a RIR_FLAG_GENERATOR container.  rng: long[3 * chains] =
   *  (seed48, doubleToRawLongBits(nextNextGaussian), haveNextNextGaussian) per chain, continued in place */
  public static native long generatorCreate(ByteBuffer rir, int device);

  public static native int generatorOutputs(long handle);

  public static native void generatorEval(long handle, double[] draws, long iterations, long chains, long[] rng, double[] out);

  public static native void generatorDestroy(long handle);

  /** rn_sample_generate: model.sample(config).predict(gen) with the draws on the device; rngOut as generatorEval's rng */
  public static native void sampleGenerate(long model, ByteBuffer config, long generator, long[] seeds, double[] out, long[] rngOut);

  /** rn_optimize: Optimizer.lbfgs for a batch of starts; x0 == null: every start at 0 (the reference's start) */
  public static native void optimize(long handle, double[] x0, int starts, int m, double eps, int maxEvals, double[] x, int[] info);

  /** rn_sampler_track_diagnostics: Trace.thin(thin).diagnostics accumulated on the device over the sampler's following
   *  sampling iterations; sampler is an rn_sampler handle of the staged API */
  public static native void samplerTrackDiagnostics(long sampler, int thin);

  /** rn_sampler_tracked_diagnostics: out [n][2] = rHat, effectiveSampleSize over the tracked draws of every chain (every rank
   *  of an attached communicator calls it) */
  public static native void samplerTrackedDiagnostics(long sampler, double[] out);
  /** rn_sampler_trajectory_lengths: the pooled histogram of U-turn counts (trajectory_adaptation = RN_ADAPT_POOLED, after the
   *  first sampling call) into counts (null: size only); returns maxSteps + 1 */
  public static native int samplerTrajectoryLengths(long sampler, long[] counts);

  /** rn_sampler_save: the staged sampler's whole state into a direct ByteBuffer (page-locked memory from hostAlloc is written by
   *  DMA); out == null returns the size only.  Returns the checkpoint's bytes */
  public static native long samplerSave(long sampler, ByteBuffer out);

  /** rn_sampler_restore: a new staged sampler whose chains are the blobs' chains, concatenated in order (lens: bytes of each) */
  public static native long samplerRestore(long model, ByteBuffer config, ByteBuffer[] blobs, long[] lens);

  /** rn_checkpoint_info, no device: out = [version, phase, n, chains, chainOffset, warmDone, trackKept, totalBytes] */
  public static native void checkpointInfo(ByteBuffer blob, long len, long[] out);

  /** rn_checkpoint_slice, no device: chains [begin, end) as a checkpoint of their own; out == null returns the size only */
  public static native long checkpointSlice(ByteBuffer blob, long len, long begin, long end, ByteBuffer out);

  public static native String lastError();
}
