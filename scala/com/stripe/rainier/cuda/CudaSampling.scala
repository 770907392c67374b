package com.stripe.rainier.cuda

import java.nio.{ByteBuffer, ByteOrder}
import com.stripe.rainier.compute.CudaCompiler
import com.stripe.rainier.core._
import com.stripe.rainier.sampler._

/** The batched replacement for `Model.sample` (core/Model.scala:13-24) and `Model.density()` (core/Model.scala:38-50).
  *
  * `sample` keeps the reference's signature.  Instead of looping `Driver.sample` over chains on one JVM thread it
  * lowers the `SamplerConfig` to an `rn_config` and runs every chain in ONE `rn_sample` call; `Stats`, `MassMatrix`
  * and `Trace` objects are rebuilt on the host so rainier-notebook (HTMLProgress) and `Trace.diagnostics/predict`
  * keep working unchanged.  Only the built-in samplers/tuners can be lowered; anything else is an explicit error --
  * there is no CPU fallback.
  *
  * Requires one mechanical change in rainier-sampler: the constructor parameters of `HMCSampler`, `EHMCSampler`,
  * `DualAvgTuner` and the windowed tuners become `val`s (they are private today: HMC.scala:3, EHMC.scala:3-6,
  * DualAvg.scala:3) so that they can be read here.
  *
  * Seeding rule (SURVEY.md 8c): chain c behaves exactly like a single-chain reference run with
  * `ScalaRNG(seeds(c))`; seeds are drawn from the implicit rng (`rng.standardUniform`-derived longs), one per chain.
  *
  * NOT COMPILED in the rainier_b200 repository (no JVM toolchain in its build image); see INTEGRATION.md.
  */
object CudaSampling {
  /** trajectoryAdaptation: rn_config.trajectory_adaptation (0 per chain, the reference's EHMC; 1 pooled: one shared
    * trajectory length per sampling iteration, drawn from all chains' U-turn counts, EHMCSampler only) */
  def sample(model: Model, config: SamplerConfig = SamplerConfig.default, nChains: Int = 4, device: Int = 0,
             trajectoryAdaptation: Int = 0)(
      implicit rng: RNG = RNG.default,
      progress: Progress = SilentProgress): Trace = {
    val cm = CudaCompiler.compileTargets(model.targetGroup, withGradient = false, device = device)
    try {
      val n = cm.nVars
      val cfg = lower(config)
      cfg.putInt(OffTrajAdaptation, trajectoryAdaptation)
      val seeds = Array.fill(nChains)((rng.standardUniform * (1L << 48)).toLong)
      // results land in page-locked memory (one DMA, no staging copy); read back through a DoubleBuffer view
      val sampleBytes = nChains.toLong * config.iterations * n * 8
      val sampleBuf = Native.hostAlloc(device, sampleBytes).order(ByteOrder.LITTLE_ENDIAN)
      val samples = sampleBuf.asDoubleBuffer()
      try {
      val dense = cfg.getInt(OffMassTuner) == 2
      val mass = new Array[Double](nChains * (if (dense) n * n else n))
      val statsBuf = ByteBuffer.allocateDirect(nChains * Native.statsSize()).order(ByteOrder.LITTLE_ENDIAN)
      1.to(nChains).foreach(progress.start)
      Native.sampleDirect(cm.handle, cfg, seeds, sampleBuf, mass, statsBuf)
      val chains = 0.until(nChains).toList.map { c =>
        0.until(config.iterations).toList.map { i =>
          val row = new Array[Double](n)
          samples.position((c * config.iterations + i) * n)
          samples.get(row)
          row
        }
      }
      val masses: List[MassMatrix] = 0.until(nChains).toList.map { c =>
        cfg.getInt(OffMassTuner) match {
          case 0 => IdentityMassMatrix
          case 2 => DenseMassMatrix(java.util.Arrays.copyOfRange(mass, c * n * n, (c + 1) * n * n))
          case _ => DiagonalMassMatrix(java.util.Arrays.copyOfRange(mass, c * n, (c + 1) * n))
        }
      }
      val stats = 0.until(nChains).toList.map(c => readStats(statsBuf, c, config.statsWindow))
      stats.zip(masses).zipWithIndex.foreach { case ((s, m), c) => progress.finish(c + 1, "Complete", s, m) }
      Trace(chains, masses, stats, model)
      } finally Native.hostFree(device, sampleBuf)
    } finally cm.close()
  }

  // ---- rn_config field offsets (include/rainier_cuda.h; checked against Native.configSize at class load) ----
  private val OffIterations = 4; private val OffWarmup = 8; private val OffStatsWindow = 12
  private val OffSampler = 16; private val OffNSteps = 20; private val OffMaxSteps = 24; private val OffMinSteps = 28
  private val OffBufSize = 32; private val OffPCount = 40
  private val OffStepTuner = 48; private val OffDelta = 56; private val OffStaticStep = 64
  private val OffMassTuner = 72; private val OffInitWindow = 76; private val OffExpansion = 80
  private val OffSkipFirst = 88; private val OffSkipLast = 92; private val OffTrajAdaptation = 100
  require(Native.configSize() == 152, "rn_config layout changed")

  private def lower(config: SamplerConfig): ByteBuffer = {
    val b = ByteBuffer.allocateDirect(Native.configSize()).order(ByteOrder.LITTLE_ENDIAN)
    Native.defaultConfig(b)
    b.putInt(OffIterations, config.iterations).putInt(OffWarmup, config.warmupIterations).putInt(OffStatsWindow, config.statsWindow)
    config.sampler() match {
      case s: HMCSampler  => b.putInt(OffSampler, 0).putInt(OffNSteps, s.nSteps)
      case s: EHMCSampler =>
        b.putInt(OffSampler, 1).putInt(OffMaxSteps, s.maxSteps).putInt(OffMinSteps, s.minSteps)
          .putInt(OffBufSize, s.bufSize).putDouble(OffPCount, s.pCount)
      case other => sys.error(s"${other.getClass} cannot be lowered to the GPU; only HMCSampler/EHMCSampler")
    }
    config.stepSizeTuner() match {
      case t: DualAvgTuner    => b.putInt(OffStepTuner, 0).putDouble(OffDelta, t.delta)
      case StaticStepSize(ss) => b.putInt(OffStepTuner, 1).putDouble(OffStaticStep, ss)
      case other              => sys.error(s"${other.getClass} cannot be lowered to the GPU")
    }
    config.massMatrixTuner() match {
      case _: IdentityMassMatrixTuner => b.putInt(OffMassTuner, 0)
      case t: DenseMassMatrixTuner    => windowed(b, 2, t)
      case t: DiagonalMassMatrixTuner => windowed(b, 1, t)
      case StaticMassMatrix(IdentityMassMatrix) => b.putInt(OffMassTuner, 0)
      case other => sys.error(s"${other.getClass}: static non-identity matrices go through rn_config.static_matrix_elements (C ABI only)")
    }
    b
  }
  private def windowed(b: ByteBuffer, kind: Int, t: WindowedMassMatrixTuner): ByteBuffer =
    b.putInt(OffMassTuner, kind).putInt(OffInitWindow, t.initialWindowSize).putDouble(OffExpansion, t.windowExpansion)
      .putInt(OffSkipFirst, t.skipFirst).putInt(OffSkipLast, t.skipLast)

  /** rn_chain_stats -> Stats (sampler/Stats.scala:3-17).  gradientTimes / iterationTimes (read by HTMLProgress.scala:57,65
    * through `.mean`) receive one entry each: device time of the sampling launches / this chain's gradient evaluations,
    * and / iterations of the batch -- all chains advance together, there is no per-call wall clock to record. */
  private def readStats(buf: ByteBuffer, c: Int, window: Int): Stats = {
    val o = c * Native.statsSize()
    val s = new Stats(window)
    s.gradientEvaluations = buf.getLong(o)
    s.iterations = buf.getInt(o + 16)
    s.divergences = buf.getInt(o + 20)
    s.energyVariance.mean(0) = buf.getDouble(o + 40)
    s.energyVariance.raw(0) = buf.getDouble(o + 48)
    s.energyTransitions2 = buf.getDouble(o + 56)
    s.energyVariance.samples = buf.getInt(o + 64)
    s.stepSizes.add(buf.getDouble(o + 96)) // means; full ring contents are available through rn_config.stats_rings
    s.acceptanceRates.add(buf.getDouble(o + 104))
    s.gradsPerIteration.add(buf.getDouble(o + 112))
    s.gradientTimes.add(buf.getDouble(o + 144))
    s.iterationTimes.add(buf.getDouble(o + 152))
    s
  }

  /** Checkpoint of a staged sampler (rn_sampler_save, DESIGN.md 3.6): its whole state in page-locked memory (one DMA per
    * chunk), to be written to a file or restored in another process or on another device.  Free with Native.hostFree. */
  def save(sampler: Long, device: Int = 0): ByteBuffer = {
    val buf = Native.hostAlloc(device, Native.samplerSave(sampler, null))
    Native.samplerSave(sampler, buf)
    buf
  }

  /** rn_sampler_restore: a staged sampler (handle) that continues the blobs' chains, concatenated in order, with the same bits
    * as the uninterrupted run.  `config` must agree with the checkpoints' semantic fields; `iterations` may grow, so that a
    * finished run can be extended.  Each blob's bytes are its limit. */
  def restore(model: Long, config: SamplerConfig, blobs: Seq[ByteBuffer]): Long =
    Native.samplerRestore(model, lower(config), blobs.toArray, blobs.map(_.limit.toLong).toArray)

  /** `Model.density()` for API completeness (Optimizer.lbfgs, JMH): one crossing per update -- NOT the fast path. */
  def density(model: Model, device: Int = 0): DensityFunction = {
    val cm = CudaCompiler.compileTargets(model.targetGroup, withGradient = false, device = device)
    new DensityFunction {
      val nVars = cm.nVars
      private val out = new Array[Double](nVars + 1)
      def update(vars: Array[Double]): Unit = Native.densityBatch(cm.handle, vars, 1, out)
      def density = out(0)
      def gradient(index: Int) = out(index + 1)
    }
  }

  /** `Trace.predict` (core/Trace.scala:34-41) with the requirement values of ALL draws computed by one native call.
    * Mirrors `Generator.prepare` (core/Generator.scala:59-94): same requirement list (`requirements.toList.take(
    * Generator.MaxRequirements)`), same Evaluator contents, `get` applied per draw in the reference's order, so a
    * generator consumes the RNG exactly as before.  `CudaCompiler.compileFunction` = the unchanged `Translator` +
    * RIR serialisation with RIR_FLAG_FUNCTION (the `Compiler.compile(inputs, outputs)` seam, compute/Compiler.scala:22-30). */
  def predict[T, U](trace: Trace, value: T, device: Int = 0)(implicit tg: ToGenerator[T, U], rng: RNG): List[U] = {
    val gen = tg(value)
    val params = trace.model.parameters
    val reqs = gen.requirements.toList.take(Generator.MaxRequirements)
    val draws = trace.chains.flatten
    if (reqs.isEmpty)
      draws.map(a => gen.get(rng, new Evaluator(params.zip(a).toMap)))
    else {
      val n = params.size; val m = reqs.size
      val h = Native.functionCreate(CudaCompiler.compileFunction(params.map(_.param), reqs), device)
      try {
        val flat = new Array[Double](draws.size * n)
        draws.zipWithIndex.foreach { case (a, i) => System.arraycopy(a, 0, flat, i * n, n) }
        val out = new Array[Double](draws.size * m)
        Native.functionEval(h, flat, draws.size.toLong, out)
        draws.zipWithIndex.map { case (a, i) =>
          gen.get(rng, new Evaluator((params.zip(a) ++ reqs.zipWithIndex.map { case (r, j) => r -> out(i * m + j) }).toMap))
        }
      } finally Native.functionDestroy(h)
    }
  }

  /** `Model.optimize` (core/Model.scala:26-30): `Optimizer.lbfgs(density())` (optimizer/Optimizer.scala:6-24) fused into
    * one kernel; the single reference start x = 0, m = 5, eps = 0.1.  `optimizeMultiStart` returns the best of several
    * starts (an extension: the reference has one start). */
  def optimize[T, U](model: Model, t: T, device: Int = 0)(implicit toGen: ToGenerator[T, U], rng: RNG): U = {
    val cm = CudaCompiler.compileTargets(model.targetGroup, withGradient = false, device = device)
    try {
      val x = new Array[Double](cm.nVars); val info = new Array[Int](1)
      Native.optimize(cm.handle, null, 1, 5, 0.1, 10000, x, info)
      if ((info(0) & 2) != 0) throw new RuntimeException("dginit") // LBFGS.java:253-254
      toGen(t).prepare(model.parameters).apply(x)
    } finally cm.close()
  }
}
