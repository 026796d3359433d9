package org.apache.spark.mllib.optimization

import org.apache.spark.Logging
import org.apache.spark.annotation.DeveloperApi
import org.apache.spark.mllib.linalg.{DenseVector, SparseVector, Vector, Vectors}
import org.apache.spark.rdd.RDD

/** Drop-in for staple/spark-agd's optimizer: same package, class, constructor, setters, `optimize`
  * and `run`, but the loop executes natively on the box's H100s through NativeAGD (JNI over
  * include/agd_b200.h).  Source only -- no JVM in the build image.
  *
  * Deployment: ONE executor JVM per GPU box (or `local[N]`), owning all of the box's GPUs.  Data path: each RDD
  * partition is packed by the executor task that computes it -- `mapPartitionsWithIndex`, never the driver -- into
  * primitive arrays of at most 1 GiB and handed to GPU `partition % G` (the analogue of `.cache()`); after that no row
  * crosses the JVM boundary again, and the whole of `run` (AGD.scala:177-338) is one native call made by a one-task job
  * on that executor.  System properties (read on the driver, shipped in the closures):
  *   -Dagd.devices=0,1,...   GPUs of the box (default 0)
  *   -Dagd.store=f64|f32|bf16  HBM storage of dense features.  f64 (default) keeps every `Double` exact; f32 is the
  *                           benchmarked layout (half the bytes, twice the examples/s) and ROUNDS features to fp32 --
  *                           exact when the RDD was built from floats; bf16 (d % 128 == 0) selects the wgmma kernel
  *   -Dagd.flags=0|1|2       agd_params.flags: 0 = the reference's evaluations, fused sweeps; 1 = AGD_FLAG_MEMOIZE_FX;
  *                           2 = AGD_FLAG_NO_FUSE */
@DeveloperApi
class AcceleratedGradientDescent(private var gradient: Gradient, private var updater: Updater) extends Optimizer {
  private var convergenceTol = 1e-4; private var numIterations = 100; private var regParam = 0.0
  private var L0 = 1.0; private var Lexact = Double.PositiveInfinity
  private var beta = 0.5; private var alpha = 0.9; private var mayRestart = true

  def setConvergenceTol(tol: Double): this.type = { convergenceTol = tol; this }
  def setNumIterations(iters: Int): this.type = { numIterations = iters; this }
  def setRegParam(reg: Double): this.type = { regParam = reg; this }
  def setL0(v: Double): this.type = { L0 = v; this }
  def setLexact(v: Double): this.type = { Lexact = v; this }
  def setBeta(v: Double): this.type = { beta = v; this }
  def setAlpha(v: Double): this.type = { alpha = v; this }
  def setMayRestart(v: Boolean): this.type = { mayRestart = v; this }
  def setGradient(g: Gradient): this.type = { gradient = g; this }
  def setUpdater(u: Updater): this.type = { updater = u; this }

  def optimize(data: RDD[(Double, Vector)], initialWeights: Vector): Vector =
    AcceleratedGradientDescent.run(data, gradient, updater, convergenceTol, numIterations, regParam,
      initialWeights, L0, Lexact, beta, alpha, mayRestart)._1
}

@DeveloperApi
object AcceleratedGradientDescent extends Logging {
  private def flags: Int = sys.props.get("agd.flags").map(_.trim.toInt).getOrElse(0)
  private def devices: Array[Int] =
    sys.props.get("agd.devices").map(_.split(',').map(_.trim.toInt)).getOrElse(Array(0))
  private def storeDtype: Int = sys.props.get("agd.store").map(_.trim.toLowerCase).getOrElse("f64") match {
    case "f64" => NativeAGD.F64
    case "f32" => NativeAGD.F32
    case "bf16" => NativeAGD.BF16
    case other => throw new IllegalArgumentException(s"agd.store must be f64, f32 or bf16 (got $other)")
  }

  /** Doubles per packed chunk: 2^27 = 1 GiB, far below the 2^31 - 1 elements a Java array can hold. */
  private val ChunkDoubles = 1 << 27

  /** Runs on the executor: packs one partition chunk by chunk and loads it onto GPU `p % G`.  Returns (p, rows). */
  private def loadPartition(p: Int, rows: Iterator[(Double, Vector)], d: Int, devs: Array[Int], store: Int): (Int, Long) = {
    val h = NativeAGD.sharedHandle(devs)
    val dev = p % devs.length
    val chunkRows = math.max(1, ChunkDoubles / d)
    var total = 0L
    val it = rows.buffered
    while (it.hasNext) {
      if (it.head._2.isInstanceOf[DenseVector]) {
        // dense run: up to chunkRows consecutive DenseVector rows, copied once into one primitive array
        val x = new Array[Double](math.min(chunkRows.toLong * d, ChunkDoubles.toLong).toInt)
        val labels = new Array[Double](chunkRows)
        var n = 0
        while (n < chunkRows && it.hasNext && it.head._2.isInstanceOf[DenseVector]) {
          val (label, v) = it.next()
          require(v.size == d, s"feature vector of size ${v.size} in partition $p, weights have size $d")
          System.arraycopy(v.asInstanceOf[DenseVector].values, 0, x, n * d, d)
          labels(n) = label
          n += 1
        }
        NativeAGD.loadDense(h, dev, x, labels, n, d, store)
        total += n
      } else {
        // sparse run: SparseVector rows as CSR, at most ChunkDoubles stored entries per call
        val rowptr = new scala.collection.mutable.ArrayBuffer[Long](); rowptr += 0L
        val idx = new scala.collection.mutable.ArrayBuffer[Int]()
        val values = new scala.collection.mutable.ArrayBuffer[Double]()
        val labels = new scala.collection.mutable.ArrayBuffer[Double]()
        while (it.hasNext && !it.head._2.isInstanceOf[DenseVector] && values.length < ChunkDoubles) {
          val (label, v) = it.next()
          require(v.size == d, s"feature vector of size ${v.size} in partition $p, weights have size $d")
          val s = v match { case sv: SparseVector => sv; case other => Vectors.dense(other.toArray).toSparse }
          idx ++= s.indices; values ++= s.values
          rowptr += values.length.toLong
          labels += label
        }
        // CSR shards store fp32 or fp64 values
        NativeAGD.loadCsr(h, dev, rowptr.toArray, idx.toArray, values.toArray, labels.toArray, labels.length, d,
          if (store == NativeAGD.BF16) NativeAGD.F32 else store)
        total += labels.length
      }
    }
    (p, total)
  }

  def run(data: RDD[(Double, Vector)], gradient: Gradient, updater: Updater, convergenceTol: Double,
          numIterations: Int, regParam: Double, initialWeights: Vector, L0: Double, Lexact: Double, beta: Double,
          alpha: Double, mayRestart: Boolean): (Vector, Array[Double]) = {
    val g = NativeAGD.gradientId(gradient); val u = NativeAGD.updaterId(updater)   // fail before touching data
    val d = initialWeights.size
    val devs = devices; val store = storeDtype; val fl = flags
    val sc = data.sparkContext
    // job 1 (executor side): drop what a previous optimize() left in HBM, then pack + load every partition in parallel
    sc.parallelize(Seq(0), 1).foreach(_ => NativeAGD.clear(NativeAGD.sharedHandle(devs)))
    val loaded = data.mapPartitionsWithIndex((p, rows) => Iterator(loadPartition(p, rows, d, devs, store))).collect()
    logInfo("AcceleratedGradientDescent: %d rows in %d partitions resident on %d GPU(s)".format(
      loaded.map(_._2).sum, loaded.length, devs.length))
    // job 2 (one task on the executor that holds the shards): the whole loop, natively
    val w0 = initialWeights.toArray.clone()
    val (w, history, stats) = sc.parallelize(Seq(0), 1).map { _ =>
      val w = w0.clone()
      val stats = new Array[Double](8)
      val hist = NativeAGD.run(NativeAGD.sharedHandle(devs), g, u, convergenceTol, numIterations, regParam, w, L0,
        Lexact, beta, alpha, mayRestart, fl, stats)
      (w, hist, stats)
    }.first()
    if (stats(5) != 0.0) logWarning("Unable to compute loss function.")                       // AGD.scala:310
    logInfo("AcceleratedGradientDescent.run finished. Last 10 losses %s".format(                // AGD.scala:334-335
      history.takeRight(10).mkString(", ")))
    (Vectors.dense(w), history)
  }
}
