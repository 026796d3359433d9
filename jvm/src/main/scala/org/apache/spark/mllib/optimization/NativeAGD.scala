package org.apache.spark.mllib.optimization

/** JNI surface of libagd_jni.so (jvm/src/main/c/agd_jni.c) over include/agd_b200.h.
  * Source only: this image has no JVM, so the facade is not compiled or run here; tests/test_jvm_binding.py checks
  * these declarations against the C shim (names and arities). */
private[optimization] object NativeAGD {
  System.loadLibrary("agd_jni")

  @native def create(devices: Array[Int]): Long
  @native def destroy(handle: Long): Unit
  @native def clear(handle: Long): Unit
  @native def loadDense(handle: Long, dev: Int, x: Array[Double], labels: Array[Double], rows: Long, d: Int,
                        storeDtype: Int): Unit
  @native def loadCsr(handle: Long, dev: Int, rowptr: Array[Long], idx: Array[Int], values: Array[Double],
                      labels: Array[Double], rows: Long, d: Int, storeDtype: Int): Unit
  @native def rows(handle: Long, dev: Int): Long
  @native def run(handle: Long, gradient: Int, updater: Int, convergenceTol: Double, numIterations: Int,
                  regParam: Double, weights: Array[Double], L0: Double, Lexact: Double, beta: Double, alpha: Double,
                  mayRestart: Boolean, flags: Int, stats: Array[Double]): Array[Double]
  @native def smooth(handle: Long, gradient: Int, weights: Array[Double], grad: Array[Double]): Double

  /** AGD_F64 / AGD_F32 / AGD_BF16 of include/agd_b200.h. */
  val F64 = 0; val F32 = 1; val BF16 = 2

  /** Closed enums of include/agd_b200.h; anything else has no GPU implementation and is rejected. */
  def gradientId(g: Gradient): Int = g match {
    case _: LogisticGradient => 0
    case _: LeastSquaresGradient => 1
    case _: HingeGradient => 2
    case other => throw new UnsupportedOperationException(
      s"${other.getClass.getName} has no H100 kernel (Logistic/LeastSquares/Hinge only; there is no CPU fallback)")
  }
  def updaterId(u: Updater): Int = u match {
    case _: SimpleUpdater => 0
    case _: SquaredL2Updater => 1
    case _: L1Updater => 2
    case other => throw new UnsupportedOperationException(
      s"${other.getClass.getName} has no H100 kernel (Simple/SquaredL2/L1 only; there is no CPU fallback)")
  }

  /** The one native handle of THIS JVM (an executor, or the driver in local mode): it owns the box's GPUs and keeps the
    * shards in HBM between the load job and the run job.  Task threads share it; agd_load_* is thread-safe per device. */
  private var handle = 0L
  private var handleDevices: Array[Int] = null
  def sharedHandle(devices: Array[Int]): Long = synchronized {
    if (handle == 0L || !java.util.Arrays.equals(handleDevices, devices)) {
      if (handle != 0L) destroy(handle)
      handle = create(devices)
      handleDevices = devices.clone()
    }
    handle
  }
  def releaseShared(): Unit = synchronized { if (handle != 0L) { destroy(handle); handle = 0L } }
}
