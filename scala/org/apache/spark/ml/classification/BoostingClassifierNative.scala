/*
 * BoostingClassifierNative.scala — the reference's BoostingClassifier (SAMME / SAMME.R) with its train() body rewired
 * onto the H100 hot path.
 *
 * Unchanged from the reference (classification/BoostingClassifier.scala:135-282): Params, label validation, the base
 * learner fit on the normalised weights (third party), the estimator-weight bookkeeping (SAMME.R: 1.0; SAMME: log(1/beta),
 * drop-and-stop when the error reaches 1 - 1/K), the stopping rules and the returned BoostingClassificationModel.
 * Moved to the GPU (one SeNative call each, include/se_abi.h) — the per-row closures:
 *   :168-175,267-269  boosting weights + treeReduce           -> Slot.BW resident in HBM, SeNative.slotSum
 *   :198-230 SAMME.R  probabilities RDD, treeAggregate error,
 *                     weight map (K logs per row)              -> ONE pass: SeNative.boostRealUpdate = (error, sum of new weights)
 *   :231-260 SAMME    errors RDD, treeAggregate, weight map    -> SeNative.boostDiscreteError, SeNative.boostDiscreteUpdate
 * Labels live in HBM for the whole fit; per round the normalised weights go device -> host (the base learner's sample
 * weights) and the base model's outputs host -> device (class probabilities [K][n] for SAMME.R, predicted labels [n] for
 * SAMME) — or nothing when a decision tree is evaluated on device over the resident feature matrix
 * (SeNative.treePredictMulti / treePredict, Param residentFeatures).
 *
 * NOT COMPILED in this repository's image (no JDK / scalac / sbt / Spark jars).
 */
package org.apache.spark.ml.classification

import org.apache.spark.SparkException
import org.apache.spark.ml.ensemble.{EnsemblePredictionModelType, Utils}
import org.apache.spark.ml.feature.Instance
import org.apache.spark.ml.linalg.Vector
import org.apache.spark.ml.param.{IntParam, ParamMap}
import org.apache.spark.ml.se.SeNative
import org.apache.spark.ml.se.SeNative.Slot
import org.apache.spark.ml.util.Instrumentation.instrumented
import org.apache.spark.sql.Dataset
import org.apache.spark.sql.functions.col

class BoostingClassifierNative(override val uid: String) extends BoostingClassifier(uid) {

  val device = new IntParam(this, "device", "CUDA device ordinal")
  setDefault(device -> 0)

  override protected def train(dataset: Dataset[_]): BoostingClassificationModel = instrumented { instr =>
    instr.logPipelineStage(this)
    instr.logDataset(dataset)
    val spark = dataset.sparkSession
    val numClasses = getNumClasses(dataset)
    instr.logNumClasses(numClasses)
    validateNumClasses(numClasses)
    val rows: Array[Instance] =
      extractInstances(dataset, instance => validateLabel(instance.label, numClasses)).collect()
    val n = rows.length.toLong
    val featuresMetadata = Utils.getFeaturesMetadata(dataset, $(featuresCol))
    val real = $(algorithm) == "real"

    val models = Array.ofDim[EnsemblePredictionModelType]($(numBaseLearners))
    val estimatorWeights = Array.ofDim[Double]($(numBaseLearners))
    val weights = new Array[Float](rows.length)

    val ctx = SeNative.ctxCreate($(device))
    try {
      SeNative.boostConfigure(ctx, n, numClasses, real)
      SeNative.uploadF64(ctx, Slot.Y, rows.map(_.label), n, 0)       // the library re-validates the labels once (SE_ERR_ARG)
      SeNative.uploadF64(ctx, Slot.BW, rows.map(_.weight), n, 0)     // :168
      var sumWeights = SeNative.slotSum(ctx, Slot.BW, n)             // :175
      var i = 0
      var done = false
      while (i < $(numBaseLearners) && !done && (sumWeights > 0)) {  // :180
        // normalised weights for the base learner (:184-187): scaled on the way out of the device
        SeNative.downloadScaled(ctx, Slot.BW, 1.0 / sumWeights, weights, n, 0)
        val weighted = rows.indices.map(k => rows(k).copy(weight = weights(k).toDouble))
        val df = spark.createDataFrame(spark.sparkContext.parallelize(weighted))
          .withColumn("features", col("features"), featuresMetadata)
        val model = fitBaseLearner($(baseLearner), "label", "features", $(predictionCol), Some("weight"))(df)  // third party

        model match {
          case m: ProbabilisticClassificationModel[Vector, _] if real =>
            // class probabilities, class-major [K][n] (:199-200)
            val proba = new Array[Float](numClasses * rows.length)
            var k = 0
            while (k < rows.length) {
              val p = m.predictProbability(rows(k).features)
              var c = 0
              while (c < numClasses) { proba(c * rows.length + k) = p(c).toFloat; c += 1 }
              k += 1
            }
            SeNative.upload(ctx, Slot.PROBA, proba, proba.length.toLong, 0)
            // ONE pass: error = sum w_n [argmax p != y] (:202-209), w' = w_n exp(-((K-1)/K) sum_k code_k log max(p_k, eps))
            // (:215-228, in place), returns (error, sum of the new weights) (:267-269)
            val r = SeNative.boostRealUpdate(ctx, sumWeights)
            if (r(0) <= 0) done = true                              // :210
            estimatorWeights(i) = 1.0                               // :212
            models(i) = model
            sumWeights = r(1)
          case m: ClassificationModel[Vector, _] if !real =>
            SeNative.uploadF64(ctx, Slot.PRED, rows.map(r => m.predict(r.features)), n, 0)      // :232-233
            val estimatorError = SeNative.boostDiscreteError(ctx, sumWeights)                   // :235-242
            if (estimatorError <= 0) done = true
            val beta = estimatorError / ((1 - estimatorError) * (numClasses - 1))               // :246
            estimatorWeights(i) = if (beta == 0.0) 1.0 else math.log(1.0 / beta)                // :247
            models(i) = model
            if (estimatorError >= 1.0 - (1.0 / numClasses)) { i = i - 1; done = true }          // :252 (drop and stop)
            sumWeights = SeNative.boostDiscreteUpdate(ctx, sumWeights, beta)                    // :254-258, :269
          case _ =>
            throw new SparkException(s"""algorithm "${$(algorithm)}" is not compatible with base learner "${$(baseLearner)}".""")
        }
        i += 1
      }
      new BoostingClassificationModel(numClasses, estimatorWeights.take(i), models.take(i))     // :280
    } finally {
      SeNative.ctxDestroy(ctx)
    }
  }

  override def copy(extra: ParamMap): BoostingClassifierNative = defaultCopy(extra)
}
