/*
 * GBMRegressionModelNative.scala — the reference's GBMRegressionModel with transform() evaluated per PARTITION on the
 * H100 instead of per row on the JVM (regression/GBMRegressor.scala:531-539:
 *     sum = init.predict(x); for (i <- models) sum += models(i).predict(slice(subspaces(i))(x)) * weights(i)).
 *
 * Two routes, both through org.apache.spark.ml.se.SeNative (include/se_abi.h):
 *   every member is a DecisionTreeRegressionModel with continuous splits
 *       -> the partition's features go to HBM once (uploadRowmajor), the trees are flattened and concatenated
 *          (FlatTree, GBMRegressorNative.scala) with their feature indices mapped through subspaces(i), and
 *          SeNative.forestPredict writes init + Σ weights(i)·tree_i(x) in one pass over the uint8 rank matrix
 *          (se_forest_predict: no [M][n] intermediate);
 *   anything else
 *       -> each member predicts on the host into Slot.P ([M][n]) and SeNative.aggRun forms the weighted sum
 *          (SE_AGG_GBM_REGRESSOR), as INTEGRATION.md §3 describes for every model family.
 * predict(features: Vector) for single rows stays the reference's.
 *
 * NOT COMPILED in this repository's image (no JDK / scalac / sbt / Spark jars).
 */
package org.apache.spark.ml.regression

import org.apache.spark.ml.ensemble.EnsemblePredictionModelType
import org.apache.spark.ml.linalg.Vector
import org.apache.spark.ml.param.ParamMap
import org.apache.spark.ml.se.SeNative
import org.apache.spark.ml.se.SeNative.{Agg, Slot}
import org.apache.spark.ml.tree.{ContinuousSplit, InternalNode, Node}
import org.apache.spark.sql.{DataFrame, Dataset, Row}
import org.apache.spark.sql.functions.col

class GBMRegressionModelNative(
    uid: String,
    weights: Array[Double],
    subspaces: Array[Array[Int]],
    models: Array[EnsemblePredictionModelType],
    init: EnsemblePredictionModelType,
    val device: Int = 0)
    extends GBMRegressionModel(uid, weights, subspaces, models, init) {

  private def continuousOnly(node: Node): Boolean = node match {
    case n: InternalNode => n.split.isInstanceOf[ContinuousSplit] && continuousOnly(n.leftChild) && continuousOnly(n.rightChild)
    case _ => true
  }

  private lazy val flatForest: Option[(Array[Int], FlatTree)] = {
    val trees = models.collect { case t: DecisionTreeRegressionModel if continuousOnly(t.rootNode) => t }
    if (trees.length != models.length || models.isEmpty) None
    else {
      val flats = trees.zip(subspaces).map { case (t, sub) =>
        val f = FlatTree(t)
        f.copy(feature = f.feature.map(j => if (j < 0) j else sub(j)))   // HasSubBag.slice (:81-84) folded into the node
      }
      val offsets = flats.scanLeft(0)(_ + _.feature.length)
      Some((offsets, FlatTree(flats.flatMap(_.feature), flats.flatMap(_.threshold), flats.flatMap(_.left),
        flats.flatMap(_.right), flats.flatMap(_.value))))
    }
  }

  /** Predictions of one partition (rows in partition order). */
  private[regression] def predictPartition(rows: Array[Vector]): Array[Double] = {
    val n = rows.length
    if (n == 0) return Array.emptyDoubleArray
    val ctx = SeNative.ctxCreate(device)
    try {
      val out = new Array[Float](n)
      flatForest match {
        case Some((offsets, forest)) if init.isInstanceOf[DummyRegressionModel] =>
          val d = rows.head.size
          SeNative.slotAlloc2d(ctx, Slot.X, d.toLong, n.toLong)
          val chunk = math.max(1, (1 << 22) / d)
          var done = 0
          while (done < n) {
            val m = math.min(chunk, n - done)
            val buf = new Array[Float](m * d)
            var r = 0
            while (r < m) { rows(done + r).foreachActive((j, x) => buf(r * d + j) = x.toFloat); r += 1 }
            SeNative.uploadRowmajor(ctx, Slot.X, buf, m.toLong, d, done.toLong)
            done += m
          }
          SeNative.slotAlloc2d(ctx, Slot.RAW, 1L, n.toLong)
          // a DummyRegressionModel predicts a constant: it is the `init` of the sum (:532)
          SeNative.forestPredict(ctx, 0, models.length, offsets, forest.feature, forest.threshold, forest.left, forest.right,
            forest.value, weights, init.predict(rows.head), Slot.RAW, 0)
        case _ =>
          // host members into Slot.P, weighted sum on the device; a non-constant init is added on the host below
          SeNative.aggConfigure(ctx, Agg.GbmRegressor, models.length, 0, 1, 0, n.toLong)
          var i = 0
          while (i < models.length) {
            val sub = subspaces(i)
            SeNative.uploadF64(ctx, Slot.P, rows.map(x => models(i).predict(slice(sub)(x))), n.toLong, i.toLong * n)
            i += 1
          }
          SeNative.aggRun(ctx, weights, Array(0.0))
      }
      SeNative.download(ctx, Slot.RAW, out, n.toLong, 0L)
      val constantInit = flatForest.isDefined && init.isInstanceOf[DummyRegressionModel]
      if (constantInit) out.map(_.toDouble) else rows.zip(out).map { case (x, s) => init.predict(x) + s }
    } finally SeNative.ctxDestroy(ctx)
  }

  override def transform(dataset: Dataset[_]): DataFrame = {
    transformSchema(dataset.schema, logging = true)
    val spark = dataset.sparkSession
    val featuresIdx = dataset.schema.fieldIndex($(featuresCol))
    val outSchema = dataset.schema.add($(predictionCol), org.apache.spark.sql.types.DoubleType)
    val model = this
    val rdd = dataset.toDF.rdd.mapPartitions { it =>
      val part = it.toArray
      val pred = model.predictPartition(part.map(_.getAs[Vector](featuresIdx)))
      part.iterator.zip(pred.iterator).map { case (row, p) => Row.fromSeq(row.toSeq :+ p) }
    }
    spark.createDataFrame(rdd, outSchema)
  }

  override def copy(extra: ParamMap): GBMRegressionModelNative =
    copyValues(new GBMRegressionModelNative(uid, weights, subspaces, models, init, device), extra).setParent(parent)
}
