// compat/visualOdometry.h -- drop-in for the reference's visualOdometry.h (reference
// src/visualOdometry.h:27-46): same function names and parameter types, implemented over the H100
// C-ABI (include/vo_b200.h) in libvo_facade.so.
#ifndef VISUAL_ODOM_H
#define VISUAL_ODOM_H

#include "feature.h"
#include "bucket.h"
#include "utils.h"       // as the reference does (src/visualOdometry.h:22)
#include "Frame.h"

// FAST refill (< 2000 features) -> bucketing (rows/10, 1 per bucket) -> circular matching -> 1-px
// round-trip check; on return currentVOFeatures.points = pointsLeft_t1.        src/visualOdometry.cpp:81-129
void matchingFeatures(cv::Mat& imageLeft_t0, cv::Mat& imageRight_t0, cv::Mat& imageLeft_t1, cv::Mat& imageRight_t1,
                      FeatureSet& currentVOFeatures,
                      Points& pointsLeft_t0, Points& pointsRight_t0, Points& pointsLeft_t1, Points& pointsRight_t1);

// solvePnPRansac(500 / 0.5 px / 0.999, ITERATIVE, extrinsic guess = translation) + Rodrigues.
// `translation` is in/out (3x1 CV_64F), `rotation` out (3x3 CV_64F).            src/visualOdometry.cpp:132-193
// mono_rotation = true (the header default, as in the reference; its main() passes false, src/main.cpp:181): `rotation`
// comes from findEssentialMat(RANSAC, 0.999, 1.0) + recoverPose on (pointsLeft_t0, pointsLeft_t1) (:146-157), the PnP then
// only updates `translation`.
void trackingFrame2Frame(cv::Mat& projMatrl, cv::Mat& projMatrr, Points& pointsLeft_t0, Points& pointsLeft_t1,
                         cv::Mat& points3D_t0, cv::Mat& rotation, cv::Mat& translation, bool mono_rotation = true);

// imshow visualisation in the reference (src/visualOdometry.cpp:195-224); a no-op here.
void displayTracking(cv::Mat& imageLeft_t1, Points& pointsLeft_t0, Points& pointsLeft_t1);

// ---- additions of this library (not in the reference) ---------------------------------------------
// The inline OpenCV calls of reference src/main.cpp:170-171 (triangulatePoints + convertPointsFromHomogeneous)
// as one function: fills points3D (N x 1 CV_32FC3).
void triangulateStereo(cv::Mat& projMatrl, cv::Mat& projMatrr, Points& pointsLeft, Points& pointsRight, cv::Mat& points3D);
// Inlier indices of the last trackingFrame2Frame call (the reference only prints how many there are).
const std::vector<int>& lastPnPInliers();
// CUDA device of the process-wide context the facade creates lazily (default 0).
void voCompatSetDevice(int device);

#endif
