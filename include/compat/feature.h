// compat/feature.h -- drop-in for the reference's feature.h: every function below has the same name,
// parameter types and in-place vector semantics as its counterpart in reference src/feature.h:27-79,
// but is implemented over the H100 C-ABI (include/vo_b200.h) in libvo_facade.so.  A translation unit of
// the reference that includes "feature.h" keeps compiling when this directory shadows src/.
// (Points / Status are plain aliases: the mangled signatures are the reference's.)
#ifndef FEATURE_H
#define FEATURE_H

#include "vo_cv.h"
#include <vector>

typedef std::vector<cv::Point2f> Points;
typedef std::vector<uchar> Status;

// tracked feature set: positions in the current left image + frames survived   (src/feature.h:33-43)
struct FeatureSet {
    Points points;
    std::vector<int> ages;
    int size() { return (int)points.size(); }
    void clear() { points.clear(); ages.clear(); }
};

// kept for source compatibility; the reference never uses it either            (src/feature.h:27-31)
struct FeaturePoint { cv::Point2f point; int id; int age; };

// ---- detection ------------------------------------------------------------------------------------
void featureDetectionFast(cv::Mat image, Points& points);                    // src/feature.cpp:39-47   -> vo_fast_detect
void featureDetectionGoodFeaturesToTrack(cv::Mat image, Points& points);     // src/feature.cpp:49-62   (not built: throws)
void appendNewFeatures(cv::Mat& image, FeatureSet& current_features);       // src/feature.cpp:255-262
void appendNewFeatures(Points points_new, FeatureSet& current_features);    // src/feature.cpp:264-269
void bucketingFeatures(cv::Mat& image, FeatureSet& current_features,        // src/feature.cpp:206-253
                       int bucket_size, int features_per_bucket);

// ---- tracking -------------------------------------------------------------------------------------
// one LK call + deleteUnmatchFeatures                                         src/feature.cpp:64-74   -> vo_lk_track
void featureTracking(cv::Mat img_1, cv::Mat img_2, Points& points1, Points& points2, Status& status);
void deleteUnmatchFeatures(Points& points0, Points& points1, Status& status);   // src/feature.cpp:20-37

// the ring L0 -> R0 -> R1 -> L1 -> L0 + deleteUnmatchFeaturesCircle            src/feature.cpp:118-148 -> vo_circular_match
void circularMatching(cv::Mat img_l_0, cv::Mat img_r_0, cv::Mat img_l_1, cv::Mat img_r_1,
                      Points& points_l_0, Points& points_r_0, Points& points_l_1, Points& points_r_1,
                      Points& points_l_0_return, FeatureSet& current_features);
// status / negative-coordinate erase loops, ages += 1                          src/feature.cpp:76-116
void deleteUnmatchFeaturesCircle(Points& points0, Points& points1, Points& points2, Points& points3,
                                 Points& points0_return,
                                 Status& status0, Status& status1, Status& status2, Status& status3,
                                 std::vector<int>& ages);

// the reference's USE_CUDA variant (src/feature.cpp:150-204) has the same contract: here it IS the same call
inline void circularMatching_gpu(cv::Mat a, cv::Mat b, cv::Mat c, cv::Mat d, Points& pl0, Points& pr0, Points& pl1,
                                 Points& pr1, Points& pl0_ret, FeatureSet& fs)
{
    circularMatching(a, b, c, d, pl0, pr0, pl1, pr1, pl0_ret, fs);
}

#endif
