// oracle/refshim/refshim_cv_keyframe.h — TEST INFRASTRUCTURE ONLY.
// The OpenCV C++ API as src/KeyFrame.cc and the headers it includes use it, so that the reference's own file compiles in
// place (oracle/covis.mk -> _ref/libref_keyframe.so; the include directory refshim/keyframe puts it behind the OpenCV
// headers).  It is refshim_cv_sim3solver.h (Mat_<float>, copyTo into a rowRange / colRange view, eye, dot, the matrix
// expressions of SetPose) plus the names include/ORBextractor.h declares with: Point, Point2i, InputArray, OutputArray.
#pragma once
#include "refshim_cv_sim3solver.h"

namespace cv {
typedef Point_<int> Point2i;
typedef Point2i Point;
typedef const Mat& InputArray;
typedef Mat& OutputArray;
}  // namespace cv
