// <opencv2/opencv.hpp> for the in-place build of src/KeyFrame.cc only (oracle/covis.mk)
#include "../../refshim_cv_keyframe.h"
