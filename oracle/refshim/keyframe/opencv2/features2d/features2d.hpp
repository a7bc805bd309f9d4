// <opencv2/features2d/features2d.hpp> for the in-place build of src/KeyFrame.cc only (oracle/covis.mk)
#include "../../../refshim_cv_keyframe.h"
