// <opencv2/features2d/features2d.hpp> for the in-place build of src/LocalMapping.cc for the keyframe-insertion checkers (oracle/kfinsert.mk)
#include "../../../refshim_cv_kfinsert.h"
