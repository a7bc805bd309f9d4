// <opencv/cv.h> for the in-place build of src/LocalMapping.cc for the keyframe-insertion checkers (oracle/kfinsert.mk)
#include "../../refshim_cv_kfinsert.h"
