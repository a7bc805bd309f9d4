// <opencv2/opencv.hpp> for the in-place build of src/LocalMapping.cc only (oracle/culling.mk)
#include "../../refshim_cv_localmapping.h"
