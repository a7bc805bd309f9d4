// <opencv2/opencv.hpp> for the in-place build of src/Initializer.cc only (oracle/init.mk)
#include "../../refshim_cv_init.h"
