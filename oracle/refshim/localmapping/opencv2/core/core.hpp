// <opencv2/core/core.hpp> for the in-place build of src/LocalMapping.cc only (oracle/culling.mk)
#include "../../../refshim_cv_localmapping.h"
