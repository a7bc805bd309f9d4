// <opencv2/core/core.hpp> for the in-place build of src/PnPsolver.cc only (oracle/pnpsolver.mk)
#include "../../../refshim_cv_pnpsolver.h"
