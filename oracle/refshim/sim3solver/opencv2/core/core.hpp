// <opencv2/core/core.hpp> for the in-place build of src/Sim3Solver.cc only (oracle/sim3solver.mk)
#include "../../../refshim_cv_sim3solver.h"
