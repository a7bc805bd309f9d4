# Builds the Sim3 RANSAC checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_sim3solver.so   Sim3Solver::iterate with the minimal sets as input, and the OpenCV operations it needs
#                          (sim3solver.cpp, with init.cpp's gemm; tests/test_oracle_sim3solver.py pins them against cv2)
#   _ref/libref_sim3solver.so, _ref/libadapter_sim3solver.so   (below)
# Used as `make -f sim3solver.mk liborb_sim3solver.so` and `make -f sim3solver.mk sim3solver-ref REF=...`.
include Makefile

liborb_sim3solver.so: sim3solver.cpp sim3solver_oracle.h init.cpp init_oracle.h ../include/b200slam.h
	$(CXX) $(CXXFLAGS) -shared -o $@ sim3solver.cpp init.cpp

# The reference's OWN src/Sim3Solver.cc compiled in place against refshim/refshim_cv_sim3solver.h (behind
# refshim/sim3solver/opencv2/; it extends refshim_cv_init.h, and its arithmetic is the cv2-pinned primitives of
# sim3solver.cpp and init.cpp) with DUtils/Random.cpp, behind ref_sim3solver_glue.cpp; and the product's drop-in
# host/adapters/Sim3Solver_b200.cc behind the same glue.  Only where the reference's sources are present (REF).
S3S_FLAGS := -O2 -std=c++14 -ffp-contract=off -fPIC -shared -pthread -w -Wl,-Bsymbolic \
    -include refshim/slam_stubs_sim3solver.h -I refshim/sim3solver -I . -I ../include -I $(REF)/include -I $(REF)
S3S_DEPS := ref_sim3solver_glue.cpp sim3solver.cpp sim3solver_oracle.h init.cpp init_oracle.h \
    refshim/refshim_cv_init.h refshim/refshim_cv_sim3solver.h refshim/slam_stubs_sim3solver.h \
    refshim/sim3solver/opencv2/opencv.hpp refshim/sim3solver/opencv2/core/core.hpp ../include/b200slam.h
S3S_RANDOM := $(REF)/Thirdparty/DBoW2/DUtils/Random.cpp $(REF)/Thirdparty/DBoW2/DUtils/Timestamp.cpp
sim3solver-ref: _ref/libref_sim3solver.so sim3solver-adapters
_ref/libref_sim3solver.so: $(S3S_DEPS)
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(S3S_FLAGS) $(REF)/src/Sim3Solver.cc $(S3S_RANDOM) ref_sim3solver_glue.cpp sim3solver.cpp init.cpp -o $@
S3S_ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_sim3solver.so,)
sim3solver-adapters: $(S3S_ADAPTER_LIBS)
_ref/libadapter_sim3solver.so: $(PKG)/host/adapters/Sim3Solver_b200.cc $(S3S_DEPS) $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(S3S_FLAGS) -DB2S_ADAPTER_BUILD $(PKG)/host/adapters/Sim3Solver_b200.cc $(S3S_RANDOM) \
	    ref_sim3solver_glue.cpp sim3solver.cpp init.cpp -L$(PKG) -l:libb200slam.so \
	    -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: sim3solver-ref sim3solver-adapters
