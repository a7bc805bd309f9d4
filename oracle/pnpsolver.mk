# Builds the EPnP RANSAC checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_pnpsolver.so   PnPsolver::iterate with the minimal sets as input, and the OpenCV C API operations EPnP calls
#                         (pnpsolver.cpp; tests/test_oracle_pnpsolver.py pins them against cv2)
#   _ref/libref_pnpsolver.so, _ref/libadapter_pnpsolver.so   (below)
# Used as `make -f pnpsolver.mk liborb_pnpsolver.so` and `make -f pnpsolver.mk pnpsolver-ref REF=...`.
include Makefile

liborb_pnpsolver.so: pnpsolver.cpp pnpsolver_oracle.h ../include/b200slam.h
	$(CXX) $(CXXFLAGS) -shared -o $@ pnpsolver.cpp

# The reference's OWN src/PnPsolver.cc compiled in place against refshim/refshim_cv_pnpsolver.h (behind
# refshim/pnpsolver/opencv2/; its arithmetic is the cv2-pinned primitives of pnpsolver.cpp) with DUtils/Random.cpp,
# behind ref_pnpsolver_glue.cpp; and the product's drop-in host/adapters/PnPsolver_b200.cc behind the same glue.  Only
# where the reference's sources are present (REF).
PNP_FLAGS := -O2 -std=c++14 -ffp-contract=off -fPIC -shared -pthread -w -Wl,-Bsymbolic \
    -include refshim/slam_stubs_pnpsolver.h -I refshim/pnpsolver -I . -I ../include -I $(REF)/include -I $(REF)
PNP_DEPS := ref_pnpsolver_glue.cpp pnpsolver.cpp pnpsolver_oracle.h refshim/refshim_cv_pnpsolver.h \
    refshim/slam_stubs_pnpsolver.h refshim/pnpsolver/opencv2/core/core.hpp ../include/b200slam.h
PNP_RANDOM := $(REF)/Thirdparty/DBoW2/DUtils/Random.cpp $(REF)/Thirdparty/DBoW2/DUtils/Timestamp.cpp
pnpsolver-ref: _ref/libref_pnpsolver.so pnpsolver-adapters
_ref/libref_pnpsolver.so: $(PNP_DEPS)
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(PNP_FLAGS) $(REF)/src/PnPsolver.cc $(PNP_RANDOM) ref_pnpsolver_glue.cpp pnpsolver.cpp -o $@
PNP_ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_pnpsolver.so,)
pnpsolver-adapters: $(PNP_ADAPTER_LIBS)
_ref/libadapter_pnpsolver.so: $(PKG)/host/adapters/PnPsolver_b200.cc $(PNP_DEPS) $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(PNP_FLAGS) -DB2S_ADAPTER_BUILD $(PKG)/host/adapters/PnPsolver_b200.cc $(PNP_RANDOM) \
	    ref_pnpsolver_glue.cpp -L$(PKG) -l:libb200slam.so \
	    -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: pnpsolver-ref pnpsolver-adapters
