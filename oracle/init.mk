# Builds the monocular initialiser's CPU restatement (test infrastructure), next to the oracle of Makefile:
#   liborb_init.so   Initializer::Initialize with the minimal sets as input, and the OpenCV linear algebra it needs
#                    (init.cpp; tests/test_oracle_init.py pins the linear algebra against cv2)
#   _ref/libref_init.so, _ref/libadapter_init.so   (below)
# Used as `make -f init.mk liborb_init.so` and `make -f init.mk init-ref REF=...`.
include Makefile

liborb_init.so: init.cpp init_oracle.h ../include/b200slam.h
	$(CXX) $(CXXFLAGS) -shared -o $@ init.cpp

# The reference's OWN src/Initializer.cc compiled in place against refshim/refshim_cv_init.h (behind
# refshim/init/opencv2/opencv.hpp; its arithmetic is init.cpp's cv2-pinned primitives) with DUtils/Random.cpp, behind
# ref_init_glue.cpp; and the product's drop-in host/adapters/Initializer_b200.cc behind the same glue.  Only where the
# reference's sources are present (REF): `make -f init.mk init-ref REF=...`.
INIT_FLAGS := -O2 -std=c++14 -ffp-contract=off -fPIC -shared -pthread -w -Wl,-Bsymbolic -include refshim/slam_stubs_init.h \
    -I refshim/init -I . -I ../include -I $(REF)/include -I $(REF)
INIT_DEPS := ref_init_glue.cpp init.cpp init_oracle.h refshim/refshim_cv_init.h refshim/slam_stubs_init.h \
    refshim/init/opencv2/opencv.hpp ../include/b200slam.h
INIT_RANDOM := $(REF)/Thirdparty/DBoW2/DUtils/Random.cpp $(REF)/Thirdparty/DBoW2/DUtils/Timestamp.cpp
init-ref: _ref/libref_init.so init-adapters
_ref/libref_init.so: $(INIT_DEPS)
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(INIT_FLAGS) $(REF)/src/Initializer.cc $(INIT_RANDOM) ref_init_glue.cpp init.cpp -o $@
INIT_ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_init.so,)
init-adapters: $(INIT_ADAPTER_LIBS)
_ref/libadapter_init.so: $(PKG)/host/adapters/Initializer_b200.cc $(INIT_DEPS) $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(INIT_FLAGS) -DB2S_ADAPTER_BUILD $(PKG)/host/adapters/Initializer_b200.cc $(INIT_RANDOM) ref_init_glue.cpp \
	    init.cpp -L$(PKG) -l:libb200slam.so -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: init-ref init-adapters
