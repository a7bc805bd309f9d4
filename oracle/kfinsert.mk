# Builds the keyframe-insertion checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_kfinsert.so              the CPU restatement (kfinsert.cpp)
#   _ref/libref_kfinsert.so         the reference's OWN src/LocalMapping.cc, src/KeyFrame.cc and src/MapPoint.cc, compiled
#                                   in place and unmodified, against refshim/slam_stubs_kfinsert.h and
#                                   refshim/refshim_cv_kfinsert.h (the OpenCV forms UpdateNormalAndDepth takes, and a
#                                   real DescriptorDistance), behind
#                                   ref_kfinsert_glue.cpp (only where the reference's sources are present: REF)
#   _ref/libadapter_kfinsert.so     the product's host/adapters/LocalMapping_b200.cc behind the same glue (needs
#                                   libb200slam.so, built first by build.py)
# Every float expression is compiled as written: -ffp-contract=off.
# Used as `make -f kfinsert.mk liborb_kfinsert.so` and `make -f kfinsert.mk kfinsert-ref REF=...`.
CXX ?= g++
PKG := ../self_commit_orb-slam2_b200
KFI_FLAGS := -O2 -std=c++14 -fPIC -shared -pthread -w -ffp-contract=off -Wl,-Bsymbolic \
    -include refshim/slam_stubs_kfinsert.h -I refshim/kfinsert -I refshim -I ../include -I $(REF)/include -I $(REF)
KFI_SRCS := $(REF)/src/LocalMapping.cc $(REF)/src/KeyFrame.cc $(REF)/src/MapPoint.cc \
    $(REF)/Thirdparty/DBoW2/DBoW2/BowVector.cpp $(REF)/Thirdparty/DBoW2/DBoW2/FeatureVector.cpp
KFI_DEPS := ref_kfinsert_glue.cpp refshim/slam_stubs_kfinsert.h refshim/refshim_cv_kfinsert.h ../include/b200slam.h

liborb_kfinsert.so: kfinsert.cpp ../include/b200slam.h
	$(CXX) -O3 -march=x86-64-v3 -ffp-contract=off -std=c++17 -fPIC -Wall -shared -o $@ kfinsert.cpp

kfinsert-ref: _ref/libref_kfinsert.so kfinsert-adapters
_ref/libref_kfinsert.so: $(KFI_DEPS)
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(KFI_FLAGS) $(KFI_SRCS) ref_kfinsert_glue.cpp -o $@

ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_kfinsert.so,)
kfinsert-adapters: $(ADAPTER_LIBS)
_ref/libadapter_kfinsert.so: $(PKG)/host/adapters/LocalMapping_b200.cc $(PKG)/host/adapters/LocalMapping_b200.h \
    $(KFI_DEPS) $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(KFI_FLAGS) -DB2S_ADAPTER_BUILD -I $(PKG)/host $(KFI_SRCS) $(PKG)/host/adapters/LocalMapping_b200.cc \
	    ref_kfinsert_glue.cpp -L$(PKG) -l:libb200slam.so -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: kfinsert-ref kfinsert-adapters
