# Builds the keyframe-culling checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_culling.so               the CPU restatement (culling.cpp)
#   _ref/libref_localmapping.so     the reference's OWN src/LocalMapping.cc, src/KeyFrame.cc and src/MapPoint.cc, compiled
#                                   in place and unmodified with their own headers, against the stand-ins of
#                                   refshim/slam_stubs_localmapping.h and refshim/refshim_cv_localmapping.h (only where the
#                                   reference's sources are present: REF)
#   _ref/libadapter_culling.so      the product's host/adapters/LocalMapping_b200.cc behind the same glue (needs
#                                   libb200slam.so, built first by build.py)
# Used as `make -f culling.mk liborb_culling.so` and `make -f culling.mk culling-ref REF=...`.
CXX ?= g++
PKG := ../self_commit_orb-slam2_b200
CULL_FLAGS := -O2 -std=c++14 -fPIC -shared -pthread -w -Wl,-Bsymbolic -include refshim/slam_stubs_localmapping.h \
    -I refshim/localmapping -I refshim -I ../include -I $(REF)/include -I $(REF)
CULL_SRCS := $(REF)/src/KeyFrame.cc $(REF)/src/MapPoint.cc $(REF)/Thirdparty/DBoW2/DBoW2/BowVector.cpp \
    $(REF)/Thirdparty/DBoW2/DBoW2/FeatureVector.cpp
CULL_DEPS := ref_culling_glue.cpp refshim/slam_stubs_localmapping.h refshim/refshim_cv_localmapping.h ../include/b200slam.h

liborb_culling.so: culling.cpp ../include/b200slam.h
	$(CXX) -O3 -march=x86-64-v3 -std=c++17 -fPIC -Wall -shared -o $@ culling.cpp

culling-ref: _ref/libref_localmapping.so culling-adapters
_ref/libref_localmapping.so: $(CULL_DEPS)
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(CULL_FLAGS) $(REF)/src/LocalMapping.cc $(CULL_SRCS) ref_culling_glue.cpp -o $@

ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_culling.so,)
culling-adapters: $(ADAPTER_LIBS)
_ref/libadapter_culling.so: $(PKG)/host/adapters/LocalMapping_b200.cc $(PKG)/host/adapters/LocalMapping_b200.h $(CULL_DEPS) \
    $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(CULL_FLAGS) -DB2S_ADAPTER_BUILD -I $(PKG)/host $(REF)/src/LocalMapping.cc $(CULL_SRCS) \
	    $(PKG)/host/adapters/LocalMapping_b200.cc ref_culling_glue.cpp -L$(PKG) -l:libb200slam.so \
	    -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: culling-ref culling-adapters
