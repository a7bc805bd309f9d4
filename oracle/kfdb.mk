# Builds the keyframe-database checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_kfdb.so         the CPU restatement (kfdb.cpp)
#   _ref/libref_kfdb.so    the reference's OWN src/KeyFrameDatabase.cc, compiled in place and unmodified, against the
#                          stand-in KeyFrame / Frame of refshim/slam_stubs_kfdb.h and the vendored DBoW2 as ORBVocabulary
#                          (only where the reference's sources are present: REF)
#   _ref/libadapter_kfdb.so the product's drop-in host/adapters/KeyFrameDatabase_b200.cc behind the same glue (needs
#                          libb200slam.so, built first by build.py)
# Used as `make -f kfdb.mk liborb_kfdb.so` and `make -f kfdb.mk ref REF=...`.
# REF: the reference's source tree (build.py passes it; the ref target needs it).
CXX ?= g++
PKG := ../self_commit_orb-slam2_b200
DBOW := $(REF)/Thirdparty/DBoW2
KFDB_FLAGS := -O2 -std=c++14 -ffp-contract=off -fPIC -shared -pthread -w -Wl,-Bsymbolic -include refshim/slam_stubs_kfdb.h \
    -I refshim -I $(REF)/include -I $(REF) -I $(DBOW)
# (DBoW2 must share the process's libstdc++.so, see Makefile)
KFDB_DBOW := $(DBOW)/DBoW2/BowVector.cpp $(DBOW)/DBoW2/FeatureVector.cpp $(DBOW)/DBoW2/ScoringObject.cpp $(DBOW)/DBoW2/FORB.cpp $(DBOW)/DUtils/Random.cpp \
    $(DBOW)/DUtils/Timestamp.cpp -nostdlib++ -l:libstdc++.so.6

liborb_kfdb.so: kfdb.cpp
	$(CXX) -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -std=c++17 -fPIC -Wall -shared -o $@ kfdb.cpp

ref: _ref/libref_kfdb.so adapters
_ref/libref_kfdb.so: ref_kfdb_glue.cpp refshim/slam_stubs_kfdb.h refshim/refshim_cv.h
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(KFDB_FLAGS) $(REF)/src/KeyFrameDatabase.cc ref_kfdb_glue.cpp $(KFDB_DBOW) -o $@

ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_kfdb.so,)
adapters: $(ADAPTER_LIBS)
_ref/libadapter_kfdb.so: $(PKG)/host/adapters/KeyFrameDatabase_b200.cc ref_kfdb_glue.cpp refshim/slam_stubs_kfdb.h \
    ../include/b200slam.h $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(KFDB_FLAGS) -DB2S_ADAPTER_BUILD -I ../include $(PKG)/host/adapters/KeyFrameDatabase_b200.cc ref_kfdb_glue.cpp \
	    $(KFDB_DBOW) -L$(PKG) -l:libb200slam.so -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: ref adapters
