# oracle/guided.mk — checkers of guided matching (DESIGN §3.9), on top of oracle/Makefile:
#   _build/liboracle_guided.so      CPU restatement (guided_oracle.cpp; travels, built anywhere)
#   _ref/libref_guided.so           the reference's own geometry_aware::GuidedMatching (both variants)
#   _ref/dropin_guided_test         Robust_model_estimation(functor, putative, true, ratio) vs the B200 shim, F / E / H
# Usage: make -f oracle/guided.mk guided-oracle | guided-ref | guided-dropin
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.PHONY: guided-oracle guided-ref guided-dropin
.DEFAULT_GOAL := guided-oracle
guided-oracle: $(BUILD)/liboracle_guided.so
guided-ref: $(OUT)/libref_guided.so
guided-dropin: $(OUT)/dropin_guided_test

$(BUILD)/liboracle_guided.so: $(HERE)guided_oracle.cpp
	@mkdir -p $(BUILD)
	$(CXX) -O2 -fPIC -std=c++17 -ffp-contract=off -shared -o $@ $(HERE)guided_oracle.cpp -lm

OMVG_GM_O := $(OBJ)/omvg/features/feature.o $(OBJ)/omvg/features/regions.o $(OBJ)/omvg/multiview/solver_fundamental_kernel.o \
             $(OBJ)/omvg/multiview/solver_homography_kernel.o $(OBJ)/omvg/numeric/numeric.o $(OBJ)/omvg/numeric/nullspace.o \
             $(OBJ)/omvg/multiview/conditioning.o $(OBJ)/omvg/multiview/projection.o
$(OUT)/libref_guided.so: $(HERE)ref_guided_driver.cpp $(OMVG_GM_O) $(STLPLUS_O)
	@mkdir -p $(OUT)
	$(CXX) $(OPT) -std=c++11 -w -shared $(OMVG_DEF) $(OMVG_INC) $(HERE)ref_guided_driver.cpp $(OMVG_GM_O) $(STLPLUS_O) -o $@ -lpthread -lm

# the essential-matrix TUs (FundamentalFromEssential, the five-point solver) as oracle/essential.mk lists them
OMVG_GD_E_O := $(patsubst %.cpp,$(OBJ)/omvg/%.o,multiview/solver_essential_five_point.cpp multiview/solver_essential_kernel.cpp \
                 multiview/essential.cpp multiview/solver_essential_three_point.cpp)
$(OUT)/dropin_guided_test: $(HERE)dropin_guided_test.cpp $(OMVG_M_O) $(STLPLUS_O) $(OMVG_GF_O) $(OMVG_GD_E_O) $(B200LIB)/libomvg_b200.so \
                           $(B200LIB)/host/GeometricFilter_B200.hpp
	$(CXX) $(OPT) -std=c++11 -w $(OMVG_DEF) $(OMVG_INC) -I$(SRC)/third_party/lemon -I$(HERE)../include \
	   $(HERE)dropin_guided_test.cpp $(OMVG_M_O) $(STLPLUS_O) $(OMVG_GF_O) $(OMVG_GD_E_O) $(OBJ)/omvg/numeric/numeric.o \
	   -L$(B200LIB) -lomvg_b200 -Wl,-rpath,'$$ORIGIN/../../openmvg_b200' -o $@ -lpthread -lm
