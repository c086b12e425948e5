# oracle/localbg_ref.mk -- TEST INFRASTRUCTURE, not product code.
#
# The reference's local amino-acid composition correction (-sc 5 / -scwin) for the tests:
#   oracle/_ref/libhhref_localbg.so      oracle/localbg_shim.cpp linked against the reference objects of
#                                        oracle/ref_build.mk (same sources, same flags)
#   oracle/_ref/hh_dropin_check_localbg  the drop-in check with --sc / --scwin (oracle/localbg_dropin.cpp; needs
#                                        libhhg.so like hh_dropin_check)
#
# Usage:  make -f oracle/localbg_ref.mk -j8        (from the repo root, after oracle/ref_build.mk)
include oracle/ref_build.mk

.DEFAULT_GOAL := localbg

localbg: $(OUT)/libhhref_localbg.so $(OUT)/hh_dropin_check_localbg

$(OUT)/libhhref_localbg.so: oracle/localbg_shim.cpp $(OUT)/libhhref.a
	$(CXX) $(CXXFLAGS) $(INC) -shared -o $@ oracle/localbg_shim.cpp \
	    -Wl,--whole-archive $(OUT)/libhhref.a -Wl,--no-whole-archive -lgomp

$(OUT)/hh_dropin_check_localbg: oracle/localbg_dropin.cpp oracle/ref_gpu_adapter.cpp $(OUT)/libhhref.a \
                                hh-suite_b200/libhhg.so include/hhg.h
	$(CXX) $(CXXFLAGS) $(INC) -o $@ oracle/localbg_dropin.cpp -Wl,--whole-archive $(OUT)/libhhref.a -Wl,--no-whole-archive \
	    -Lhh-suite_b200 -lhhg -Wl,-rpath,'$$ORIGIN/../../hh-suite_b200' -lgomp
