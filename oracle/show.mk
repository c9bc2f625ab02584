# TEST INFRASTRUCTURE ONLY.  make -C oracle -f show.mk show
# Builds oracle/_ref/libdsm_ref_show.so: the serial reference oracle of the `ref` target of oracle/Makefile (same
# compiler and flags) plus the debug_show hook of ref_debug_show.cpp, with oracle/shim_show first on the include path
# (its cv::imshow keeps the image shown).  Skipped where the reference sources are absent.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

show:
	@if [ -f $(REF_SRC)/fusion_functions.cpp ]; then \
	  mkdir -p $(OUT) && \
	  $(CXX) -I$(HERE)shim_show $(REF_FLAGS) -DDSM_REF_SERIAL -ftrivial-auto-var-init=zero -o $(OUT)/libdsm_ref_show.so $(HERE)ref_debug_show.cpp && \
	  echo "built serial reference oracle with the debug_show hook into $(OUT)"; \
	else echo "reference sources not present at $(REF_SRC): keeping prebuilt $(OUT)/libdsm_ref_show.so"; fi
.PHONY: show
