# TEST INFRASTRUCTURE ONLY.  The reference's own pybind11 module (src/cityflow.cpp) built from the same
# priority-ordered copy of the reference as refdump_lcorder (lc_order_patch.sh explains the one change), into
# oracle/_ref/lcorder/.  With laneChange=true it is the reference whose Python surface -- vehicle ids of shadows,
# lookups by id, the replay log -- a test can compare step by step.  Run from oracle/:  make -f lc_module.mk
REF      ?= /root/reference
OUT      := _ref/lcorder
PY       ?= python3
CXX      ?= g++
EXT      := $(shell $(PY) -c "import sysconfig;print(sysconfig.get_config_var('EXT_SUFFIX'))")
PYINC    := $(shell $(PY) -m pybind11 --includes)
SRCS     := utility/utility utility/barrier engine/archive engine/engine flow/flow \
            roadnet/roadnet roadnet/trafficlight vehicle/router vehicle/vehicle vehicle/lanechange

all: $(OUT)/cityflow$(EXT)

$(OUT)/cityflow$(EXT): lc_order_patch.sh $(REF)/src/cityflow.cpp $(addprefix $(REF)/src/,$(addsuffix .cpp,$(SRCS)))
	mkdir -p $(OUT)
	set -e; tmp=$$(mktemp -d); trap 'rm -rf "$$tmp"' EXIT; cp -r $(REF)/src $$tmp/src; sh lc_order_patch.sh $$tmp/src; \
	$(CXX) -std=c++17 -O2 -fPIC -ffp-contract=off -DRAPIDJSON_HAS_STDSTRING=1 -I$$tmp/src -I$(REF)/extern/milo \
	    -I$(REF)/extern/rapidjson/include -w -shared $(PYINC) $$tmp/src/cityflow.cpp \
	    $(addprefix $$tmp/src/,$(addsuffix .cpp,$(SRCS))) -lpthread -o $@

.PHONY: all
