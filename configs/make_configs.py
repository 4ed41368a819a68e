#!/usr/bin/env python
"""Write configs/*.xml in the reference's XML schema (config/PathPlan_City.xml, UAV.xml, Trainer.xml,
buildings.xml) for the H100 plug-ins.  buildings.xml is regenerated from the city stored in
tests/golden/env_golden.npz (the 26 cylinders of the reference's config/buildings.xml, recorded by
tests/golden/make_golden.py), printed with repr() so the doubles round-trip exactly."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
g = np.load(os.path.join(HERE, "..", "tests", "golden", "env_golden.npz"))

with open(os.path.join(HERE, "buildings.xml"), "w") as f:
    f.write("<?xml version='1.0' encoding='utf-8'?>\n<buildings>\n")
    for cx, cy, cz, R, H in g["buildings"]:
        f.write("    <Threaten>\n        <Threaten_Type>building</Threaten_Type>\n        <position>\n"
                "            <x>%r</x>\n            <y>%r</y>\n            <z>%r</z>\n        </position>\n"
                "        <_R>%r</_R>\n        <_H>%r</_H>\n    </Threaten>\n" % (float(cx), float(cy), float(cz), float(R), float(H)))
    f.write("</buildings>\n")

open(os.path.join(HERE, "PathPlan_City_B200.xml"), "w").write("""<simulator>
    <env>
        <Env_Type>PathPlan_City_B200</Env_Type>
        <len>500</len>
        <width>500</width>
        <h>100</h>
        <eps>0.1</eps>
        <Is_AC>0</Is_AC>
        <Is_FL>0</Is_FL>
        <Is_On_Policy>0</Is_On_Policy>
        <FL_Loop>3</FL_Loop>
        <print_loop>2</print_loop>
        <num_UAV>4096</num_UAV>
        <scenario_pool>2048</scenario_pool>
        <Agent>
            <xml_path_agent>./configs/UAV_B200.xml</xml_path_agent>
            <Trainer>
                <Trainer_path>./configs/Trainer_DQN_B200.xml</Trainer_path>
            </Trainer>
        </Agent>
        <Obstacles>
            <buildings>./configs/buildings.xml</buildings>
        </Obstacles>
    </env>
    <record_epo>10</record_epo>
    <num_episodes>50</num_episodes>
    <max_eps_episode>1</max_eps_episode>
    <min_eps>0.1</min_eps>
    <TARGET_UPDATE>3</TARGET_UPDATE>
</simulator>
""")

open(os.path.join(HERE, "UAV_B200.xml"), "w").write("""<Agent>
    <Agent_Type>UAV</Agent_Type>
    <name>UAV_</name>
    <update_function_name>update_PathPlan27</update_function_name>
    <state_function_name>state_PathPlan</state_function_name>
    <APF_Enabled>0</APF_Enabled>
    <Min_V>0.6</Min_V>
    <Max_V>1</Max_V>
    <Steering_angle>30</Steering_angle>
    <climb_rate>1.0</climb_rate>
    <Max_Step>150</Max_Step>
    <sub_granularity>30</sub_granularity>
    <map_granularity>1</map_granularity>
</Agent>
""")

# the same UAV with the reference's flight-power block (config/UAV.xml:27-36): enables the energy accumulator
uav = open(os.path.join(HERE, "UAV_B200.xml")).read()
open(os.path.join(HERE, "UAV_energy_B200.xml"), "w").write(uav.replace("</Agent>", """    <Power_param>
        <Fly_power>
            <P_i>89</P_i>
            <v_0>4.05</v_0>
            <d_0>0.6</d_0>
            <rho>1.225</rho>
            <s>0.05</s>
            <A>0.5</A>
            <P_b>79</P_b>
            <F_b>120</F_b>
        </Fly_power>
        <Communication_power>3</Communication_power>
    </Power_param>
</Agent>"""))

for name, ttype, net, extra in (("Trainer_DQN_B200.xml", "DQN_Trainer_B200", "QValueNet_SAC", ""),
                                ("Trainer_DDQN_B200.xml", "DDQN_Trainer_B200", "QValueNet_SAC", ""),
                                ("Trainer_DuelingDQN_B200.xml", "DuelingDQN_Trainer_B200", "VAnet2", "")):
    open(os.path.join(HERE, name), "w").write("""<Trainer>
    <Trainer_Type>%s</Trainer_Type>
    <Is_Train>1</Is_Train>
    <NetWork>%s</NetWork>
    <h>1</h>
    <w>100</w>
    <channel>1</channel>
    <hiden_dim>64</hiden_dim>
    <output>27</output>
    <replay_size>1048576</replay_size>
    <LEARNING_RATE>0.0005</LEARNING_RATE>
    <Batch_Size>4096</Batch_Size>
    <gamma>0.99</gamma>
    <Update_loop>3</Update_loop>
    <max_epoch>100</max_epoch>
    <save_loop>1000000000</save_loop>
</Trainer>
""" % (ttype, net))
# SAC with discrete actions (SAC_Trainer's IS_Continuous = 0 branch, PolicyNet_SAC / QValueNet_SAC) on the 27-action step:
# the shipped SAC learning rates, alpha lr, tau, gamma and target entropy (config/Trainer.xml)
open(os.path.join(HERE, "Trainer_SAC_discrete_B200.xml"), "w").write("""<Trainer>
    <Trainer_Type>SAC_Trainer_B200</Trainer_Type>
    <Is_Train>1</Is_Train>
    <IsPriority_Replay>0</IsPriority_Replay>
    <actor>
        <NetWork>PolicyNet_SAC</NetWork>
        <h>1</h>
        <w>100</w>
        <channel>1</channel>
        <hiden_dim>64</hiden_dim>
        <output>27</output>
        <lr>0.0001</lr>
    </actor>
    <critic>
        <NetWork>QValueNet_SAC</NetWork>
        <h>1</h>
        <w>100</w>
        <channel>1</channel>
        <hiden_dim>64</hiden_dim>
        <output>27</output>
        <lr>0.001</lr>
    </critic>
    <SAC_param>
        <IS_Continuous>0</IS_Continuous>
        <alpha_lr>0.0001</alpha_lr>
        <target_entropy>1</target_entropy>
        <gamma>0.99</gamma>
        <tau>0.05</tau>
    </SAC_param>
    <replay_size>1048576</replay_size>
    <LEARNING_RATE>0.0005</LEARNING_RATE>
    <Batch_Size>4096</Batch_Size>
    <max_epoch>100</max_epoch>
    <save_loop>1000000000</save_loop>
</Trainer>
""")
print("wrote", sorted(os.listdir(HERE)))
